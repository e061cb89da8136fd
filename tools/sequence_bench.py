"""Camera-track fit benchmark: calibrate.fit_camera(groups=..., smoothness=...) on jittered-track camera fields, 1024 frames of
640 x 480 as 4 sequences of 256 and as 1 of 1024, and a 256-frame "fit, then rectify.upright(focal="fill_common")" pipeline.
Prints one JSON line: the GPU and its power limit; per layout the ms per call, evaluations, status counts, the pass, reduce and
sequence-step kernel ms (torch.profiler, a separate run) with the step's share of each evaluation, and the track RMS error
(degrees) of the smoothed, per-frame and grouped fits against the true track.

    python tools/sequence_bench.py [--frames 1024] [--sigma 0.1] [--reps 5]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from perspectivefields_b200 import calibrate, panocam, rectify  # noqa: E402

H, W = 480, 640


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        name, power = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
    except Exception:   # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def track(n, seed=0):
    """A slow sinusoidal roll / pitch track (degrees) with N(0, 1 degree) jitter per frame: (true [n, 2], jittered [n, 2])."""
    t = np.arange(n)
    true = np.stack([6.0 * np.sin(2 * np.pi * t / 600.0) + 2.0, 4.0 * np.cos(2 * np.pi * t / 800.0) - 3.0], axis=1)
    return true, true + np.random.default_rng(seed).normal(0.0, 1.0, (n, 2))


def fields(cams):
    ups, lats = panocam.camera_fields([0.8] * len(cams), [H] * len(cams), [W] * len(cams), np.radians(cams[:, 1]).tolist(),
                                      np.radians(cams[:, 0]).tolist(), [0.0] * len(cams), [0.0] * len(cams))
    return [{"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l} for u, l in zip(ups, lats)]


def rms(out, true):
    got = np.array([[float(o["pred_roll"]), float(o["pred_pitch"])] for o in out])
    return float(np.sqrt(np.mean((got - true) ** 2)))


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def kernel_ms(fn):
    """ms per call of the fit's pass, reduce and sequence-step kernels (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {"pass": 0.0, "reduce": 0.0, "step": 0.0}
    for e in prof.key_averages():
        for key, pat in (("pass", "fit_pass_kernel"), ("reduce", "fit_reduce_kernel"), ("step", "fit_seq_step_kernel")):
            if pat in e.key:
                tot[key] += e.device_time_total / 1e3
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--sigma", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-iterations", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sequence_bench needs a CUDA device")
    name, power = gpu_info()
    n = args.frames
    true, cams = track(n)
    res = fields(cams)
    out = {"gpu": name, "power_limit": power, "frames": n, "size": [H, W], "sigma_deg": args.sigma, "max_iterations": args.max_iterations}
    per_frame = calibrate.fit_camera(res, max_iterations=args.max_iterations)
    out["rms_per_frame_deg"] = rms(per_frame, true)
    for nseq in (4, 1):
        L = n // nseq
        groups = [i // L for i in range(n)]
        fit = lambda: calibrate.fit_camera(res, groups=groups, smoothness=args.sigma, max_iterations=args.max_iterations)
        ms = timed(fit, args.reps)
        r = fit()
        evals = int(r[0]["fit_iterations"]) if nseq == 1 else max(int(o["fit_iterations"]) for o in r)
        st = [int(o["fit_status"]) for o in r]
        k = kernel_ms(fit)
        launches = args.max_iterations   # the step kernels run every launch; stopped sequences exit at once
        grouped = calibrate.fit_camera(res, groups=groups, max_iterations=args.max_iterations)
        out[f"{nseq}x{L}"] = {"ms_per_call": ms, "evaluations": evals, "status_counts": {s: st.count(s) for s in sorted(set(st))},
                              "pass_ms": k["pass"], "reduce_ms": k["reduce"], "step_ms": k["step"],
                              "step_share_of_evaluation": k["step"] / max(k["pass"] + k["reduce"] + k["step"], 1e-12),
                              "step_ms_per_launch": k["step"] / launches,
                              "rms_smoothed_deg": rms(r, true), "rms_grouped_deg": rms(grouped, true)}
    del res
    torch.cuda.empty_cache()
    m = 256
    res = fields(cams[:m])
    imgs = [torch.from_numpy(np.random.default_rng(k).integers(0, 256, (H, W, 3), dtype=np.uint8)).cuda() for k in range(m)]

    def pipeline():
        c = calibrate.fit_camera(res, groups=[0] * m, smoothness=args.sigma, max_iterations=args.max_iterations)
        return rectify.upright(imgs, c, focal="fill_common")

    out["pipeline_256_ms"] = timed(pipeline, args.reps)
    p = pipeline()
    out["pipeline_256_status_counts"] = {s: int((p["status"] == s).sum()) for s in (0, 1, 2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
