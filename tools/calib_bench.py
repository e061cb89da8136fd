"""Time the camera fit (csrc/calib.cuh) with CUDA events and torch.profiler, in one process:

    python tools/calib_bench.py [--iters 10] [--out results/calib_bench.json]

* ``fit_camera`` on 256 seeded noisy camera fields of 640 x 480 (2 degrees of angular noise on up, 1 degree on latitude, 1 %
  outliers): centred least squares, and uncentred Huber (delta 2 degrees);
* ``inference_batch`` of PersNet-360Cities on 32 images of 640 x 480, alone and followed by ``fit_camera``.

Each pass reads 12 B per pixel (two float32 up components and one latitude), 0.94 GB for the batch; a device-to-device copy
that reads as many bytes is timed in the same run.  Prints one JSON object with the GPU's name and power limit."""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from metrics_bench import copy_ms, gpu_info, kernel_ms, timed  # noqa: E402


def noisy_batch(n, h, w, seed=0):
    from perspectivefields_b200 import panocam

    g = torch.Generator().manual_seed(seed)
    u = lambda lo, hi: (torch.rand(n, generator=g, dtype=torch.float64) * (hi - lo) + lo).tolist()
    roll, pitch, vfov = u(-40, 40), u(-60, 60), u(35, 100)
    cx, cy = u(-0.1, 0.1), u(-0.1, 0.1)
    focal = [1 / (2 * math.tan(math.radians(v) / 2)) for v in vfov]
    ups, lats = panocam.camera_fields(focal, [h] * n, [w] * n, [math.radians(p) for p in pitch], [math.radians(r) for r in roll], cx, cy)
    gd = torch.Generator(device="cuda").manual_seed(seed)
    up = torch.stack(ups).permute(0, 3, 1, 2)                                  # [n, 2, H, W] view of the [n, H, W, 2] fields
    ang = torch.atan2(up[:, 1], up[:, 0]) + math.radians(2.0) * torch.randn((n, h, w), generator=gd, device="cuda")
    out = torch.rand((n, h, w), generator=gd, device="cuda") < 0.01
    ang = torch.where(out, (torch.rand((n, h, w), generator=gd, device="cuda") * 2 - 1) * math.pi, ang)
    pu = torch.stack([torch.cos(ang), torch.sin(ang)], dim=1).contiguous()
    pl = (torch.stack(lats) + torch.randn((n, h, w), generator=gd, device="cuda")).contiguous()
    return [{"pred_gravity_original": a, "pred_latitude_original": b} for a, b in zip(pu.unbind(0), pl.unbind(0))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("calib_bench needs a CUDA device")
    import pf_test_util as U
    from oracle import weights_gen as wg
    from perspectivefields_b200 import calibrate

    res = {"gpu": gpu_info(), "cases": {}}
    n, h, w = 256, 480, 640
    results = noisy_batch(n, h, w)
    nbytes = 12 * n * h * w
    cms = copy_ms(nbytes, args.iters)
    for name, kw in (("centred_l2", {"principal_point": False}), ("uncentred_huber", {"principal_point": True, "huber": math.radians(2.0)})):
        fn = lambda: calibrate.fit_camera(results, **kw)
        ms = timed(fn, args.iters)
        out = fn()
        its = torch.stack([o["fit_iterations"] for o in out]).float()
        st = torch.stack([o["fit_status"] for o in out])
        km = kernel_ms(fn, "fit_")
        pass_ms = sum(v for k, v in km.items() if "pass" in k)
        batch_passes = float(its.mean())      # evaluations of the whole batch's pixels (blocks of stopped images exit at once)
        res["cases"][name] = {
            "ms_per_call": ms, "launched_pass_pairs": int(its.max()), "mean_evaluations": batch_passes,
            "status_counts": torch.bincount(st, minlength=3).tolist(), "pixel_passes_per_s": float(its.sum()) * h * w / ms * 1e3,
            "kernel_ms_per_call": km, "pass_kernel_ms_per_batch_pass": pass_ms / batch_passes, "bytes_per_batch_pass": nbytes,
            "pass_GB_per_s": nbytes / (pass_ms / batch_passes) / 1e6, "copy_ms_same_bytes_read": cms,
            "pass_time_over_copy_time": (pass_ms / batch_passes) / cms}
    del results
    m = U.make_model("PersNet-360Cities", seed=0, device="cuda")[0]
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(32, h, w, seed=1)]
    inf_ms = timed(lambda: m.inference_batch(imgs), max(args.iters // 2, 3))
    both_ms = timed(lambda: calibrate.fit_camera(m.inference_batch(imgs)), max(args.iters // 2, 3))
    res["cases"]["inference_then_fit_b32_640x480"] = {"inference_ms": inf_ms, "inference_and_fit_ms": both_ms, "fit_share": (both_ms - inf_ms) / both_ms}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
