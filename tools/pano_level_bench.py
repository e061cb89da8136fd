"""Time panorama levelling with CUDA events, in one process:

    python tools/pano_level_bench.py [--iters 10] [--out results/pano_level_bench.json]

* ``rectify.rotate_panoramas`` on 64 uint8 panoramas of 2048 x 1024 x 3 (seeded, random rotations, bilinear), the kernel alone
  (torch.profiler) and the whole call, next to a device-to-device copy of the same bytes;
* ``calibrate.fit_panorama`` for 64 panoramas x 8 views of 320 x 320 (rectify.DEFAULT_LEVEL_VIEWS; exact fields of the views'
  effective cameras under seeded tilts, with seeded noise), least squares, 50 evaluations at most;
* one ``rectify.level_panoramas`` call on 16 of the panoramas with a seeded random-weights PersNet-360Cities model.

Prints one JSON object with the GPU's name and power limit."""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from metrics_bench import gpu_info, kernel_ms, timed  # noqa: E402


def random_rotations(n, deg, seed):
    """n rotations by up to deg degrees about random axes, float64 [n, 3, 3] on the host."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = rng.standard_normal(3)
        k /= np.linalg.norm(k)
        K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
        a = math.radians(rng.uniform(-deg, deg))
        out.append(np.eye(3) + math.sin(a) * K + (1.0 - math.cos(a)) * K @ K)
    return out


def fit_inputs(npano, seed):
    """Noisy exact fields of DEFAULT_LEVEL_VIEWS' effective cameras under seeded tilts -> (results, views, panorama_of)."""
    import oracle_pano_level as opl
    from perspectivefields_b200 import panocam, rectify
    rng = np.random.default_rng(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    views = list(rectify.DEFAULT_LEVEL_VIEWS)
    foc, hs, ws, els, rolls = [], [], [], [], []
    for _ in range(npano):
        T = opl.tilt(math.radians(rng.uniform(-20, 20)), math.radians(rng.uniform(-20, 20)))
        for vfov, w, h, az, el, roll, ar in views:
            _, e2, r2 = opl.decompose(T @ opl.crop_rotation(az, el, roll))
            foc.append(opl.crop_focal(vfov, w, ar) / h); hs.append(h); ws.append(w); els.append(math.radians(e2)); rolls.append(math.radians(r2))
    n = len(hs)
    ups, lats = panocam.camera_fields(foc, hs, ws, els, rolls, [0.0] * n, [0.0] * n, "cuda")
    results = [{"pred_gravity_original": (u + 0.03 * torch.randn(u.shape, generator=g, device="cuda")).permute(2, 0, 1),
                "pred_latitude_original": l + torch.randn(l.shape, generator=g, device="cuda")} for u, l in zip(ups, lats)]
    return results, views * npano, [P for P in range(npano) for _ in views]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pano_level_bench needs a CUDA device")
    import pf_test_util as U
    from perspectivefields_b200 import calibrate, rectify

    res = {"gpu": gpu_info(), "cases": {}}
    n, hp, wp = 64, 1024, 2048
    gen = torch.Generator(device="cuda").manual_seed(0)
    blob = torch.randint(0, 256, (n, hp, wp, 3), dtype=torch.uint8, generator=gen, device="cuda")
    panos = list(blob.unbind(0))
    rots = torch.from_numpy(np.stack(random_rotations(n, 30.0, 1))).cuda()
    rotate = lambda: rectify.rotate_panoramas(panos, rots)
    dst = torch.empty_like(blob)
    copy = lambda: dst.copy_(blob)
    nbytes = 2 * blob.numel()
    case = {"bytes_read_and_written": nbytes}
    case["call_ms"] = timed(rotate, args.iters)
    case["kernel_ms"] = sum(kernel_ms(rotate, "rotate_panoramas_kernel").values())
    case["copy_ms"] = timed(copy, args.iters)
    case["kernel_GBps"] = nbytes / case["kernel_ms"] / 1e6
    case["copy_GBps"] = nbytes / case["copy_ms"] / 1e6
    res["cases"]["rotate_64_2048x1024x3_u8_bilinear"] = case
    del blob, dst, panos
    torch.cuda.empty_cache()

    results, views, pano_of = fit_inputs(64, 2)
    fit = lambda: calibrate.fit_panorama(results, views, pano_of)
    its = torch.stack([f["fit_iterations"] for f in fit()]).float()
    res["cases"]["fit_panorama_64x8_320x320_l2"] = {"ms": timed(fit, args.iters), "mean_evaluations": float(its.mean())}

    model = U.make_model("PersNet-360Cities", seed=0, device="cuda")[0]
    small = [torch.randint(0, 256, (hp, wp, 3), dtype=torch.uint8, generator=gen, device="cuda") for _ in range(16)]
    level = lambda: rectify.level_panoramas(model, small)
    res["cases"]["level_panoramas_16_2048x1024_8x320x320"] = {"ms": timed(level, max(1, args.iters // 2), warmup=2)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
