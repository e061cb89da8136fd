"""Time the upright warp (csrc/rectify.cuh) with CUDA events and torch.profiler, in one process:

    python tools/rectify_bench.py [--iters 20] [--out results/rectify_bench.json]

``rectify.upright`` on 256 seeded uint8 images of 640 x 480 x 3 -> 640 x 480, bilinear, with device-resident cameras (roll and
pitch in [-30, 30] degrees, general vfov in [50, 90]), for each focal mode.  The bytes moved are the input read plus the
output written; a device-to-device copy of as many bytes is timed in the same run.  Prints one JSON object with the GPU's name
and power limit."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from metrics_bench import copy_ms, gpu_info, kernel_ms, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rectify_bench needs a CUDA device")
    from perspectivefields_b200 import rectify

    n, h, w = 256, 480, 640
    g = torch.Generator(device="cuda").manual_seed(0)
    imgs = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g).unbind(0)
    u = lambda lo, hi: (torch.rand(n, dtype=torch.float64, device="cuda", generator=g) * (hi - lo) + lo).unbind(0)
    roll, pitch, gv = u(-30, 30), u(-30, 30), u(50, 90)
    zero = torch.zeros(n, dtype=torch.float64, device="cuda").unbind(0)
    cams = [dict(zip(rectify.CAMERA_KEYS, c)) for c in zip(roll, pitch, gv, zero, zero)]
    nbytes = n * h * w * 3                       # read, and as many written
    res = {"gpu": gpu_info(), "images": n, "size": [h, w], "bytes_moved": 2 * nbytes, "cases": {}}
    cms = copy_ms(nbytes, args.iters)
    res["copy_ms_same_bytes"] = cms
    for focal in ("same", "fill", 60.0):
        fn = lambda: rectify.upright(imgs, cams, focal=focal, outputs=())
        ms = timed(fn, args.iters)
        km = kernel_ms(fn, "rectify_")
        warp = sum(v for k, v in km.items() if "warp" in k)
        st = torch.bincount(fn()["status"], minlength=3).tolist()
        res["cases"][str(focal)] = {"ms_per_call": ms, "views_per_s": n / ms * 1e3, "kernel_ms_per_call": km,
                                    "warp_GB_per_s": 2 * nbytes / warp / 1e6 if warp else None,
                                    "warp_time_over_copy_time": warp / cms if warp else None, "status_counts": st}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
