"""Time pf_draw_fields (the perspective-field overlay of draw_perspective_fields, batched) on one GPU; print one JSON line.

    python tools/draw_bench.py [--canvases 256] [--density 10] [--reps 50] [--out DIR]

256 canvases of 640 x 480 (latitude fill and lines + 8 x 11 arrows each) in one call, CUDA events around many calls after a
warm-up.  Bytes the kernel must move: 3 (image) + 4 (latitude) + 3 (output) B per pixel; the up field is read at the arrow
lattice only.  The achieved GB/s is compared with the HBM copy rate measured in the same run (a device-to-device copy of
1 GiB): a kernel far below it is bound by its arithmetic (16 samples per pixel), not by HBM.  The card's name and power limit
are read in the same run.  With --out, one canvas is written as a PNG there."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from perspectivefields_b200 import _batch, panocam, viz  # noqa: E402


def card(index):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:     # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(index), "power_limit": f"unavailable ({type(e).__name__})"}


def copy_peak(dev):
    a = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
    b = torch.empty_like(a)
    best = 0.0
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); b.copy_(a); e1.record()
        torch.cuda.synchronize()
        best = max(best, 2 * a.numel() / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    del a, b
    torch.cuda.empty_cache()
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--canvases", type=int, default=256)
    ap.add_argument("--density", type=int, default=10)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("draw_bench.py needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    n, H, W = a.canvases, 480, 640
    rs = np.random.RandomState(0)
    el, roll = rs.uniform(-0.6, 0.6, n), rs.uniform(-0.4, 0.4, n)
    focal = rs.uniform(0.6, 1.6, n)
    ups, lats = panocam.camera_fields(focal, [H] * n, [W] * n, el, roll, [0.0] * n, [0.0] * n, dev)
    lats = [torch.deg2rad(l) for l in lats]
    imgs = [t for t in torch.randint(0, 256, (n, H, W, 3), dtype=torch.uint8, device=dev)]
    ups_c = [_batch.up_view(u, H, W) for u in ups]

    def call():
        return viz._draw(imgs, ups_c, lats, [viz.GREEN] * n, a.density, 20, 0.4, 0.9)

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.reps
    bytes_ = n * H * W * (3 + 4 + 3)
    gbs = bytes_ / (ms * 1e-3) / 1e9
    peak = copy_peak(dev)
    res = {"metric": "draw_fields", "canvas": f"{W}x{H}", "canvases": n, "density": a.density, "ms_per_call": round(ms, 3),
           "canvases_per_s": round(n / (ms * 1e-3), 1), "GB_per_s": round(gbs, 1), "hbm_copy_GB_per_s": round(peak, 1),
           "hbm_fraction": round(gbs / peak, 3), "bound": "HBM" if gbs / peak > 0.6 else "arithmetic", **card(dev.index)}
    if a.out:
        from PIL import Image
        os.makedirs(a.out, exist_ok=True)
        Image.fromarray(call()[0].cpu().numpy()).save(os.path.join(a.out, "draw_bench_canvas0.png"))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
