"""Time pf_pano_views (PanoCam.crop_distortion, batched) on one GPU and print one JSON line.

    python tools/pano_bench.py [--views 256] [--reps 50]

A seeded 2048 x 1024 panorama and 256 views of 640 x 480 mixing xi in {0, 0.5, 0.9}; CUDA events around many launches after a
warm-up.  Two runs: every output (crop + ntheta + nphi + up + lat + xy_map: 31 B/pixel) and crop + up + lat (15 B/pixel).  Written
GB/s is compared with the write-only peak measured in the same run (the better of torch's fill_ and pf_op_fill_stream over 1 GiB,
as bench.py measures it).  If both runs reach the same fraction of that peak the kernel is bound by its stores; if the smaller
run's bandwidth falls well below, by its float64 arithmetic (the per-pixel work is the same in both runs except the reverse
projection of ``up``).  The oracle's CPU time for a few views is printed for context, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle_pano as op  # noqa: E402
from perspectivefields_b200 import _native  # noqa: E402

FIELDS = ("ntheta", "nphi", "up", "lat", "xy_map")


def write_peak(L, dev):
    a = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    best = 0.0
    for fn in (lambda: a.fill_(3), lambda: _native.check(L.pf_op_fill_stream(a.data_ptr(), a.numel() // 4, 1.0, st))):
        for _ in range(4):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            best = max(best, a.numel() / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    del a
    torch.cuda.empty_cache()
    return best


def card(index):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:     # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(index), "power_limit": f"unavailable ({type(e).__name__})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=256)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--oracle-views", type=int, default=3)
    a = ap.parse_args()
    L = _native.lib()
    dev = torch.device("cuda", torch.cuda.current_device())
    rs = np.random.RandomState(0)
    pano = op.make_panorama(0, 1024, 2048)
    H, W, n = 480, 640, a.views
    views = [(float(rs.uniform(250, 600)), [0.0, 0.5, 0.9][i % 3], H, W, float(rs.uniform(-180, 180)), float(rs.uniform(-30, 30)),
              float(rs.uniform(-10, 10))) for i in range(n)]
    descs = (_native.pf_pano_view * n)()
    for i, v in enumerate(views):
        descs[i] = _native.pf_pano_view(H, W, *v[:2], *v[4:], i * 3 * H * W, i * H * W)
    src = torch.from_numpy(pano).to(dev)
    im = torch.empty(n * 3 * H * W, dtype=torch.uint8, device=dev)
    blobs = {k: torch.empty((2 if k in ("up", "xy_map") else 1) * n * H * W, dtype=torch.float32, device=dev) for k in FIELDS}
    offset = torch.empty(n, dtype=torch.float64, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    peak = write_peak(L, dev)

    def run(sel):
        p = lambda k: blobs[k].data_ptr() if k in sel else None
        _native.check(L.pf_pano_views(dev.index, src.data_ptr(), pano.shape[0], pano.shape[1], descs, n, im.data_ptr(), p("ntheta"),
                                      p("nphi"), p("up"), p("lat"), p("xy_map"), offset.data_ptr(), status.data_ptr(), st))

    res = {"workload": f"pf_pano_views: {n} views of {W}x{H} (xi 0 / 0.5 / 0.9) from a 2048x1024 uint8 panorama", "write_peak_GBps": round(peak, 1)}
    for name, sel in (("all_outputs", FIELDS), ("im_up_lat", ("up", "lat"))):
        for _ in range(5):
            run(sel)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            run(sel)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.reps
        bpp = 3 + sum(8 if k in ("up", "xy_map") else 4 for k in sel)
        gbs = n * H * W * bpp / (ms * 1e-3) / 1e9
        res[name] = {"ms_per_call": round(ms, 3), "views_per_s": round(n / (ms * 1e-3), 1), "bytes_per_pixel": bpp,
                     "written_GBps": round(gbs, 1), "frac_of_write_peak": round(gbs / peak, 3)}
    fa, fb = res["all_outputs"]["frac_of_write_peak"], res["im_up_lat"]["frac_of_write_peak"]
    res["bound_by"] = "stores" if fb > 0.8 * fa else "float64 arithmetic (special functions)"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        t0 = time.perf_counter()
        for v in views[:a.oracle_views]:
            op.crop_distortion_full(pano, *v)
        res["oracle_cpu_s_per_view"] = round((time.perf_counter() - t0) / a.oracle_views, 3)
    res.update(card(dev.index))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
