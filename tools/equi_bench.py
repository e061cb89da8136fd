"""Time pf_equi_views (PanoCam.crop_equi, batched) on one GPU and print one JSON line.

    python tools/equi_bench.py [--views 256] [--reps 50]

A seeded 2048 x 1024 RGB panorama and 256 pinhole views of 640 x 480 (vfov 50-90 degrees, any azimuth, elevation within
+-30, roll within +-10); CUDA events around many launches after a warm-up.  Three runs: uint8 bilinear (the crop_equi /
get_image case), float32 bilinear (12 B written per pixel instead of 3) and uint8 nearest.  Written GB/s is compared with the
write-only peak measured in the same run (tools/pano_bench.py's write_peak).  For context, pf_pano_views writing only the crop
of the same views (xi = 0, f from the same vfov) is timed too.  The card's name and power limit are printed with the numbers."""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle_pano as op  # noqa: E402
from pano_bench import card, write_peak  # noqa: E402
from perspectivefields_b200 import _native  # noqa: E402


def timed(fn, reps):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=256)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    L = _native.lib()
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream(dev).cuda_stream
    rs = np.random.RandomState(0)
    pano = op.make_panorama(0, 1024, 2048)
    H, W, n = 480, 640, a.views
    views = [(float(rs.uniform(50, 90)), float(rs.uniform(-180, 180)), float(rs.uniform(-30, 30)), float(rs.uniform(-10, 10))) for _ in range(n)]
    peak = write_peak(L, dev)
    res = {"workload": f"pf_equi_views: {n} views of {W}x{H} from a 2048x1024 RGB panorama", "write_peak_GBps": round(peak, 1)}
    srcs = {"uint8": torch.from_numpy(pano).to(dev), "float32": torch.from_numpy(pano.astype(np.float32)).to(dev)}
    for name, dtype, mode in (("uint8_bilinear", "uint8", 0), ("float32_bilinear", "float32", 0), ("uint8_nearest", "uint8", 1)):
        es = 4 if dtype == "float32" else 1
        descs = (_native.pf_equi_view * n)()
        for i, (vfov, az, el, roll) in enumerate(views):
            descs[i] = _native.pf_equi_view(H, W, vfov, az, el, roll, W / H, i * 3 * H * W * es)
        out = torch.empty(n * 3 * H * W * es, dtype=torch.uint8, device=dev)
        src = srcs[dtype]
        code = _native.PF_EQUI_F32 if dtype == "float32" else _native.PF_EQUI_U8
        ms = timed(lambda: _native.check(L.pf_equi_views(dev.index, src.data_ptr(), 1024, 2048, 3, code, descs, n, mode, 0, 0, out.data_ptr(), st)),
                   a.reps)
        gbs = out.numel() / (ms * 1e-3) / 1e9
        res[name] = {"ms_per_call": round(ms, 3), "views_per_s": round(n / (ms * 1e-3), 1), "bytes_per_pixel": 3 * es,
                     "written_GBps": round(gbs, 1), "frac_of_write_peak": round(gbs / peak, 3)}
        del out
    pdescs = (_native.pf_pano_view * n)()
    for i, (vfov, az, el, roll) in enumerate(views):
        pdescs[i] = _native.pf_pano_view(H, W, H / (2 * math.tan(math.radians(vfov) / 2)), 0.0, az, -el, roll, i * 3 * H * W, 0)
    im = torch.empty(n * 3 * H * W, dtype=torch.uint8, device=dev)
    src = srcs["uint8"]
    ms = timed(lambda: _native.check(L.pf_pano_views(dev.index, src.data_ptr(), 1024, 2048, pdescs, n, im.data_ptr(), None, None, None, None,
                                                     None, None, None, st)), a.reps)
    res["pano_views_crop_only"] = {"ms_per_call": round(ms, 3), "views_per_s": round(n / (ms * 1e-3), 1)}
    res.update(card(dev.index))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
