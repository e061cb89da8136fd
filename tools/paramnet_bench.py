"""Time ParamNet on given fields (``PerspectiveFields.param_net`` / ``param_losses``, pf_param_forward) with CUDA events, in one
process:

    python tools/paramnet_bench.py [--iters 10] [--out results/paramnet_bench.json]

256 ground-truth field pairs at the 320 x 320 working size (seeded cameras -> ``camera_fields`` -> ``targets_from_fields``), run
through the centred ParamNet (ConvNeXt-T on the 320 x 320 fields) and the uncentred one (ConvNeXt-T on their 64 x 64 nearest
sub-sample), each after a warm-up.  Reports ms per call, calls/s and field pairs/s, the per-kernel device time of one call from
torch.profiler in a pass of its own, and the GPU's name and power limit read in the same run.  Prints one JSON object."""
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

from metrics_bench import gpu_info, kernel_ms, timed  # noqa: E402


def gt_fields(m, n, seed=0):
    from perspectivefields_b200 import panocam

    g = torch.Generator().manual_seed(seed)
    u = lambda lo, hi: (torch.rand(n, generator=g, dtype=torch.float64) * (hi - lo) + lo).tolist()
    roll, pitch, vfov, cx, cy = u(-30, 30), u(-40, 40), u(40, 90), u(-0.1, 0.1), u(-0.1, 0.1)
    h, w = m.net_size()
    ups, lats = panocam.camera_fields([1 / (2 * math.tan(math.radians(v) / 2)) for v in vfov], [h] * n, [w] * n,
                                      [math.radians(p) for p in pitch], [math.radians(r) for r in roll], cx, cy)
    t = m.targets_from_fields(ups, lats)
    inputs = [{"roll": a, "pitch": b, "vfov": c, "general_vfov": c, "rel_cx": d, "rel_cy": e} for a, b, c, d, e in zip(roll, pitch, vfov, cx, cy)]
    return {"pred_gravity": t["gt_gravity"], "pred_latitude": t["gt_latitude"]}, inputs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paramnet_bench needs a CUDA device")
    import pf_test_util as U

    res = {"gpu": gpu_info(), "n": args.n, "cases": {}}
    for name, version in (("centred_320x320", "Paramnet-360Cities-edina-centered"), ("uncentred_64x64", "Paramnet-360Cities-edina-uncentered")):
        m = U.make_model(version, seed=0, device="cuda")[0]
        preds, inputs = gt_fields(m, args.n)
        ms = timed(lambda: m.param_net(preds), args.iters)
        loss_ms = timed(lambda: m.param_losses(preds, inputs), args.iters)
        res["cases"][name] = {"version": version, "param_net_ms_per_call": ms, "calls_per_s": 1e3 / ms, "field_pairs_per_s": args.n * 1e3 / ms,
                              "param_losses_ms_per_call": loss_ms, "kernel_ms_per_call": kernel_ms(lambda: m.param_net(preds), "")}
        del m, preds
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
