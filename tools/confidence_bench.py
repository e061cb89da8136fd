"""Time the head-confidence maps and the weighted camera fit with CUDA events, in one process:

    python tools/confidence_bench.py [--iters 10] [--rounds 3] [--out results/confidence_bench.json]

* ``inference_batch`` of PersNet-360Cities on bench.py's C2 batch (32 uint8 images of 640 x 480, seeded as bench.py's timed leg on
  rank 0: 1000 + rank), with ``confidence`` off and
  on, for ``logits=True`` and ``logits=False``: the four models are warmed up, then timed in alternation for ``--rounds`` rounds
  (median ms per call reported, with every round's value);
* ``fit_camera`` on tools/calib_bench.py's seeded batch (256 noisy camera fields of 640 x 480), unweighted and with per-pixel weights
  of both fields (seeded uniform in [0.5, 2]), centred least squares, in alternation.

Prints one JSON object with the GPU's name and power limit."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from calib_bench import noisy_batch  # noqa: E402
from metrics_bench import gpu_info, timed  # noqa: E402


def alternate(fns, iters, rounds):
    """{name: [ms per call of each round]}: every function warmed up, then all timed once per round, in turn."""
    for fn in fns.values():
        timed(fn, 1, warmup=3)
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            out[k].append(timed(fn, iters, warmup=1))
    return {k: {"ms_median": statistics.median(v), "ms_rounds": v} for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("confidence_bench needs a CUDA device")
    import pf_test_util as U
    from oracle import weights_gen as wg
    from perspectivefields_b200 import calibrate

    res = {"gpu": gpu_info(), "cases": {}}
    imgs = wg.synth_images(32, 480, 640, 1000)        # bench.py's C2 inputs of its timed leg on rank 0 (seed 1000 + rank)
    fns = {}
    for logits in (True, False):
        for conf in (False, True):
            m = U.make_model("PersNet-360Cities", seed=0, device="cuda", model_kwargs={"logits": logits, "confidence": conf})[0]
            fns[f"logits_{logits}_confidence_{conf}"] = (lambda m=m: m.inference_batch(imgs))
    res["cases"]["inference_b32_640x480"] = alternate(fns, args.iters, args.rounds)
    del fns
    torch.cuda.empty_cache()
    n, h, w = 256, 480, 640
    results = noisy_batch(n, h, w)
    g = torch.Generator(device="cuda").manual_seed(1)
    wts = [tuple(torch.rand((h, w), generator=g, device="cuda") * 1.5 + 0.5 for _ in range(2)) for _ in range(n)]
    fits = {"unweighted": lambda: calibrate.fit_camera(results), "weighted": lambda: calibrate.fit_camera(results, weights=wts)}
    res["cases"]["fit_camera_256_640x480_centred_l2"] = alternate(fits, args.iters, args.rounds)
    for k, fn in fits.items():
        its = torch.stack([o["fit_iterations"] for o in fn()]).float()
        res["cases"]["fit_camera_256_640x480_centred_l2"][k]["mean_evaluations"] = float(its.mean())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
