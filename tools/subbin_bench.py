"""Time the sub-bin decode of the classification heads with CUDA events, in one process:

    python tools/subbin_bench.py [--iters 10] [--rounds 5] [--out results/subbin_bench.json]

* ``inference_batch`` of PersNet-360Cities on bench.py's C2 batch (32 uint8 images of 640 x 480, seeded as bench.py's timed leg on
  rank 0: 1000 + rank), resident on the device, with ``decode="argmax"`` and ``decode="subbin"``, for ``logits=True`` and
  ``logits=False``: the four models are warmed up, then timed in alternation for ``--rounds`` rounds (median ms per call, with
  every round's value);
* the decode kernels alone through their entry points at n = 32, 320 x 320, for both heads: the argmax and sub-bin decode of
  logits (pf_op_argmax_decode / pf_op_subbin_decode) and of the fused 1x1 conv (pf_op_pred_argmax_decode /
  pf_op_pred_subbin_decode), in alternation.

Prints one JSON object with the GPU's name and power limit."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from confidence_bench import alternate  # noqa: E402
from metrics_bench import gpu_info  # noqa: E402


def op_cases(n=32, hw=320 * 320):
    """{name: fn} of the four decode instantiations per head on seeded inputs at n x hw pixels."""
    from perspectivefields_b200 import _native

    L = _native.lib()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(0)
    feat = torch.relu(torch.randn(n * hw, 64, generator=g, device="cuda"))
    fns = {}
    for head, nc, coff, grav in (("gravity", 73, 0, 1), ("latitude", 180, 32, 0)):
        w = torch.randn(nc, 32, generator=g, device="cuda") * 0.3
        b = torch.randn(nc, generator=g, device="cuda") * 0.1
        logits = torch.empty(n, nc, hw, device="cuda")
        _native.check(L.pf_op_pred_tail(feat.data_ptr(), 64, coff, w.data_ptr(), b.data_ptr(), logits.data_ptr(), n, hw, nc, 0, st))
        field = torch.empty(n, 2 if grav else 1, hw, device="cuda")
        a = (logits, w, b, field)   # kept alive by the closures
        fns[f"{head}_logits_argmax"] = lambda a=a, nc=nc, grav=grav: _native.check(
            L.pf_op_argmax_decode(a[0].data_ptr(), a[3].data_ptr(), n, hw, nc, grav, st))
        fns[f"{head}_logits_subbin"] = lambda a=a, nc=nc, grav=grav: _native.check(
            L.pf_op_subbin_decode(a[0].data_ptr(), a[3].data_ptr(), None, n, hw, nc, grav, st))
        fns[f"{head}_fused_argmax"] = lambda a=a, nc=nc, grav=grav, coff=coff: _native.check(
            L.pf_op_pred_argmax_decode(feat.data_ptr(), 64, coff, a[1].data_ptr(), a[2].data_ptr(), a[3].data_ptr(), n, hw, nc, grav, st))
        fns[f"{head}_fused_subbin"] = lambda a=a, nc=nc, grav=grav, coff=coff: _native.check(
            L.pf_op_pred_subbin_decode(feat.data_ptr(), 64, coff, a[1].data_ptr(), a[2].data_ptr(), a[3].data_ptr(), None, n, hw, nc, grav, st))
    return fns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("subbin_bench needs a CUDA device")
    import pf_test_util as U
    from oracle import weights_gen as wg

    res = {"gpu": gpu_info(), "cases": {}}
    imgs = [torch.from_numpy(im).cuda() for im in wg.synth_images(32, 480, 640, 1000)]   # bench.py's C2 inputs (seed 1000 + rank)
    fns = {}
    for logits in (True, False):
        for decode in ("argmax", "subbin"):
            m = U.make_model("PersNet-360Cities", seed=0, device="cuda", model_kwargs={"logits": logits, "decode": decode})[0]
            fns[f"logits_{logits}_{decode}"] = (lambda m=m: m.inference_batch(imgs))
    res["cases"]["inference_b32_640x480_resident"] = alternate(fns, args.iters, args.rounds)
    del fns
    torch.cuda.empty_cache()
    res["cases"]["decode_ops_n32_320x320"] = alternate(op_cases(), 10 * args.iters, args.rounds)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
