"""Time one ParamNet training step (``PerspectiveFields.param_net_backward``: pf_param_train_forward, the loss rule under torch
autograd, pf_param_backward and the accumulation into ``.grad``) with CUDA events, in one process:

    python tools/paramnet_train_bench.py [--iters 5] [--out results/paramnet_train_bench.json]

Cases: 64 and 256 centred pairs (ConvNeXt-T on 320 x 320 fields) and 256 uncentred pairs (on their 64 x 64 nearest sub-sample),
seeded ground-truth camera fields.  Beside each, the same step in PyTorch eager on the same GPU as the baseline:
``oracle.model.convnext_t`` + ``metrics.param_net_losses`` with autograd in fp32, TF32 off (256 centred pairs as four
accumulated micro-batches of 64, which is the same sum).  Also: the per-kernel device time of one step from torch.profiler in a
pass of its own, the algorithmic FLOP rate of all GEMM-engine launches of a step (pf_profile_*: forward, recompute, data and
weight gradients; MMA count 3 per product at fp32), the workspace per pair, and the GPU's name and power limit read in the same
run.  Prints one JSON object."""
import argparse
import ctypes
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from metrics_bench import gpu_info, kernel_ms, timed  # noqa: E402
from paramnet_bench import gt_fields  # noqa: E402


def eager_step(sd, cfg, lw, preds, gt, chunk=64):
    from oracle import model as om
    from perspectivefields_b200 import metrics

    for p in sd.values():
        p.grad = None
    n = preds["pred_gravity"].shape[0]
    for i in range(0, n, chunk):
        images = torch.cat((preds["pred_gravity"][i:i + chunk], preds["pred_latitude"][i:i + chunk]), 1)
        if cfg["param_net"] != "ParamNet":
            images = F.interpolate(images, (cfg["input_size"], cfg["input_size"]))
        raw = om.convnext_t(sd, images)
        losses = metrics.param_net_losses(raw, gt[i:i + chunk], cfg["param_net"], cfg["predict_params"], lw)
        (sum(losses.values()) * (min(chunk, n - i) / n)).backward()


def gemm_rate(m, step):
    """One step's GEMM-engine launches, timed by the engine's per-launch events (pf_profile_*, per-launch CSV): (all launches ms,
    algorithmic TFLOP/s; weight-gradient launches ms, TFLOP/s).  The weight-gradient GEMMs are the grouped GEMM-mode launches
    (engine_cfg 5, groups > 1; one group per chunk of rows), the only grouped ones of a step."""
    import csv
    import tempfile

    eng = m._get_engine()
    L = eng.L
    buf = (ctypes.c_double * 21)()
    path = os.path.join(tempfile.mkdtemp(), "launches.csv")
    L.pf_profile_enable(eng.handle, 1)
    torch.cuda.synchronize()
    L.pf_profile_read(eng.handle, buf)
    step()
    torch.cuda.synchronize()
    os.environ["PF_PROFILE_CSV"] = path
    L.pf_profile_read(eng.handle, buf)
    del os.environ["PF_PROFILE_CSV"]
    L.pf_profile_enable(eng.handle, 0)
    rows = list(csv.DictReader(open(path)))
    tot = [0.0, 0.0, 0.0, 0.0]
    for r in rows:
        ms = float(r["ms"])
        flops = 2.0 * int(r["M"]) * int(r["N"]) * int(r["K"]) * int(r["groups"])
        tot[0] += ms
        tot[1] += flops
        if r["engine_cfg"] == "5" and int(r["groups"]) > 1:
            tot[2] += ms
            tot[3] += flops
    rate = lambda f, ms: f / (ms * 1e-3) / 1e12 if ms > 0 else 0.0
    return tot[0], rate(tot[1], tot[0]), tot[2], rate(tot[3], tot[2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paramnet_train_bench needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    import pf_test_util as U
    from perspectivefields_b200 import metrics
    from perspectivefields_b200.variants import VARIANTS, make_cfg

    res = {"gpu": gpu_info(), "cases": {}}
    for name, version, n in (("centred_320x320_64", "Paramnet-360Cities-edina-centered", 64),
                             ("centred_320x320_256", "Paramnet-360Cities-edina-centered", 256),
                             ("uncentred_64x64_256", "Paramnet-360Cities-edina-uncentered", 256)):
        m, sd = U.make_model(version, seed=0, device="cuda")
        preds, inputs = gt_fields(m, n)
        params = m.param_net_parameters()

        def step():
            for p in params.values():
                p.grad = None
            m.param_net_backward(preds, inputs)

        ms = timed(step, args.iters, warmup=2)
        eng = m._get_engine()
        ws = eng.L.pf_param_train_workspace_bytes(eng.handle, n)
        gms, tflops, wms, wtflops = gemm_rate(m, step)
        case = {"version": version, "pairs": n, "ms_per_step": ms, "pairs_per_s": n * 1e3 / ms, "workspace_bytes_per_pair": ws / n,
                "gemm_engine_ms_per_step": gms, "gemm_engine_algorithmic_tflops": tflops, "wgrad_ms_per_step": wms,
                "wgrad_algorithmic_tflops": wtflops, "mma_per_product": 3,
                "kernel_ms_per_step": dict(sorted(kernel_ms(step, "", reps=2).items(), key=lambda kv: -kv[1])[:25])}
        cfg = VARIANTS[version]
        lw = float(make_cfg(version).MODEL.PARAM_DECODER.LOSS_WEIGHT)
        gt = torch.from_numpy(metrics.param_targets(inputs, n, cfg["param_net"], cfg["predict_params"])).cuda()
        esd = {k: v.float().cuda().requires_grad_(True) for k, v in sd.items() if k.startswith("param_net.backbone.")}
        del m, params
        torch.cuda.empty_cache()
        try:
            ems = timed(lambda: eager_step(esd, cfg, lw, preds, gt), max(1, args.iters // 2), warmup=1)
            case.update({"eager_fp32_ms_per_step": ems, "eager_fp32_pairs_per_s": n * 1e3 / ems, "speedup_vs_eager": ems / ms})
        except torch.cuda.OutOfMemoryError:
            case["eager_fp32_ms_per_step"] = "not measured (out of memory)"
        res["cases"][name] = case
        del esd, preds
        torch.cuda.empty_cache()
        print(name, json.dumps({k: v for k, v in case.items() if k != "kernel_ms_per_step"}), file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
