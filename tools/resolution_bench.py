"""Images/s of the resident forward at several working sizes (``PerspectiveFields(version, resize=(H, W))``), with the
per-kernel split of one profiled pass (CUDA events around every launch, ``pf_profile_kernels_*``), including the attention core.

    python tools/resolution_bench.py [--version V] [--batch 32] [--steps 10] [--warmup 3] [--sizes 320x320,320x448,384x512,512x512]

Same measurement as bench.py's resident leg: the batch (480 x 640 synthetic uint8 images, a synthetic checkpoint in a temporary
hub cache) is uploaded once, every step is one ``pf_forward`` on the device blob, timed with CUDA events.  One JSON line per size,
then a summary line.  Writes nothing into the repository tree.
"""
import argparse
import ctypes
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--version", default="Paramnet-360Cities-edina-centered")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="320x320,320x448,384x512,512x512")
    ap.add_argument("--image", default="480x640", help="input image size H x W")
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16"])
    args = ap.parse_args()

    import torch

    from oracle import weights_gen as wg
    from oracle.variants import VARIANTS
    from perspectivefields_b200 import PerspectiveFields, _native

    hub = tempfile.mkdtemp(prefix="pf_resbench_")
    os.environ["TORCH_HOME"] = hub
    os.makedirs(os.path.join(hub, "hub", "checkpoints"), exist_ok=True)
    torch.save({"model": wg.synth_state_dict(args.version, 0)}, os.path.join(hub, "hub", "checkpoints", VARIANTS[args.version]["ckpt"]))
    ih, iw = (int(x) for x in args.image.split("x"))
    imgs = wg.synth_images(args.batch, ih, iw, 7)
    L = _native.lib()
    summary = {}
    for spec in args.sizes.split(","):
        h, w = (int(x) for x in spec.split("x"))
        m = PerspectiveFields(args.version, resize=(h, w), precision=args.precision).cuda()
        eng = m._get_engine()
        blob, offsets = eng.stage_images(imgs)
        hs, ws = [ih] * args.batch, [iw] * args.batch
        for _ in range(args.warmup):
            eng.forward(args.batch, hs, ws, blob=blob, offsets=offsets)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.steps):
            eng.forward(args.batch, hs, ws, blob=blob, offsets=offsets)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / args.steps
        # per-kernel split: a separate pass (the event records cost a few percent)
        _native.check(L.pf_profile_kernels_enable(eng.handle, 700 * 2))
        for _ in range(2):
            eng.forward(args.batch, hs, ws, blob=blob, offsets=offsets)
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(1 << 16)
        nbytes = _native.check(L.pf_profile_kernels_read(eng.handle, buf, len(buf)))
        _native.check(L.pf_profile_kernels_enable(eng.handle, 0))
        per_kernel = {}
        for line in buf.raw[:nbytes].decode().splitlines()[1:]:
            name, cnt, kms = line.rsplit(",", 2)
            per_kernel[name] = round(float(kms) / 2, 3)
        per_kernel = dict(sorted(per_kernel.items(), key=lambda kv: -kv[1]))
        res = {"net_hw": [h, w], "attention_keys": (h // 32) * (w // 32), "images_per_s": round(args.batch * 1000.0 / ms, 1),
               "ms_per_step": round(ms, 3), "batch": args.batch, "precision": args.precision,
               "attention_ms_per_step": per_kernel.get("attention_mma_launch"), "per_kernel_ms_per_step": per_kernel,
               "gpu": torch.cuda.get_device_name()}
        print(json.dumps(res), flush=True)
        summary[spec] = res["images_per_s"]
        del m, eng
        torch.cuda.empty_cache()
    print(json.dumps({"version": args.version, "images_per_s": summary}), flush=True)


if __name__ == "__main__":
    main()
