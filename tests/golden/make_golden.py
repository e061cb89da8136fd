"""Generate tests/golden/*.npz from the UNMODIFIED reference (run in the build container only).

    python tests/golden/make_golden.py

For every zoo version: write the synthetic checkpoint (oracle/weights_gen.py, seed 0) into a private
TORCH_HOME hub cache, construct ``perspective2d.PerspectiveFields(version).eval()`` through the reference's
own loader (perspectivefields.py:178-192), run ``inference_batch`` on CPU fp32 on two synthetic images
(480x640 uniform noise, 360x500 smooth), and store a strided sub-sample of every returned tensor together
with float64 checksums.  The fixtures pin oracle/model.py to the reference (tests/test_oracle_golden.py)
on machines without a checkout of the reference (PF_REFERENCE_ROOT names one).
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import weights_gen as wg  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402
from oracle.variants import VARIANTS  # noqa: E402

STRIDE = 5
LOGIT_STRIDE = 16
SEED = 0


def golden_images():
    return wg.synth_images(1, 480, 640, SEED) + wg.smooth_images(1, 360, 500, SEED)


def golden_stride(shape):
    """Spatial sub-sampling stride: 5, or 16 for the wide logit tensors of the classification variant."""
    return LOGIT_STRIDE if (len(shape) == 3 and shape[0] > 3) else STRIDE


def subsample(t):
    t = t.detach().cpu().to(torch.float32)
    if t.ndim >= 2:
        st = golden_stride(t.shape)
        t = t[..., ::st, ::st]
    return t.numpy()


def main():
    th = tempfile.mkdtemp(prefix="pf_golden_")
    os.environ["TORCH_HOME"] = th
    p2d = load_reference()
    os.makedirs(os.path.join(th, "hub", "checkpoints"), exist_ok=True)
    torch.set_num_threads(8)
    manifest = {"stride": STRIDE, "logit_stride": LOGIT_STRIDE, "seed": SEED, "torch": torch.__version__, "versions": {}}
    imgs = golden_images()
    for ver, cfg in VARIANTS.items():
        sd = wg.synth_state_dict(ver, SEED)
        torch.save({"model": sd}, os.path.join(th, "hub", "checkpoints", cfg["ckpt"]))
        model = p2d.PerspectiveFields(ver).eval()
        ref_sd = model.state_dict()
        assert all(torch.equal(ref_sd[k], v) for k, v in sd.items())
        out = model.inference_batch(imgs)
        arrays, keys = {}, []
        for i, res in enumerate(out):
            keys.append(list(res.keys()))
            for k, v in res.items():
                if isinstance(v, str):
                    continue
                arrays[f"{i}/{k}"] = subsample(v)
                v64 = v.detach().double()
                arrays[f"{i}/{k}/stats"] = np.array([v64.sum().item(), v64.abs().sum().item(), v64.numel()], np.float64)
                arrays[f"{i}/{k}/shape"] = np.array(v.shape, np.int64)
        fn = "golden_" + ver.replace("-", "_") + ".npz"
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", fn), **arrays)
        manifest["versions"][ver] = {"file": fn, "keys": keys, "n_state_tensors": len(ref_sd),
                                     "n_params": int(sum(v.numel() for v in ref_sd.values()))}
        print(ver, "->", fn, {k: a.shape for k, a in list(arrays.items())[:3]})
    with open(os.path.join(ROOT, "tests", "golden", "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
