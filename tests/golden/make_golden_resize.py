"""Generate tests/golden/golden_resize.npz from the UNMODIFIED reference at working sizes other than 320 x 320
(run where a checkout of the reference exists; PF_REFERENCE_ROOT names it):

    PF_REFERENCE_ROOT=<reference checkout> python tests/golden/make_golden_resize.py

The reference reads its working size from ``cfg.DATALOADER.RESIZE`` (perspectivefields.py:155, gravity_head.py:136,
latitude_head.py:135).  Its constructor merges the variant's yaml and then calls ``cfg.freeze()`` before it builds any module;
this script wraps the freeze of the shim's ``CfgNode`` (oracle/ref_shim.py) so that RESIZE is overridden at exactly that
point, and runs the reference's own code unmodified.  For every zoo version and every size below: the synthetic checkpoint
of make_golden.py (oracle/weights_gen.py, seed 0), ``inference_batch`` on the two golden images, and per returned tensor a
seeded sample of SAMPLE elements (tests/oracle_resize.py:sample_index; the indices are redrawn by the test, not stored), its
shape, its maximum magnitude and float64 sum / abs-sum checksums of the whole tensor.  The file stays below 0.4 MB;
tests/test_resize_host.py reads it.
384 x 512: 12 x 16 = 192 attention keys; 448 x 448: 14 x 14 = 196 keys (both above 112: the key-block attention path).
"""
import contextlib
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from make_golden import golden_images  # noqa: E402
from oracle import weights_gen as wg  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402
from oracle.variants import VARIANTS  # noqa: E402
from oracle_resize import sample_index  # noqa: E402

SIZES = ((384, 512), (448, 448))
SEED = 0


def put(arrays, key, v):
    """key -> sampled float32 elements; key/meta = float64 [max |v|, sum, abs-sum, *shape] of the whole tensor (one entry: every
    npz member costs a few hundred bytes of headers)."""
    a = v.detach().cpu().double().numpy().reshape(-1)
    idx = sample_index(key, a.size)
    arrays[key] = (a if idx is None else a[idx]).astype(np.float32)
    arrays[key + "/meta"] = np.array([np.abs(a).max() if a.size else 0.0, a.sum(), np.abs(a).sum(), *v.shape], np.float64)


@contextlib.contextmanager
def resize_override(net_hw):
    """cfg.DATALOADER.RESIZE = [H, W] in every CfgNode frozen inside the block (the reference freezes its config right after
    merge_from_file, before building the backbone, heads and ``aug``)."""
    CfgNode = sys.modules["yacs.config"].CfgNode
    freeze = CfgNode.freeze

    def freeze_with_resize(self):
        if "DATALOADER" in self:
            self.DATALOADER.RESIZE = list(net_hw)
        return freeze(self)

    CfgNode.freeze = freeze_with_resize
    try:
        yield
    finally:
        CfgNode.freeze = freeze


def main():
    th = tempfile.mkdtemp(prefix="pf_golden_resize_")
    os.environ["TORCH_HOME"] = th
    p2d = load_reference()
    os.makedirs(os.path.join(th, "hub", "checkpoints"), exist_ok=True)
    torch.set_num_threads(8)
    imgs = golden_images()
    arrays = {"sizes": np.array(SIZES, np.int64)}
    for net_hw in SIZES:
        tag = "%dx%d" % net_hw
        for ver, cfg in VARIANTS.items():
            sd = wg.synth_state_dict(ver, SEED)
            torch.save({"model": sd}, os.path.join(th, "hub", "checkpoints", cfg["ckpt"]))
            with resize_override(net_hw):
                model = p2d.PerspectiveFields(ver).eval()
            assert list(model.cfg.DATALOADER.RESIZE) == list(net_hw)
            assert (model.aug.new_h, model.aug.new_w) == net_hw
            with torch.no_grad():
                out = model.inference_batch(imgs)
            for i, res in enumerate(out):
                arrays[f"{tag}/{ver}/{i}/keys"] = np.array(list(res.keys()))
                for k, v in res.items():
                    if not isinstance(v, str):
                        put(arrays, f"{tag}/{ver}/{i}/{k}", v)
            print(net_hw, ver, "pred_gravity", tuple(out[0]["pred_gravity"].shape), flush=True)
    fn = os.path.join(ROOT, "tests", "golden", "golden_resize.npz")
    np.savez_compressed(fn, **arrays)
    print("->", fn, os.path.getsize(fn), "bytes")


if __name__ == "__main__":
    main()
