"""Generate tests/golden/reference_surface.json.gz and tests/golden/reference_outputs.npz from the UNMODIFIED reference
(run where a checkout of it exists; PF_REFERENCE_ROOT names it):

    PF_REFERENCE_ROOT=<reference checkout> python tests/golden/make_golden_reference.py

reference_surface.json.gz: per variant, the reference model's state-dict keys and shapes, its configuration tree after
merge_from_file (perspectivefields.py:124-131) and its model_zoo entry.  reference_outputs.npz: the reference's outputs on
seeded synthetic checkpoints and images (oracle/weights_gen.py) for tests/test_oracle_vs_reference.py, and PanoCam fields
for random camera parameters (tests/test_oracle_panocam.py).  Large arrays keep a seeded sample of their elements (every
file stays below 1 MB) plus the maximum magnitude of the whole array, the denominator of the relative-error metric.
"""
import gzip
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import weights_gen as wg  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402
from oracle.schema import state_dict_schema  # noqa: E402
from oracle.variants import VARIANTS  # noqa: E402

SAMPLE = 4096     # elements kept of an array larger than this


def _plain(v):
    if isinstance(v, dict):
        return {k: _plain(x) for k, x in v.items()}
    if isinstance(v, tuple):
        return list(v)
    return v


def _put(store, key, a):
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    store[key + ".absmax"] = np.array(np.abs(a).max() if a.size else 0.0)
    if a.size > SAMPLE:
        idx = np.sort(np.random.default_rng(len(key)).choice(a.size, SAMPLE, replace=False))
        store[key + ".idx"] = idx
        a = a[idx]
    store[key] = a


def main():
    th = tempfile.mkdtemp(prefix="pf_ref_")
    os.environ["TORCH_HOME"] = th
    ck = os.path.join(th, "hub", "checkpoints")
    os.makedirs(ck, exist_ok=True)
    mod = load_reference()

    def model(version, sd):
        torch.save({"model": sd}, os.path.join(ck, VARIANTS[version]["ckpt"]))
        return mod.PerspectiveFields(version).eval()

    surface = {}
    for version in VARIANTS:
        m = model(version, {k: torch.zeros(s) for k, s in state_dict_schema(version)})
        surface[version] = {"state_dict": [[k, list(t.shape)] for k, t in m.state_dict().items()], "cfg": _plain(dict(m.cfg)),
                            "model_zoo": _plain(mod.perspectivefields.model_zoo[version])}
    with gzip.open(os.path.join(HERE, "reference_surface.json.gz"), "wt") as f:
        json.dump(surface, f, sort_keys=True)

    store = {}
    version = "PersNet_Paramnet-GSV-uncentered"        # tests/test_oracle_vs_reference.py::test_live_outputs_match
    ref = model(version, wg.synth_state_dict(version, 3)).inference_batch(wg.smooth_images(1, 300, 420, 5))
    store["live.keys"] = np.array([k for k, v in ref[0].items() if not isinstance(v, str)])
    for k, v in ref[0].items():
        if not isinstance(v, str):
            _put(store, "live." + k, v.numpy())

    version = "Paramnet-360Cities-edina-centered"      # test_float_input_branch_matches_reference
    m = model(version, wg.synth_state_dict(version, 0))
    img = wg.smooth_images(1, 200, 260, 9)[0].astype(np.float32) + 0.25
    _put(store, "float.resized", m.aug.apply_image(img))
    ref = m.inference(img)
    store["float.keys"] = np.array([k for k, v in ref.items() if not isinstance(v, str)])
    for k, v in ref.items():
        if not isinstance(v, str):
            _put(store, "float." + k, v.numpy())

    from perspective2d.utils.panocam import PanoCam     # tests/test_oracle_panocam.py::test_oracle_matches_live_reference
    rs = np.random.RandomState(3)
    for i in range(6):
        f, el, roll = rs.uniform(0.3, 2.0), rs.uniform(-1.4, 1.4), rs.uniform(-3.1, 3.1)
        cx, cy = rs.uniform(-0.3, 0.3, 2)
        w, h = int(rs.randint(2, 60)), int(rs.randint(2, 60))
        store[f"pano{i}.case"] = np.array([f, w, h, el, roll, cx, cy])
        store[f"pano{i}.up"] = PanoCam.get_up_general(f, w, h, el, roll, cx, cy)
        store[f"pano{i}.lat"] = PanoCam.get_lat_general(f, w, h, el, roll, cx, cy)
    np.savez_compressed(os.path.join(HERE, "reference_outputs.npz"), **store)


if __name__ == "__main__":
    main()
