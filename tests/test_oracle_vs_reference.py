"""CPU: the oracle against what the unmodified reference produced, stored by tests/golden/make_golden_reference.py
(reference_surface.json.gz: state-dict schema, configuration tree and model_zoo entry per variant; reference_outputs.npz:
outputs on seeded synthetic checkpoints and images, large arrays as a seeded sample of their elements)."""
import gzip
import json
import os

import numpy as np
import pytest

from oracle import model as om
from oracle import weights_gen as wg
from oracle.schema import state_dict_schema
from oracle.variants import VARIANTS

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
with gzip.open(os.path.join(GOLDEN, "reference_surface.json.gz"), "rt") as _f:
    SURFACE = json.load(_f)
OUT = np.load(os.path.join(GOLDEN, "reference_outputs.npz"))


def _rel_err(prefix, key, mine):
    """max|ref - mine| / max|ref| over the stored elements of reference output `prefix.key`"""
    a = np.asarray(mine, dtype=np.float64).reshape(-1)
    k = f"{prefix}.{key}"
    if k + ".idx" in OUT:
        a = a[OUT[k + ".idx"]]
    return np.abs(OUT[k] - a).max() / max(float(OUT[k + ".absmax"]), 1e-30)


@pytest.mark.parametrize("version", list(VARIANTS))
def test_schema_matches_reference(version):
    ref = SURFACE[version]["state_dict"]
    assert [k for k, _ in ref] == [k for k, _ in state_dict_schema(version)]
    for (k, s), (_, rs) in zip(state_dict_schema(version), ref):
        assert tuple(rs) == tuple(s), k


def test_live_outputs_match():
    version = "PersNet_Paramnet-GSV-uncentered"
    sd = wg.synth_state_dict(version, 3)
    ora = om.inference_batch(sd, version, wg.smooth_images(1, 300, 420, 5))
    assert [k for k, v in ora[0].items() if not isinstance(v, str)] == list(OUT["live.keys"])
    for k in OUT["live.keys"]:
        err = _rel_err("live", k, ora[0][k].numpy())
        assert err < 1e-4, (k, err)


def test_float_input_branch_matches_reference():
    """perspectivefields.py:47-66: non-uint8 images go through F.interpolate instead of PIL (pins oracle.model.inference_float /
    resize_float, which tests/test_gpu_forward.py uses as the referee for the CUDA float branch)."""
    version = "Paramnet-360Cities-edina-centered"
    sd = wg.synth_state_dict(version, 0)
    img = wg.smooth_images(1, 200, 260, 9)[0].astype(np.float32) + 0.25
    assert _rel_err("float", "resized", om.resize_float(img, 320, 320)) == 0.0
    ora = om.inference_float(sd, version, img)
    for k in OUT["float.keys"]:
        err = _rel_err("float", k, ora[k].numpy())
        assert err < 1e-4, (k, err)


def test_yaml_configuration_matches_reference():
    """perspectivefields_b200/config/*.yaml (defaults + per-variant overrides, parsed with PyYAML) give every inference-relevant
    field the value the reference's yacs tree has after merge_from_file (perspectivefields.py:124-131)."""
    from perspectivefields_b200 import variants as V

    for version in VARIANTS:
        ref = SURFACE[version]["cfg"]
        mine = V.make_cfg(version)

        def walk(a, b, path):
            for k, v in a.items():
                assert k in b, (version, path + k)
                if isinstance(v, dict):
                    walk(v, b[k], path + k + ".")
                else:
                    rv = b[k]
                    rv = list(rv) if isinstance(rv, (list, tuple)) else rv
                    v = list(v) if isinstance(v, tuple) else v
                    assert rv == v, (version, path + k, rv, v)
        walk(mine, ref, "")
        zoo = V.model_zoo[version]
        assert json.loads(json.dumps(zoo)) == SURFACE[version]["model_zoo"]
