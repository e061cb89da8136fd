"""CPU: ParamNet on given fields and its training losses, pinned to the unmodified reference by tests/golden/paramnet.npz
(tests/golden/make_golden_paramnet.py).

* ``oracle.model.param_net`` on the seeded camera and random fields of tests/oracle_paramnet.py reproduces the reference's raw
  backbone output and eval dict for the centred, 360Cities-uncentred and GSV-uncentred configurations;
* ``metrics.param_targets`` + ``metrics.param_net_losses`` (the rule ``PerspectiveFields.param_losses`` runs on the GPU), on
  CPU on the reference's raw output, reproduce its training-branch losses to 1e-6 relative, LOSS_WEIGHT 0.1 included.
"""
import os

import numpy as np
import pytest
import torch

import oracle_paramnet as op
from oracle import model as om
from oracle import panocam as oracle_panocam
from oracle.variants import VARIANTS as ORACLE_VARIANTS
from perspectivefields_b200 import metrics
from perspectivefields_b200.variants import VARIANTS, make_cfg

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "paramnet.npz")
CONFIGS = [c[0] for c in op.CONFIGS]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def fields():
    return op.inputs(oracle_panocam.get_up_general, oracle_panocam.get_lat_general)


def _config(name):
    return next(c for c in op.CONFIGS if c[0] == name)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("name", CONFIGS)
def test_oracle_param_net_matches_reference(golden, fields, name):
    _, version, seed = _config(name)
    taps = {}
    with torch.no_grad():
        out = om.param_net(op.param_state(version, seed), ORACLE_VARIANTS[version], fields[0], fields[1], taps)
    # the same ATen CPU kernels in the same order as the reference's modules: only the summation order of a few reductions may
    # differ, far below 1e-5 of the largest output
    assert _rel(taps["cnx.out"], golden[f"{name}/raw"]) < 1e-5
    keys = [k[len(name) + 6:] for k in golden if k.startswith(name + "/eval/")]
    assert keys
    for k in keys:
        ref = golden[f"{name}/eval/{k}"]
        got = out[k].numpy()
        if k == "pred_rel_focal" and VARIANTS[version]["param_net"] == "ParamNetConvNextRegress":
            # scipy fsolve: rows where it converges agree closely; it does not converge for every random field
            ok = np.isfinite(ref) & (np.abs(got - ref) <= 1e-3 * np.maximum(np.abs(ref), 1.0))
            assert ok[:op.N_CAMERAS].all(), (k, got, ref)
            continue
        assert got.shape == ref.shape, k
        assert _rel(got, ref) < 1e-5, k


@pytest.mark.parametrize("name", CONFIGS)
def test_param_losses_rule_matches_reference(golden, name):
    _, version, _ = _config(name)
    v = VARIANTS[version]
    raw = torch.from_numpy(golden[f"{name}/raw"])
    n = raw.shape[0]
    gt = torch.from_numpy(metrics.param_targets(op.targets(n), n, v["param_net"], v["predict_params"]))
    weight = float(make_cfg(version).MODEL.PARAM_DECODER.LOSS_WEIGHT)
    got = metrics.param_net_losses(raw, gt, v["param_net"], v["predict_params"], weight)
    ref_keys = [k[len(name) + 6:] for k in golden if k.startswith(name + "/loss/")]
    assert list(got) == ref_keys
    for k in ref_keys:
        ref = float(golden[f"{name}/loss/{k}"])
        assert got[k].dtype == torch.float32 and got[k].dim() == 0
        assert abs(got[k].item() - ref) <= 1e-6 * abs(ref), (k, got[k].item(), ref)


def test_loss_weight_of_each_variant():
    weights = {version: float(make_cfg(version).MODEL.PARAM_DECODER.LOSS_WEIGHT) for _, version, _ in op.CONFIGS}
    assert weights == {"Paramnet-360Cities-edina-centered": 1.0, "Paramnet-360Cities-edina-uncentered": 1.0,
                       "PersNet_Paramnet-GSV-uncentered": 0.1}


def test_param_targets_rule():
    v = VARIANTS["Paramnet-360Cities-edina-centered"]
    x = [{"roll": 10, "pitch": np.float32(-20.3), "vfov": 55.5}]
    gt = metrics.param_targets(x, 1, v["param_net"], v["predict_params"])
    # float64 quotient, then one rounding to float32 (np.float32(-20.3) / 90 in float32 would round twice)
    np.testing.assert_array_equal(gt, np.array([[10 / 90, float(np.float32(-20.3)) / 90, 55.5 / 90, 0, 0]], np.float32))
    with pytest.raises(KeyError):
        metrics.param_targets([{"roll": 1.0, "pitch": 2.0}], 1, v["param_net"], v["predict_params"])
    with pytest.raises(ValueError):
        metrics.param_targets(x, 2, v["param_net"], v["predict_params"])
    with pytest.raises(TypeError):
        metrics.param_targets([{"roll": torch.tensor(1.0), "pitch": 2.0, "vfov": 3.0}], 1, v["param_net"], v["predict_params"])
    u = VARIANTS["PersNet_Paramnet-GSV-uncentered"]
    with pytest.raises(KeyError):
        metrics.param_targets([{"roll": 1.0, "pitch": 2.0, "vfov": 3.0}], 1, u["param_net"], u["predict_params"])
