"""CPU: the gradients of ParamNet's training losses, pinned to the unmodified reference by tests/golden/paramnet_grads.npz
(tests/golden/make_golden_paramnet_grads.py).

float64 autograd through ``oracle.model.convnext_t`` (with the uncentred class's nearest resample in front) and
``metrics.param_net_losses`` -- the oracle the GPU gradients of ``PerspectiveFields.param_net_backward`` are tested against -- on
the seeded fields and targets of tests/oracle_paramnet.py reproduces the reference's float32 gradients of
``sum(pn(preds, batched_inputs).values())`` for the three configurations: every parameter's gradient norm, sum, sampled entries and
(for the small tensors) every entry, and the two field gradients' norms and samples.

Bound: the reference computes in float32, so each of its gradients carries the rounding of a float32 forward and backward through
ConvNeXt-T, about 1e-5 of the tensor's norm; 1e-4 of the norm leaves a margin.  Sums are checked against the norm times sqrt(numel)
(a sum can cancel to almost nothing).
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_paramnet as op
import paramnet_grads_fixture as fx
from oracle import model as om
from oracle import panocam as oracle_panocam
from perspectivefields_b200 import metrics
from perspectivefields_b200.variants import VARIANTS, make_cfg

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "paramnet_grads.npz")
BOUND = 1e-4


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def fields():
    return op.inputs(oracle_panocam.get_up_general, oracle_panocam.get_lat_general)


@pytest.mark.parametrize("name,version,seed", op.CONFIGS)
def test_oracle_gradients_match_reference(golden, fields, name, version, seed):
    cfg = VARIANTS[version]
    sd = {k: v.double().requires_grad_(True) for k, v in op.param_state(version, seed).items() if k.startswith("param_net.backbone.")}
    g = fields[0].double().requires_grad_(True)
    la = fields[1].double().requires_grad_(True)
    images = torch.cat((g, la), 1)
    if cfg["param_net"] != "ParamNet":
        images = F.interpolate(images, (cfg["input_size"], cfg["input_size"]))
    raw = om.convnext_t(sd, images)
    n = g.shape[0]
    gt = torch.from_numpy(metrics.param_targets(op.targets(n), n, cfg["param_net"], cfg["predict_params"])).double()
    lw = float(make_cfg(version).MODEL.PARAM_DECODER.LOSS_WEIGHT)
    sum(metrics.param_net_losses(raw, gt, cfg["param_net"], cfg["predict_params"], lw).values()).backward()
    tensors = {k: p.grad for k, p in sd.items()}
    tensors["input/pred_gravity"] = g.grad
    tensors["input/pred_latitude"] = la.grad
    names = [str(k) for k in golden[f"{name}/names"]]
    assert names == list(tensors)
    full, off = golden[f"{name}/full"], 0
    for i, (k, t) in enumerate(tensors.items()):
        flat = t.reshape(-1).numpy()
        assert flat.size == golden[f"{name}/numel"][i], k
        ref_norm = golden[f"{name}/norm"][i]
        tol = BOUND * ref_norm
        assert abs(np.linalg.norm(flat) - ref_norm) <= tol, k
        assert abs(flat.sum() - golden[f"{name}/sum"][i]) <= tol * np.sqrt(flat.size), k
        assert np.abs(flat[fx.sample_idx(k, flat.size)] - golden[f"{name}/val"][i]).max() <= tol, k
        if flat.size <= fx.FULL_MAX:
            assert np.linalg.norm(flat - full[off:off + flat.size]) <= tol, k
            off += flat.size
    assert off == full.size
