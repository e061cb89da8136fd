"""GPU: ``PerspectiveFields.param_net`` / ``param_losses``, ParamNet on the caller's fields (pf_param_forward).

1. Bit-identity with the forward: ParamNet on the stacked fields of one ``inference_batch`` returns that call's parameters
   exactly, for both ParamNet classes, both precisions and a rectangular working size; the first k rows alone give the same rows.
2. Oracle parity on ground-truth fields (camera fields -> ``targets_from_fields`` -> ``param_net``) at 1e-3 per key.
3. ``param_losses`` against the oracle's raw outputs passed through the same rule, within the bound a 1e-3 error of the raw
   outputs implies; GSV-uncentred exercises LOSS_WEIGHT 0.1.
4. Rejected calls raise before any launch; the C ABI rejects its bad arguments with an error code.
5. Strided inputs give the results of contiguous ones.  6. Neither call synchronises with the host.
"""
import math

import numpy as np
import pytest
import torch

import oracle_paramnet as op
import pf_test_util as U
from oracle import model as om
from oracle import weights_gen as wg
from oracle.variants import VARIANTS as ORACLE_VARIANTS
from perspectivefields_b200 import PerspectiveFields, _native, metrics, panocam
from perspectivefields_b200.variants import VARIANTS, make_cfg

pytestmark = pytest.mark.gpu

CENTRED = "Paramnet-360Cities-edina-centered"
GSV_UNC = "PersNet_Paramnet-GSV-uncentered"
_MODELS = {}


def _model(version, **kw):
    """(model on cuda, reference-layout state dict), one per (version, options) for the whole module."""
    key = (version, tuple(sorted(kw.items())))
    if key not in _MODELS:
        _MODELS[key] = U.make_model(version, seed=0, device="cuda", model_kwargs=kw)
    return _MODELS[key]


def _launches():
    return _native.lib().pf_kernel_launch_count()


def _stacked(results):
    return {"pred_gravity": torch.stack([r["pred_gravity"] for r in results]), "pred_latitude": torch.stack([r["pred_latitude"] for r in results])}


def _class_keys(version):
    if VARIANTS[version]["param_net"] == "ParamNet":
        return ["pred_roll", "pred_pitch", "pred_vfov", "pred_rel_focal"]
    return ["pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy", "pred_rel_focal"]


# ------------------------------------------------------------------------------------------------ 1. bit-identity
@pytest.mark.parametrize("version,kw", [
    (CENTRED, {}), (CENTRED, {"precision": "bf16"}), (GSV_UNC, {}), (GSV_UNC, {"precision": "bf16"}),
    ("PersNet_Paramnet-GSV-centered", {"resize": (256, 384)})])
def test_param_net_is_bit_identical_to_the_forward(version, kw):
    m, _ = _model(version, **kw)
    res = m.inference_batch(wg.smooth_images(5, 240, 320, seed=4))
    preds = _stacked(res)
    out = m.param_net(preds)
    assert list(out) == _class_keys(version)
    for k, v in out.items():
        assert v.dtype == torch.float32 and v.shape == (5,) and v.device == preds["pred_gravity"].device, k
        assert torch.equal(v, torch.stack([r[k] for r in res])), k
    for k_rows in (1, 3):     # a smaller batch changes the tiles of every GEMM, not a row's result
        sub = m.param_net({k: v[:k_rows] for k, v in preds.items()})
        for k, v in sub.items():
            assert torch.equal(v, out[k][:k_rows]), (k_rows, k)


# ------------------------------------------------------------------------------------------------ 2. oracle parity
def _gt_fields(m, version, n=6, seed=7):
    """Seeded cameras -> ground-truth fields at the working size -> ``targets_from_fields`` -> ``param_net`` predictions."""
    rs = np.random.RandomState(seed)
    roll, pitch, vfov = rs.uniform(-30, 30, n), rs.uniform(-40, 40, n), rs.uniform(40, 90, n)
    h, w = m.net_size()
    r, p, v = [math.radians(x) for x in roll], [math.radians(x) for x in pitch], [math.radians(x) for x in vfov]
    if VARIANTS[version]["param_net"] == "ParamNet":
        ups, lats = panocam.pinhole_fields(v, [h] * n, [w] * n, p, r)
    else:
        cx, cy = rs.uniform(-0.1, 0.1, n), rs.uniform(-0.1, 0.1, n)
        ups, lats = panocam.camera_fields([1 / (2 * math.tan(x / 2)) for x in v], [h] * n, [w] * n, p, r, cx, cy)
    t = m.targets_from_fields(ups, lats)
    return {"pred_gravity": t["gt_gravity"], "pred_latitude": t["gt_latitude"]}


_ORACLE = {}


def _oracle(version, sd, preds):
    """oracle.model.param_net on the same float32 fields: (result dict, raw backbone output [n, 5])."""
    if version not in _ORACLE:
        taps = {}
        with torch.no_grad():
            out = om.param_net(sd, ORACLE_VARIANTS[version], preds["pred_gravity"].cpu(), preds["pred_latitude"].cpu(), taps)
        _ORACLE[version] = (out, taps["cnx.out"])
    return _ORACLE[version]


@pytest.mark.parametrize("version", [CENTRED, "Paramnet-360Cities-edina-uncentered", GSV_UNC])
def test_param_net_matches_oracle_on_ground_truth_fields(version):
    m, sd = _model(version)
    preds = _gt_fields(m, version)
    out = m.param_net(preds)
    ref, _ = _oracle(version, sd, preds)
    for k, v in out.items():
        e = U.rel_err(v, ref[k])
        assert e < 1e-3, (version, k, e)


# ------------------------------------------------------------------------------------------------ 3. losses
@pytest.mark.parametrize("version", [CENTRED, GSV_UNC])
def test_param_losses_match_oracle(version):
    m, sd = _model(version)
    preds = _gt_fields(m, version)
    n = preds["pred_gravity"].shape[0]
    batched_inputs = op.targets(n)
    got = m.param_losses(preds, batched_inputs)
    _, raw = _oracle(version, sd, preds)
    v = VARIANTS[version]
    gt = torch.from_numpy(metrics.param_targets(batched_inputs, n, v["param_net"], v["predict_params"]))
    weight = float(make_cfg(version).MODEL.PARAM_DECODER.LOSS_WEIGHT)
    ref = metrics.param_net_losses(raw, gt, v["param_net"], v["predict_params"], weight)
    assert list(got) == list(ref)
    # the bound a raw error of at most eps_k = 1e-3 max_i |raw[i, k]| per output (the 1e-3 bar of test 2) implies:
    #   L1:  |mean(|x' - g| m) - mean(|x - g| m)| <= mean(|x' - x| m) <= w sum_{k<3} eps_k / 5
    #   MSE: |(x' - g)^2 - (x - g)^2| = |x' - x| |x' + x - 2g| <= eps_k (2 |x - g| + eps_k), averaged over the rows, times w
    # plus 1e-6 relative for float32 rounding of the sums
    eps = 1e-3 * raw.double().abs().max(0).values
    d = (raw.double() - gt.double()).abs()
    if v["param_net"] == "ParamNet":
        bounds = {"param-l1-loss": weight * eps[:3].sum().item() / 5}
    else:
        bounds = {f"param/{k}-loss": weight * (eps[j] * (2 * d[:, j] + eps[j])).mean().item() for j, k in enumerate(v["predict_params"])}
    for k, val in got.items():
        assert val.dtype == torch.float32 and val.dim() == 0 and val.is_cuda, k
        r = ref[k].item()
        assert abs(val.item() - r) <= bounds[k] + 1e-6 * abs(r), (version, k, val.item(), r, bounds[k])


# ------------------------------------------------------------------------------------------------ 4. errors
def test_rejected_calls_launch_nothing():
    m, _ = _model(CENTRED)
    h, w = m.net_size()
    g = torch.zeros((2, 2, h, w), device="cuda")
    l = torch.zeros((2, 1, h, w), device="cuda")
    ok_inputs = [{"roll": 1.0, "pitch": 2.0, "vfov": 60.0}] * 2
    m.param_net({"pred_gravity": g, "pred_latitude": l})        # the engine exists: what follows measures the calls alone
    torch.cuda.synchronize()
    persnet = _model("PersNet-360Cities")[0]
    cpu_model = PerspectiveFields(CENTRED)
    cases = [
        (persnet, {"pred_gravity": g, "pred_latitude": l}, None),                                    # no ParamNet in the variant
        (cpu_model, {"pred_gravity": g.cpu(), "pred_latitude": l.cpu()}, None),                      # CPU model
        (m, {"pred_gravity": g[:, :, :, :w - 32], "pred_latitude": l[:, :, :, :w - 32]}, None),      # not the working size
        (m, {"pred_gravity": g[:, :1], "pred_latitude": l}, None),                                   # one gravity channel
        (m, {"pred_gravity": g[0], "pred_latitude": l[0]}, None),                                    # no batch dimension
        (m, {"pred_gravity": g.double(), "pred_latitude": l}, None),                                 # dtype
        (m, {"pred_gravity": g.cpu(), "pred_latitude": l.cpu()}, None),                              # device
        (m, {"pred_gravity": g[:0], "pred_latitude": l[:0]}, None),                                  # n = 0
        (m, {"pred_gravity": g, "pred_latitude": l[:1]}, None),                                      # mismatched n
        (m, {"pred_gravity": g}, None),                                                              # missing key
        (m, {"pred_gravity": g, "pred_latitude": l}, [{"roll": 1.0, "pitch": 2.0}] * 2),             # missing target key
        (m, {"pred_gravity": g, "pred_latitude": l}, ok_inputs[:1]),                                 # targets for another n
        (m, {"pred_gravity": g, "pred_latitude": l}, [{"roll": torch.tensor(1.0, device="cuda"), "pitch": 2.0, "vfov": 3.0}] * 2),
    ]
    for i, (model, preds, inputs) in enumerate(cases):
        calls = [lambda: model.param_losses(preds, inputs)] if inputs is not None else \
            [lambda: model.param_net(preds), lambda: model.param_losses(preds, ok_inputs)]
        for call in calls:
            before = _launches()
            with pytest.raises((ValueError, TypeError, KeyError, RuntimeError)):
                call()
            assert _launches() == before, i


def test_c_abi_rejects_bad_arguments_before_launching():
    m, _ = _model(CENTRED)
    eng = m._get_engine()
    L = eng.L
    h, w = m.net_size()
    g = torch.zeros((2, 2, h, w), device="cuda")
    l = torch.zeros((2, 1, h, w), device="cuda")
    p = torch.empty((2, 8), device="cuda")
    need = L.pf_param_workspace_bytes(eng.handle, 2)
    assert need > 0
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    before = _launches()
    assert L.pf_param_workspace_bytes(eng.handle, 0) < 0
    assert L.pf_param_forward(eng.handle, 0, g.data_ptr(), l.data_ptr(), p.data_ptr(), None, ws.data_ptr(), need, s) < 0
    assert L.pf_param_forward(eng.handle, 2, None, l.data_ptr(), p.data_ptr(), None, ws.data_ptr(), need, s) < 0
    assert L.pf_param_forward(eng.handle, 2, g.data_ptr(), None, p.data_ptr(), None, ws.data_ptr(), need, s) < 0
    assert L.pf_param_forward(eng.handle, 2, g.data_ptr(), l.data_ptr(), None, None, ws.data_ptr(), need, s) < 0
    assert L.pf_param_forward(eng.handle, 2, g.data_ptr(), l.data_ptr(), p.data_ptr(), None, None, need, s) < 0
    assert L.pf_param_forward(eng.handle, 2, g.data_ptr(), l.data_ptr(), p.data_ptr(), None, ws.data_ptr(), need - 4097, s) < 0
    assert b"workspace" in L.pf_last_error()
    assert L.pf_param_forward(eng.handle, 2, g.data_ptr(), l.data_ptr(), p.data_ptr(), None, ws.data_ptr() + 16, need, s) < 0
    pe = _model("PersNet-360Cities")[0]._get_engine()
    assert L.pf_param_workspace_bytes(pe.handle, 1) < 0
    assert L.pf_param_forward(pe.handle, 2, g.data_ptr(), l.data_ptr(), p.data_ptr(), None, ws.data_ptr(), need, s) < 0
    assert b"ParamNet" in L.pf_last_error()
    assert _launches() == before


# ------------------------------------------------------------------------------------------------ 5. strided inputs
def test_strided_inputs_match_contiguous_ones():
    m, _ = _model(GSV_UNC)
    preds = _gt_fields(m, GSV_UNC, n=3, seed=9)
    g, l = preds["pred_gravity"], preds["pred_latitude"]
    g_nc = g.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)          # [n, 2, H, W] view of [n, H, W, 2] storage
    l_nc = torch.cat([l, l], dim=3)[..., ::2]
    l_nc.copy_(l)
    assert not g_nc.is_contiguous() and not l_nc.is_contiguous()
    a, b = m.param_net(preds), m.param_net({"pred_gravity": g_nc, "pred_latitude": l_nc})
    for k in a:
        assert torch.equal(a[k], b[k]), k
    inputs = op.targets(3)
    la, lb = m.param_losses(preds, inputs), m.param_losses({"pred_gravity": g_nc, "pred_latitude": l_nc}, inputs)
    for k in la:
        assert torch.equal(la[k], lb[k]), k


# ------------------------------------------------------------------------------------------------ 6. no synchronisation
@pytest.mark.parametrize("version", [CENTRED, GSV_UNC])
def test_calls_do_not_synchronise(version):
    m, _ = _model(version)
    preds = _gt_fields(m, version, n=2, seed=3)
    inputs = op.targets(2)
    m.param_net(preds)
    m.param_losses(preds, inputs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = m.param_net(preds)
        losses = m.param_losses(preds, inputs)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert all(torch.isfinite(v).all() for v in out.values())
    assert all(torch.isfinite(v) for v in losses.values())
