"""GPU: ParamNet training, ``PerspectiveFields.param_net_parameters`` / ``param_net_backward`` (pf_param_train_forward +
pf_param_backward).

1. Every parameter gradient and both field gradients match float64 autograd through ``oracle.model.convnext_t`` +
   ``metrics.param_net_losses`` to 1e-3 normwise relative error per tensor (three configurations, camera and random fields, a
   rectangular working size), and to a looser bound at ``precision="bf16"``.
2. The losses are ``param_losses``' bit for bit; ``param_net`` is unchanged by a backward.
3. Two identical calls give bit-identical gradients; two calls without ``zero_grad`` give exactly twice one call.
4. Parameter semantics: ``state_dict()``, in-place updates reaching ``param_net`` / ``inference_batch``, ``load_state_dict`` in place.
5. Five SGD steps follow the same five steps of the oracle on the CPU.
6. Rejected calls launch nothing; the C ABI returns PF_ERR_ARG before any launch.  7. Nothing synchronises with the host.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_paramnet as op
import pf_test_util as U
from oracle import model as om
from oracle import panocam as oracle_panocam
from oracle import weights_gen as wg
from perspectivefields_b200 import PerspectiveFields, _native, metrics
from perspectivefields_b200.variants import VARIANTS, make_cfg

pytestmark = pytest.mark.gpu

CENTRED = "Paramnet-360Cities-edina-centered"
GSV_UNC = "PersNet_Paramnet-GSV-uncentered"
VERSIONS = [c[1] for c in op.CONFIGS]
PF_ERR_ARG = -1


def _model(version, seed=0, **kw):
    return U.make_model(version, seed=seed, device="cuda", model_kwargs=kw)


def _launches():
    return _native.lib().pf_kernel_launch_count()


def _fields(kind, n, h, w, seed):
    """(gravity [n, 2, h, w], sin(latitude) [n, 1, h, w]) float32 on the CPU: seeded camera fields or random fields."""
    rs = np.random.RandomState(seed)
    if kind == "random":
        g = torch.Generator().manual_seed(seed)
        return torch.randn((n, 2, h, w), generator=g), torch.rand((n, 1, h, w), generator=g) * 2 - 1
    ups, lats = [], []
    for _ in range(n):
        roll, pitch, vfov = rs.uniform(-30, 30), rs.uniform(-40, 40), rs.uniform(40, 90)
        f = 1.0 / (2.0 * math.tan(math.radians(vfov) / 2.0))
        args = (f, w, h, math.radians(pitch), math.radians(roll), 0.0, 0.0)
        ups.append(np.asarray(oracle_panocam.get_up_general(*args), np.float64).transpose(2, 0, 1))
        lats.append(np.sin(np.radians(np.asarray(oracle_panocam.get_lat_general(*args), np.float64)))[None])
    return torch.from_numpy(np.stack(ups).astype(np.float32)), torch.from_numpy(np.stack(lats).astype(np.float32))


def _oracle(sd, version, grav, lat, inputs, device="cpu"):
    """float64 autograd on `device`: (losses, {param key: grad}, (d gravity, d latitude), raw)."""
    cfg = VARIANTS[version]
    p = {k: v.double().to(device).requires_grad_(True) for k, v in sd.items() if k.startswith("param_net.backbone.")}
    g = grav.double().to(device).requires_grad_(True)
    la = lat.double().to(device).requires_grad_(True)
    images = torch.cat((g, la), 1)
    if cfg["param_net"] != "ParamNet":
        images = F.interpolate(images, (cfg["input_size"], cfg["input_size"]))
    raw = om.convnext_t(p, images)
    gt = torch.from_numpy(metrics.param_targets(inputs, grav.shape[0], cfg["param_net"], cfg["predict_params"])).double().to(device)
    lw = float(make_cfg(version).MODEL.PARAM_DECODER.LOSS_WEIGHT)
    losses = metrics.param_net_losses(raw, gt, cfg["param_net"], cfg["predict_params"], lw)
    sum(losses.values()).backward()
    return losses, {k: v.grad for k, v in p.items()}, (g.grad, la.grad), raw.detach(), gt


def _normwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _grads(params):
    return {k: p.grad.detach().clone() for k, p in params.items()}


# ------------------------------------------------------------------------------------------------ 1. oracle parity
# n = 13 centred pairs at 320 x 320: 1040 stem rows, past the 1024 partials of the depthwise and stem weight-gradient kernels,
# so their blocks take two image rows each; its float64 oracle runs on the GPU
CASES = [(v, kind, None, 3) for v in VERSIONS for kind in ("camera", "random")] + [
    (CENTRED, "camera", (256, 384), 3), (GSV_UNC, "random", (256, 384), 3), (CENTRED, "camera", None, 13)]
# the ids the cases had before the batch size was a parameter (pytest's own for the first three values), "-n<n>" otherwise
CASE_IDS = [f"{v}-{k}-{'None' if r is None else f'resize{i}'}" + ("" if n == 3 else f"-n{n}") for i, (v, k, r, n) in enumerate(CASES)]


@pytest.mark.parametrize("version,kind,resize,n", CASES, ids=CASE_IDS)
def test_gradients_match_the_oracle(version, kind, resize, n):
    m, sd = _model(version, resize=resize)
    h, w = m.net_size()
    grav, lat = _fields(kind, n, h, w, seed=31)
    inputs = op.targets(n, seed=41)
    o_losses, o_grads, (o_dg, o_dl), raw, gt = _oracle(sd, version, grav, lat, inputs, device="cuda" if n > 3 else "cpu")
    if VARIANTS[version]["param_net"] == "ParamNet":
        # the L1 loss has a kink at raw = gt: every compared entry must be clear of it
        assert (raw - gt)[:, :3].abs().min() > 1e-3
    params = m.param_net_parameters()
    assert list(params) == list(o_grads)
    losses, dfields = m.param_net_backward({"pred_gravity": grav.cuda(), "pred_latitude": lat.cuda()}, inputs, input_grads=True)
    for k, v in o_losses.items():
        assert abs(losses[k].item() - v.item()) <= 1e-4 * abs(v.item()), k
    worst = max((_normwise(params[k].grad, g), k) for k, g in o_grads.items())
    assert worst[0] <= 1e-3, worst
    assert _normwise(dfields["pred_gravity"], o_dg) <= 1e-3
    assert _normwise(dfields["pred_latitude"], o_dl) <= 1e-3
    if VARIANTS[version]["param_net"] != "ParamNet":
        # the nearest sub-sample reads few pixels: the rest of the field gradient is exactly zero, as in autograd
        assert torch.equal(dfields["pred_gravity"].cpu() == 0, o_dg.cpu() == 0)


# one bf16 product per MMA: worst error measured on an H100 6.9e-3 (DESIGN.md, ParamNet training); bound with a 3x margin
BF16_BOUND = 2e-2


@pytest.mark.parametrize("version", [CENTRED, GSV_UNC])
def test_gradients_at_bf16(version):
    m, sd = _model(version, precision="bf16")
    h, w = m.net_size()
    grav, lat = _fields("camera", 3, h, w, seed=31)
    inputs = op.targets(3, seed=41)
    _, o_grads, _, _, _ = _oracle(sd, version, grav, lat, inputs)
    params = m.param_net_parameters()
    m.param_net_backward({"pred_gravity": grav.cuda(), "pred_latitude": lat.cuda()}, inputs)
    errs = {k: _normwise(params[k].grad, g) for k, g in o_grads.items()}
    worst = max(errs.values())
    print(f"bf16 {version}: worst normwise gradient error {worst:.3g}")
    assert worst <= BF16_BOUND, max(errs, key=errs.get)


# ------------------------------------------------------------------------------------------------ 2-3. losses, determinism
@pytest.mark.parametrize("version", [CENTRED, GSV_UNC])
def test_losses_determinism_and_accumulation(version):
    m, _ = _model(version)
    h, w = m.net_size()
    grav, lat = _fields("camera", 4, h, w, seed=5)
    preds = {"pred_gravity": grav.cuda(), "pred_latitude": lat.cuda()}
    inputs = op.targets(4, seed=6)
    before = m.param_net(preds)
    ref = m.param_losses(preds, inputs)
    params = m.param_net_parameters()
    losses = m.param_net_backward(preds, inputs)
    assert list(losses) == list(ref)
    for k in ref:
        assert torch.equal(losses[k], ref[k]), k
    after = m.param_net(preds)
    for k in before:
        assert torch.equal(before[k], after[k]), k
    g1 = _grads(params)
    for p in params.values():
        p.grad = None
    m.param_net_backward(preds, inputs)
    g2 = _grads(params)
    m.param_net_backward(preds, inputs)
    for k in params:
        assert torch.equal(g1[k], g2[k]), k
        assert torch.equal(params[k].grad, 2 * g1[k]), k


# ------------------------------------------------------------------------------------------------ 4. parameters
def test_parameters_follow_updates_and_load_state_dict():
    m, _ = _model(GSV_UNC)
    params = m.param_net_parameters()
    sd = m.state_dict()
    for k, p in params.items():
        assert p.device.type == "cuda" and p.dtype == torch.float32
        assert torch.equal(p.detach().cpu(), sd[k].float().cpu()), k
    assert not any(p is q for p in params.values() for q in m.parameters())
    h, w = m.net_size()
    grav, lat = _fields("camera", 3, h, w, seed=9)
    preds = {"pred_gravity": grav.cuda(), "pred_latitude": lat.cuda()}
    imgs = wg.smooth_images(2, 240, 320, seed=4)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in params.values():
            p.mul_(1.0 + 0.01 * torch.randn(p.shape, generator=g).to(p.device))
    got = m.param_net(preds)
    got_inf = m.inference_batch(imgs)
    new_sd = m.state_dict()
    for k, p in params.items():
        assert torch.equal(new_sd[k].to(p.device), p.detach()), k
    fresh = PerspectiveFields(GSV_UNC).cuda().eval()
    fresh.load_state_dict({k: v.cpu() for k, v in new_sd.items()})
    want = fresh.param_net(preds)
    want_inf = fresh.inference_batch(imgs)
    for k in want:
        assert torch.equal(got[k], want[k]), k
    for a, b in zip(got_inf, want_inf):
        for k in ("pred_roll", "pred_pitch", "pred_general_vfov"):
            assert torch.equal(a[k], b[k]), k
    # load_state_dict writes into the existing parameters
    ptrs = {k: p.data_ptr() for k, p in params.items()}
    m.load_state_dict(fresh.state_dict())
    again = m.param_net_parameters()
    for k, p in again.items():
        assert p is params[k] and p.data_ptr() == ptrs[k]
    assert torch.equal(m.param_net(preds)["pred_roll"], want["pred_roll"])


# ------------------------------------------------------------------------------------------------ 5. training trajectory
def test_sgd_trajectory_matches_the_oracle():
    version = GSV_UNC
    m, sd = _model(version)
    h, w = m.net_size()
    grav, lat = _fields("camera", 16, h, w, seed=12)
    inputs = op.targets(16, seed=13)
    preds = {"pred_gravity": grav.cuda(), "pred_latitude": lat.cuda()}
    params = m.param_net_parameters()
    opt = torch.optim.SGD(params.values(), lr=3e-3)
    ref = {k: v.float().clone().requires_grad_(True) for k, v in sd.items() if k.startswith("param_net.backbone.")}
    ref_opt = torch.optim.SGD(ref.values(), lr=3e-3)
    cfg = VARIANTS[version]
    gt = torch.from_numpy(metrics.param_targets(inputs, 16, cfg["param_net"], cfg["predict_params"]))
    lw = float(make_cfg(version).MODEL.PARAM_DECODER.LOSS_WEIGHT)
    ours, theirs = [], []
    for _ in range(5):
        opt.zero_grad()
        ours.append(sum(m.param_net_backward(preds, inputs).values()).item())
        opt.step()
        ref_opt.zero_grad()
        images = F.interpolate(torch.cat((grav, lat), 1), (cfg["input_size"], cfg["input_size"]))
        loss = sum(metrics.param_net_losses(om.convnext_t(ref, images), gt, cfg["param_net"], cfg["predict_params"], lw).values())
        theirs.append(loss.item())
        loss.backward()
        ref_opt.step()
    print("losses", ours, theirs)
    for a, b in zip(ours, theirs):
        assert abs(a - b) <= 1e-3 * abs(b)
    assert ours[-1] < ours[0]


# ------------------------------------------------------------------------------------------------ 6. rejected calls
def test_rejected_calls_launch_nothing():
    m, _ = _model(CENTRED)
    h, w = m.net_size()
    grav, lat = _fields("random", 2, h, w, seed=1)
    good = {"pred_gravity": grav.cuda(), "pred_latitude": lat.cuda()}
    inputs = op.targets(2)
    persnet, _ = _model("PersNet-360Cities")
    cpu_model = PerspectiveFields(CENTRED)
    m.param_net_backward(good, inputs)   # first call registers the training tensors
    torch.cuda.synchronize()
    cases = [
        (persnet.param_net_parameters, (), ValueError),
        (persnet.param_net_backward, (good, inputs), ValueError),
        (cpu_model.param_net_backward, ({k: v.cpu() for k, v in good.items()}, inputs), RuntimeError),
        (m.param_net_backward, ({"pred_gravity": grav[:, :, :64].cuda(), "pred_latitude": lat.cuda()}, inputs), ValueError),
        (m.param_net_backward, ({"pred_gravity": grav.double().cuda(), "pred_latitude": lat.cuda()}, inputs), (TypeError, ValueError)),
        (m.param_net_backward, ({"pred_gravity": grav, "pred_latitude": lat.cuda()}, inputs), (TypeError, ValueError)),
        (m.param_net_backward, (good, inputs[:1]), ValueError),
        (m.param_net_backward, (good, [{"roll": 1.0, "pitch": 2.0}] * 2), KeyError),
    ]
    for fn, args, exc in cases:
        before = _launches()
        with pytest.raises(exc):
            fn(*args)
        assert _launches() == before, fn
    eng = m._get_engine()
    L = eng.L
    need = L.pf_param_train_workspace_bytes(eng.handle, 2)
    assert need > 0
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    draw = torch.zeros((2, 5), device="cuda")
    grads = torch.empty(L.pf_param_grad_numel(), device="cuda")
    s = U.stream_ptr()
    wp = ws.data_ptr()
    bad = [
        lambda: L.pf_param_backward(None, 2, draw.data_ptr(), grads.data_ptr(), None, None, wp, need, s),
        lambda: L.pf_param_backward(eng.handle, 0, draw.data_ptr(), grads.data_ptr(), None, None, wp, need, s),
        lambda: L.pf_param_backward(eng.handle, 2, None, grads.data_ptr(), None, None, wp, need, s),
        lambda: L.pf_param_backward(eng.handle, 2, draw.data_ptr(), None, None, None, wp, need, s),
        lambda: L.pf_param_backward(eng.handle, 2, draw.data_ptr(), grads.data_ptr(), grads.data_ptr(), None, wp, need, s),
        lambda: L.pf_param_backward(eng.handle, 2, draw.data_ptr(), grads.data_ptr(), None, None, wp, need - 8192, s),
        lambda: L.pf_param_backward(eng.handle, 2, draw.data_ptr(), grads.data_ptr(), None, None, wp + 16, need, s),
        lambda: L.pf_param_train_forward(eng.handle, 0, good["pred_gravity"].data_ptr(), good["pred_latitude"].data_ptr(), draw.data_ptr(), wp, need, s),
        lambda: L.pf_param_train_forward(eng.handle, 2, None, good["pred_latitude"].data_ptr(), draw.data_ptr(), wp, need, s),
        lambda: L.pf_param_train_forward(eng.handle, 2, good["pred_gravity"].data_ptr(), good["pred_latitude"].data_ptr(), None, wp, need, s),
    ]
    for call in bad:
        before = _launches()
        assert call() == PF_ERR_ARG
        assert _launches() == before
    p_eng = persnet._get_engine()
    assert L.pf_param_train_workspace_bytes(p_eng.handle, 2) == PF_ERR_ARG
    assert L.pf_param_backward(p_eng.handle, 2, draw.data_ptr(), grads.data_ptr(), None, None, wp, need, s) == PF_ERR_ARG
    assert L.pf_param_grad_entry(-1, ctypes.byref(ctypes.c_char_p()), ctypes.byref(ctypes.c_int64()), ctypes.byref(ctypes.c_int64())) == PF_ERR_ARG


def test_workspace_of_256_centred_pairs():
    m, _ = _model(CENTRED)
    eng = m._get_engine()
    need = eng.L.pf_param_train_workspace_bytes(eng.handle, 256)
    print(f"training workspace: {need / 2**30:.2f} GiB for 256 centred pairs, {need / 256 / 2**20:.1f} MiB per pair")
    assert 0 < need <= 16 * 2**30


# ------------------------------------------------------------------------------------------------ 7. no synchronisation
@pytest.mark.parametrize("version", [CENTRED, GSV_UNC])
def test_backward_does_not_synchronise(version):
    m, _ = _model(version)
    h, w = m.net_size()
    grav, lat = _fields("random", 2, h, w, seed=3)
    preds = {"pred_gravity": grav.cuda(), "pred_latitude": lat.cuda()}
    inputs = op.targets(2)
    params = m.param_net_parameters()
    m.param_net_backward(preds, inputs)        # registers the training tensors (host work, allowed to synchronise)
    with torch.no_grad():
        next(iter(params.values())).add_(1e-3)   # forces a re-derivation inside the checked call
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses, d = m.param_net_backward(preds, inputs, input_grads=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert all(torch.isfinite(v) for v in losses.values())
    assert torch.isfinite(d["pred_gravity"]).all()
