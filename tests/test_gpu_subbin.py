"""GPU: the sub-bin decode of the classification heads (PerspectiveFields(decode="subbin"), engine option "subbin",
pf_op_subbin_decode / pf_op_pred_subbin_decode) against the float32 oracle tests/oracle_subbin.py, against the argmax decode on
the same inputs, and against the true fields of synthetic cameras."""
import math

import numpy as np
import pytest
import torch

import oracle_subbin as osb
import pf_test_util as U
from oracle import weights_gen as wg
from perspectivefields_b200 import PerspectiveFields, _native, calibrate, panocam

pytestmark = pytest.mark.gpu

VERSION = "PersNet-360Cities"
NC = {"gravity": 73, "latitude": 180}
LAT_TOL, UP_TOL = 1e-5, 1e-6     # degrees / unit-vector components, the ops against the oracle


def _run_logits_op(logits, is_gravity, conf=False, refine=True):
    """[B, NC, HW] device logits -> (field [B, 2 or 1, HW], conf [B, HW] or None) through pf_op_subbin_decode / pf_op_argmax_decode."""
    B, nc, HW = logits.shape
    field = torch.full((B, 2 if is_gravity else 1, HW), float("nan"), device="cuda")
    cf = torch.full((B, HW), float("nan"), device="cuda") if conf else None
    L = _native.lib()
    if refine:
        _native.check(L.pf_op_subbin_decode(logits.data_ptr(), field.data_ptr(), cf.data_ptr() if conf else None, B, HW, nc, int(is_gravity),
                                            U.stream_ptr()))
    else:
        _native.check(L.pf_op_argmax_decode(logits.data_ptr(), field.data_ptr(), B, HW, nc, int(is_gravity), U.stream_ptr()))
    torch.cuda.synchronize()
    return field, cf


def _run_fused_op(feat, coff, w, b, B, HW, is_gravity, conf=False):
    nc = w.shape[0]
    field = torch.full((B, 2 if is_gravity else 1, HW), float("nan"), device="cuda")
    cf = torch.full((B, HW), float("nan"), device="cuda") if conf else None
    _native.check(_native.lib().pf_op_pred_subbin_decode(feat.data_ptr(), feat.shape[1], coff, w.data_ptr(), b.data_ptr(), field.data_ptr(),
                                                         cf.data_ptr() if conf else None, B, HW, nc, int(is_gravity), U.stream_ptr()))
    torch.cuda.synchronize()
    return field, cf


def _oracle(logits_bnhw, is_gravity):
    """Oracle fields [B, 2 or 1, HW] of [B, NC, HW] logits."""
    l = logits_bnhw.cpu().numpy()
    if is_gravity:
        return torch.from_numpy(osb.decode_gravity(l, axis=1))
    return torch.from_numpy(osb.decode_latitude(l, axis=1)).unsqueeze(1)


def _check_field(got, want, is_gravity):
    err = (got.cpu() - want).abs().max().item()
    assert err <= (UP_TOL if is_gravity else LAT_TOL), err
    return err


def _hand_made_logits(B, HW, nc, is_gravity, seed):
    """Peaked logits (a parabola of random width around a random sub-bin position, plus noise) with the edge cases spliced in:
    ties, symmetric neighbours, the wrap of the up head, bin 72 and the latitude poles."""
    g = torch.Generator().manual_seed(seed)
    nd = nc - 1 if is_gravity else nc
    mu = torch.rand(B, 1, HW, generator=g) * nd
    sigma = 0.5 + 2 * torch.rand(B, 1, HW, generator=g)
    c = torch.arange(nc, dtype=torch.float32).view(1, nc, 1)
    d = c - mu
    if is_gravity:
        d = torch.remainder(d + nd / 2, nd) - nd / 2
    l = -d * d / (2 * sigma * sigma) + 0.05 * torch.randn(B, nc, HW, generator=g)
    if is_gravity:
        l[:, nc - 1] = -50
        l[0, :, 0] = -5; l[0, nc - 1, 0] = 3                                # bin 72
        l[0, :, 1] = -5; l[0, 0, 1] = 2; l[0, nd - 1, 1] = 1.5; l[0, 1, 1] = 0.5   # across the wrap
    else:
        l[0, :, 0] = -5; l[0, 0, 0] = 2; l[0, 1, 0] = 1                     # pole bins
        l[0, :, 1] = -5; l[0, nc - 1, 1] = 2; l[0, nc - 2, 1] = 1.9
    l[0, :, 2] = 1.0                                                        # all tied
    l[0, :, 3] = -5; l[0, 7, 3] = 1; l[0, 6, 3] = l[0, 8, 3] = 0            # symmetric
    l[0, :, 4] = -5; l[0, 7, 4] = l[0, 20, 4] = 1                           # two-way tie
    return l.contiguous()


@pytest.mark.parametrize("is_gravity", [1, 0])
@pytest.mark.parametrize("conf", [False, True])
def test_logits_op_matches_oracle(is_gravity, conf):
    nc = 73 if is_gravity else 180
    B, HW = 3, 1000                      # HW not a multiple of 256
    l = _hand_made_logits(B, HW, nc, is_gravity, seed=nc)
    field, cf = _run_logits_op(l.cuda(), is_gravity, conf)
    _check_field(field, _oracle(l, is_gravity), is_gravity)
    if conf:   # the softmax maximum (the fp32 online sum drifts by a few 1e-6 over 180 rising maxima)
        want = 1.0 / torch.exp(l.double() - l.double().amax(1, keepdim=True)).sum(1)
        assert (cf.cpu().double() / want - 1).abs().max().item() < 2e-5


def _dyadic(B, HW, nc, seed):
    """Features, weights and bias on a coarse dyadic grid: every product and partial sum of the 1x1 conv is exact in fp32, so the
    logits are known exactly (float64 matmul) whatever the order of the sums."""
    g = torch.Generator().manual_seed(seed)
    feat = torch.randint(-8, 9, (B * HW, 64), generator=g).float() / 8
    w = torch.randint(-8, 9, (nc, 32), generator=g).float() / 16
    b = torch.randint(-8, 9, (nc,), generator=g).float() / 16
    return feat, w, b


@pytest.mark.parametrize("is_gravity", [1, 0])
@pytest.mark.parametrize("conf", [False, True])
def test_fused_op_matches_oracle(is_gravity, conf):
    nc = 73 if is_gravity else 180
    B, HW = 2, 777
    coff = 0 if is_gravity else 32
    feat, w, b = _dyadic(B, HW, nc, seed=3 * nc)
    logits = (feat[:, coff:coff + 32].double() @ w.double().t() + b.double()).float().reshape(B, HW, nc).permute(0, 2, 1).contiguous()
    field, _ = _run_fused_op(feat.cuda(), coff, w.cuda(), b.cuda(), B, HW, is_gravity, conf)
    _check_field(field, _oracle(logits, is_gravity), is_gravity)


@pytest.mark.parametrize("is_gravity", [1, 0])
def test_fused_op_equals_logits_op_bit_for_bit(is_gravity):
    """On logits written by the separate 1x1 conv kernel (pf_op_pred_tail, the logits path's tail), with and without conf."""
    nc = 73 if is_gravity else 180
    B, HW = 3, 1111
    coff = 0 if is_gravity else 32
    g = torch.Generator().manual_seed(11 + nc)
    feat = torch.relu(torch.randn(B * HW, 64, generator=g)).cuda()
    w, b = (torch.randn(nc, 32, generator=g) * 0.3).cuda(), (torch.randn(nc, generator=g) * 0.1).cuda()
    logits = torch.empty(B, nc, HW, device="cuda")
    _native.check(_native.lib().pf_op_pred_tail(feat.data_ptr(), 64, coff, w.data_ptr(), b.data_ptr(), logits.data_ptr(), B, HW, nc, 0, U.stream_ptr()))
    torch.cuda.synchronize()
    ref, _ = _run_logits_op(logits, is_gravity)
    _check_field(ref, _oracle(logits, is_gravity), is_gravity)
    for conf in (False, True):
        got, _ = _run_fused_op(feat, coff, w, b, B, HW, is_gravity, conf)
        assert torch.equal(got, ref), conf
        got, _ = _run_logits_op(logits, is_gravity, conf)
        assert torch.equal(got, ref), conf


def test_op_argument_checks():
    L = _native.lib()
    x = torch.zeros(4 * 73 * 16, device="cuda")
    f = torch.zeros(4 * 2 * 16, device="cuda")
    p, q = x.data_ptr(), f.data_ptr()
    before = L.pf_kernel_launch_count()
    assert L.pf_op_subbin_decode(None, q, None, 1, 16, 73, 1, None) == -1
    assert L.pf_op_subbin_decode(p, None, None, 1, 16, 73, 1, None) == -1
    assert L.pf_op_subbin_decode(p, q, None, 0, 16, 73, 1, None) == -1
    assert L.pf_op_subbin_decode(p, q, q + 2, 1, 16, 73, 1, None) == -1
    assert L.pf_op_pred_subbin_decode(p, 66, 0, p, p, q, None, 1, 16, 73, 1, None) == -1     # ld % 4
    assert L.pf_op_pred_subbin_decode(p, 64, 2, p, p, q, None, 1, 16, 73, 1, None) == -1     # coff % 4
    assert L.pf_op_pred_subbin_decode(p, 64, 0, p, p, q, None, 1, 16, 257, 1, None) == -1    # NC > 256
    assert L.pf_op_pred_subbin_decode(p, 64, 0, p, p, q, q + 2, 1, 16, 73, 1, None) == -1
    assert L.pf_kernel_launch_count() == before


# ------------------------------------------------------------------------------------------------ end to end
_cache = {}


def _model(**kw):
    key = tuple(sorted(kw.items()))
    if key not in _cache:
        _cache[key] = U.make_model(VERSION, seed=0, device="cuda", model_kwargs=dict(kw))[0]
    return _cache[key]


def _engine_logits(model, res, imgs, logits):
    """[n, NC, H, W] fp32 logits of both heads: the returned ones, or the debug taps of the prediction convs."""
    if logits:
        return {k: torch.stack([r["pred_" + k] for r in res]).float().cpu() for k in NC}
    model.debug_taps(True)
    try:
        model.inference_batch(imgs)
        taps = model.read_taps()
    finally:
        model.debug_taps(False)
    h, w = model.net_size()
    return {k: taps["head.raw_" + k[0]].view(len(imgs), NC[k], h, w).float().cpu() for k in NC}


@pytest.mark.parametrize("confidence", [False, True])
@pytest.mark.parametrize("resize", [None, (256, 384)])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("logits", [True, False])
def test_end_to_end(logits, precision, resize, confidence):
    kw = dict(logits=logits, precision=precision, resize=resize, confidence=confidence)
    a, s = _model(**kw), _model(decode="subbin", **kw)
    sizes = [(240, 320), (300, 200)]
    imgs = [wg.smooth_images(1, h, w, seed=21 + i)[0] for i, (h, w) in enumerate(sizes)]
    ra, rs = a.inference_batch(imgs), s.inference_batch(imgs)
    decoded = {"pred_gravity_original", "pred_latitude_original"} | (set() if logits else {"pred_gravity", "pred_latitude"})
    for x, y in zip(ra, rs):
        assert list(x) == list(y)
        for k, v in x.items():
            if k not in decoded:
                assert (v == y[k]) if isinstance(v, str) else torch.equal(v, y[k]), k
    lg = _engine_logits(s, rs, imgs, logits)
    net_hw = s.net_size()
    worst = {"up": 0.0, "lat": 0.0, "up_original": 0.0, "lat_original": 0.0}
    changed = 0
    for i, ((h, w), r) in enumerate(zip(sizes, rs)):
        up = osb.decode_gravity(lg["gravity"][i].numpy(), axis=0)
        lat = osb.decode_latitude(lg["latitude"][i].numpy(), axis=0)
        if not logits:
            worst["up"] = max(worst["up"], _check_field(r["pred_gravity"], torch.from_numpy(up), True))
            worst["lat"] = max(worst["lat"], _check_field(r["pred_latitude"][0], torch.from_numpy(lat), False))
        want_g = osb.postprocess_gravity(lg["gravity"][i].numpy(), h, w, net_hw)
        want_l = osb.postprocess_latitude(lg["latitude"][i].numpy(), h, w, net_hw)
        # F.normalize of a bilinear blend of unrelated up vectors can come near zero length, where the direction depends on the
        # last rounding of either side: compare the direction where the blend is at least 0.1 long
        scale = torch.tensor([[w / net_hw[1]], [h / net_hw[0]]]).unsqueeze(-1)
        blend = osb.pf_postprocess(torch.from_numpy(up) * scale, h, w, net_hw).norm(dim=0)
        ok = blend >= 0.1 * min(scale.min().item(), 1.0)
        eu = (r["pred_gravity_original"].cpu() - want_g).abs().amax(0)[ok].max().item()
        el = (r["pred_latitude_original"].cpu() - want_l).abs().max().item()
        worst["up_original"], worst["lat_original"] = max(worst["up_original"], eu), max(worst["lat_original"], el)
        changed += int(not torch.equal(r["pred_latitude_original"], ra[i]["pred_latitude_original"]))
    print(f"subbin end to end {kw}: max |engine - oracle| {worst}")
    assert worst["up_original"] < 2e-5 and worst["lat_original"] < 1e-4, worst
    assert changed == len(sizes)


# ------------------------------------------------------------------------------------------------ synthetic truth
def _truth(n=6, seed=0, size=320):
    rng = np.random.default_rng(seed)
    roll = rng.uniform(-30, 30, n)
    pitch = rng.uniform(-40, 40, n)
    vfov = rng.uniform(40, 90, n)
    focal = 1.0 / (2.0 * np.tan(np.radians(vfov) / 2.0))
    ups, lats = panocam.camera_fields(focal, [size] * n, [size] * n, np.radians(pitch), np.radians(roll), [0.0] * n, [0.0] * n, device="cuda")
    return roll, pitch, vfov, torch.stack(ups), torch.stack(lats)


def _quadratic_logits(ups, lats, noise, seed):
    """sigma = 1 bin parabolas around the true bin positions (the up head's 72 bins on a circle, bin 72 far below), [n, NC, H*W]."""
    n, H, W = lats.shape
    ang = torch.rad2deg(torch.atan2(ups[..., 1], ups[..., 0])).reshape(n, 1, -1)   # decode: angle = 5 p - 180
    mu_g = torch.remainder((ang + 180.0) / 5.0, 72.0)
    mu_l = lats.reshape(n, 1, -1) + 89.5                                             # decode: lat = -90 + p + 0.5
    c72 = torch.arange(72, device="cuda", dtype=torch.float32).view(1, 72, 1)
    d = torch.remainder(c72 - mu_g + 36.0, 72.0) - 36.0
    lg = torch.cat([-0.5 * d * d, torch.full((n, 1, H * W), -1e4, device="cuda")], 1)
    c180 = torch.arange(180, device="cuda", dtype=torch.float32).view(1, 180, 1)
    ll = -0.5 * (c180 - mu_l) ** 2
    if noise:
        g = torch.Generator(device="cuda").manual_seed(seed)
        lg = lg + noise * torch.randn(lg.shape, generator=g, device="cuda")
        ll = ll + noise * torch.randn(ll.shape, generator=g, device="cuda")
    return lg.contiguous(), ll.contiguous()


def _errors(ups, lats, field_g, field_l):
    n, H, W = lats.shape
    t = torch.atan2(ups[..., 1], ups[..., 0]).reshape(n, -1)
    p = torch.atan2(field_g[:, 1], field_g[:, 0])
    e_up = torch.rad2deg(torch.remainder(p.double() - t.double() + math.pi, 2 * math.pi) - math.pi).abs()
    e_lat = (field_l[:, 0].double() - lats.reshape(n, -1).double()).abs()
    return e_up.median().item(), e_lat.median().item()


def _fit(field_g, field_l, H, W):
    res = [{"pred_gravity_original": g.view(2, H, W), "pred_latitude_original": l.view(H, W)} for g, l in zip(field_g, field_l)]
    out = calibrate.fit_camera(res)
    return np.array([[float(o["pred_roll"]), float(o["pred_pitch"]), float(o["pred_vfov"])] for o in out])


def test_synthetic_truth():
    """Through pf_op_subbin_decode: 32 input channels cannot carry a per-pixel parabola on the circle to the fused op without
    fp32 cancellation, and the fused op equals this op bit for bit on the same logits (test_fused_op_equals_logits_op_bit_for_bit)."""
    roll, pitch, vfov, ups, lats = _truth()
    n, H, W = lats.shape
    truth = np.stack([roll, pitch, vfov], 1)
    lg, ll = _quadratic_logits(ups, lats, 0.0, 0)
    arg = (_run_logits_op(lg, 1, refine=False)[0], _run_logits_op(ll, 0, refine=False)[0])
    ref = (_run_logits_op(lg, 1)[0], _run_logits_op(ll, 0)[0])
    e_arg, e_ref = _errors(ups, lats, *arg), _errors(ups, lats, *ref)
    fit_arg, fit_ref = np.abs(_fit(*arg, H, W) - truth).max(0), np.abs(_fit(*ref, H, W) - truth).max(0)
    lg_n, ll_n = _quadratic_logits(ups, lats, 0.3, 1)
    e_arg_n = _errors(ups, lats, _run_logits_op(lg_n, 1, refine=False)[0], _run_logits_op(ll_n, 0, refine=False)[0])
    e_ref_n = _errors(ups, lats, _run_logits_op(lg_n, 1)[0], _run_logits_op(ll_n, 0)[0])
    print(f"synthetic truth, {n} cameras at {H}x{W}: median |up error| / |latitude error| (deg) argmax {e_arg[0]:.4f} / {e_arg[1]:.4f}, "
          f"subbin {e_ref[0]:.2e} / {e_ref[1]:.2e}; fit max |roll, pitch, vfov error| argmax {fit_arg.round(4).tolist()}, "
          f"subbin {fit_ref.tolist()}; with N(0, 0.3) logit noise argmax {e_arg_n[0]:.4f} / {e_arg_n[1]:.4f}, "
          f"subbin {e_ref_n[0]:.4f} / {e_ref_n[1]:.4f}")
    assert 0.8 < e_arg[0] < 1.7 and 0.15 < e_arg[1] < 0.35, e_arg
    assert e_ref[0] < 1e-3 and e_ref[1] < 1e-3, e_ref
    assert fit_ref.max() < 1e-2, fit_ref
    assert e_ref_n[0] < e_arg_n[0] and e_ref_n[1] < e_arg_n[1], (e_arg_n, e_ref_n)


# ------------------------------------------------------------------------------------------------ option plumbing
def test_option_errors_and_persistence():
    with pytest.raises(ValueError):
        PerspectiveFields("Paramnet-360Cities-edina-centered", decode="subbin")
    with pytest.raises(ValueError):
        PerspectiveFields(VERSION, decode="softargmax")
    with pytest.raises(ValueError):
        PerspectiveFields(VERSION, decode=None)
    reg = U.make_model("Paramnet-360Cities-edina-centered", seed=0, device="cuda")[0]
    img = [wg.smooth_images(1, 96, 128, seed=3)[0]]
    want = reg.inference_batch(img)[0]
    with pytest.raises(_native.PfError):
        reg.set_option("subbin", 1)
    assert "subbin" not in reg._options
    got = reg.inference_batch(img)[0]
    for k, v in want.items():
        assert (v == got[k]) if isinstance(v, str) else torch.equal(v, got[k]), k

    a = _model(logits=False)
    s = U.make_model(VERSION, seed=0, device="cuda", model_kwargs=dict(logits=False, decode="subbin"))[0]
    want = s.inference_batch(img)[0]["pred_latitude"]
    assert not torch.equal(want, a.inference_batch(img)[0]["pred_latitude"])
    s.load_state_dict(a.state_dict())
    s2 = s.cpu().cuda()
    assert torch.equal(s2.inference_batch(img)[0]["pred_latitude"], want)
    assert s2._options.get("subbin") == 1
