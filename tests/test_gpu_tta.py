"""GPU: flip test-time augmentation (PerspectiveFields(tta="flip"), engine option "flip_tta", pf_op_flip_merge_reg /
pf_op_flip_pred) against the float32 oracle tests/oracle_tta.py, its exact mirror-equivariance, the mirrored pre-process slots, the
merge kernels one launch at a time, and the workspace and option plumbing."""
import ctypes
import gc

import numpy as np
import pytest
import torch

import oracle_confidence as ocf
import oracle_resize as ro
import oracle_subbin as osb
import oracle_tta as ot
import pf_test_util as U
from bf16_emulation import ANGLE_KEYS, DEG_BOUND, REL_BOUND, error_table
from oracle import model as om
from oracle import weights_gen as wg
from perspectivefields_b200 import PerspectiveFields, _native

pytestmark = pytest.mark.gpu

TOL = 1e-3                   # fp32 against the oracle, relative (error_table's metric)
ANGLE_TOL = 0.1              # ParamNet angles at fp32, degrees
P360 = "PersNet-360Cities"
REGRESSION = ["Paramnet-360Cities-edina-centered", "Paramnet-360Cities-edina-uncentered", "PersNet_Paramnet-GSV-uncentered",
              "PersNet_Paramnet-GSV-centered"]
SIZES = [(240, 333), (200, 161)]      # down- and up-sampling, odd widths


def _images(sizes=SIZES, seed=40):
    return [wg.smooth_images(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(sizes)]


# The suite runs in one process, and other modules keep their models on the device: this module keeps only its most recent
# model, drops the engines (weights, workspace) of the ones before it, and releases everything when it ends.
_cache = {}


def _release():
    for m, _ in _cache.values():
        m._drop_engine()
    _cache.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _model(version, **kw):
    key = (version, tuple(sorted(kw.items())))
    if key not in _cache:
        _release()
        _cache[key] = U.make_model(version, seed=0, device="cuda", model_kwargs=dict(kw))
    return _cache[key]


@pytest.fixture(scope="module", autouse=True)
def _release_at_the_end():
    yield
    _release()


# ------------------------------------------------------------------------------------------------ op level
def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


@pytest.mark.parametrize("hw", [(5, 7), (16, 24)])
def test_regression_merge_op_matches_the_restatement(hw):
    H, W = hw
    n = 3
    g = torch.Generator().manual_seed(H * W)
    g2 = torch.nn.functional.normalize(torch.randn(2 * n, 2, H * W, generator=g), dim=1)
    l2 = torch.rand(2 * n, 1, H * W, generator=g) * 2 - 1
    go, lo = _nan(n + 1, 2, H * W), _nan(n + 1, 1, H * W)          # NaN sentinels after the last image
    dg, dl = g2.cuda(), l2.cuda()
    _native.check(_native.lib().pf_op_flip_merge_reg(dg.data_ptr(), dl.data_ptr(), go.data_ptr(), lo.data_ptr(), n, H, W, U.stream_ptr()))
    torch.cuda.synchronize()
    gn, ln_ = g2.view(2 * n, 2, H, W).numpy(), l2.view(2 * n, H, W).numpy()
    want_g = ot.merge_up(gn[:n], gn[n:]).reshape(n, 2, H * W)
    want_l = ot.merge_lat(ln_[:n], ln_[n:]).reshape(n, 1, H * W)
    assert (go[:n].cpu() - torch.from_numpy(want_g)).abs().max().item() <= 2e-7
    assert (lo[:n].cpu() - torch.from_numpy(want_l)).abs().max().item() <= 2e-7
    assert torch.isnan(go[n]).all() and torch.isnan(lo[n]).all()


def _flip_pred(feat, coff, w, b, n, H, W, is_gravity, decode, subbin=False, conf=False):
    nc = w.shape[0]
    out = _nan(n + 1, (2 if is_gravity else 1) if decode else nc, H * W)
    cf = _nan(n + 1, H * W) if conf else None
    _native.check(_native.lib().pf_op_flip_pred(feat.data_ptr(), feat.shape[1], coff, w.data_ptr(), b.data_ptr(), out.data_ptr(),
                                                cf.data_ptr() if conf else None, n, H, W, nc, int(is_gravity), int(decode), int(subbin),
                                                U.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.isnan(out[n]).all() and (not conf or torch.isnan(cf[n]).all())
    return out[:n], (cf[:n] if conf else None)


@pytest.mark.parametrize("is_gravity", [1, 0])
@pytest.mark.parametrize("hw", [(5, 7), (12, 20)])
def test_classification_merge_op(is_gravity, hw):
    """Logits form against the restatement on pf_op_pred_tail's logits of both slots (the same fma chain: equal bit for bit), then
    every decode_only form against the decode kernels on those merged logits (equal bit for bit, confidence included)."""
    H, W = hw
    n, HW = 2, hw[0] * hw[1]
    nc = 73 if is_gravity else 180
    coff = 0 if is_gravity else 32
    g = torch.Generator().manual_seed(7 + nc + HW)
    feat = torch.relu(torch.randn(2 * n * HW, 64, generator=g)).cuda()
    w, b = (torch.randn(nc, 32, generator=g) * 0.3).cuda(), (torch.randn(nc, generator=g) * 0.1).cuda()
    L = _native.lib()
    raw = torch.empty(2 * n, nc, HW, device="cuda")
    _native.check(L.pf_op_pred_tail(feat.data_ptr(), 64, coff, w.data_ptr(), b.data_ptr(), raw.data_ptr(), 2 * n, HW, nc, 0, U.stream_ptr()))
    torch.cuda.synchronize()
    r = raw.cpu().numpy().reshape(2 * n, nc, H, W)
    want = torch.from_numpy(ot.merge_logits(r[:n], r[n:], bool(is_gravity)).reshape(n, nc, HW))
    logits, _ = _flip_pred(feat, coff, w, b, n, H, W, is_gravity, decode=False)
    assert torch.equal(logits.cpu(), want)
    for subbin in (False, True):
        ref = torch.empty(n, 2 if is_gravity else 1, HW, device="cuda")
        rc = torch.empty(n, HW, device="cuda")
        _native.check(L.pf_op_subbin_decode(logits.data_ptr(), ref.data_ptr(), rc.data_ptr(), n, HW, nc, is_gravity, U.stream_ptr()) if subbin else
                      L.pf_op_argmax_decode(logits.data_ptr(), ref.data_ptr(), n, HW, nc, is_gravity, U.stream_ptr()))
        torch.cuda.synchronize()
        for conf in (False, True):
            field, cf = _flip_pred(feat, coff, w, b, n, H, W, is_gravity, decode=True, subbin=subbin, conf=conf)
            assert torch.equal(field, ref), (subbin, conf)
            if conf:
                want_c = torch.from_numpy(ocf.confidence(want.numpy(), axis=1)).float()
                assert (cf.cpu() / want_c - 1).abs().max().item() < 2e-5
                if subbin:
                    assert torch.equal(cf, rc)


def test_op_argument_checks():
    L = _native.lib()
    x = torch.zeros(4 * 64 * 35, device="cuda")
    p = x.data_ptr()
    before = L.pf_kernel_launch_count()
    assert L.pf_op_flip_merge_reg(None, p, p, p, 1, 5, 7, None) == -1
    assert L.pf_op_flip_merge_reg(p, p, p, p, 0, 5, 7, None) == -1
    assert L.pf_op_flip_pred(p, 64, 2, p, p, p, None, 1, 5, 7, 73, 1, 0, 0, None) == -1        # coff % 4
    assert L.pf_op_flip_pred(p, 64, 0, p, p, p, None, 1, 5, 7, 257, 0, 0, 0, None) == -1       # NC > 256
    assert L.pf_op_flip_pred(p, 64, 0, p, p, p, None, 1, 5, 7, 72, 1, 0, 0, None) == -1        # odd number of up bins
    assert L.pf_op_flip_pred(p, 64, 0, p, p, p, p, 1, 5, 7, 73, 1, 0, 0, None) == -1           # conf without decode
    assert L.pf_op_flip_pred(p, 64, 0, p, p, p, p + 2, 1, 5, 7, 73, 1, 1, 0, None) == -1       # unaligned conf
    assert L.pf_kernel_launch_count() == before


# ------------------------------------------------------------------------------------------------ end to end against the oracle
def _stack(res, key):
    return torch.stack([r[key] for r in res]).float().cpu()


@pytest.mark.parametrize("version", REGRESSION)
def test_regression_variants_match_the_oracle(version):
    m, sd = _model(version, tta="flip")
    imgs = _images()
    out = m.inference_batch(imgs)
    ora = ot.inference_batch(sd, version, imgs)
    table = error_table(out, ora)
    print(version, {k: round(v, 6) for k, v in table.items()})
    assert {"pred_gravity", "pred_latitude", "pred_gravity_original", "pred_latitude_original", "pred_roll"} <= set(table)
    for k, e in table.items():
        assert e < (ANGLE_TOL if k in ANGLE_KEYS else TOL), (version, k, e)


def _decoded_from_logits(lg, ll, h, w, net_hw, decode):
    """The decode and post-process of oracle_tta on given merged logits ([NC, H, W] each)."""
    if decode == "subbin":
        up, lat = osb.decode_gravity(lg.numpy(), axis=0), osb.decode_latitude(ll.numpy(), axis=0)[None]
        return (torch.from_numpy(up), torch.from_numpy(lat), osb.postprocess_gravity(lg.numpy(), h, w, net_hw),
                osb.postprocess_latitude(ll.numpy(), h, w, net_hw))
    cfg = {"gravity": "classification", "latitude": "classification", "gravity_classes": 73, "latitude_classes": 180}
    return (om.decode_bin(lg.argmax(0), 73), om.decode_bin_latitude(ll.argmax(0), 180)[None], ro.postprocess_gravity(cfg, lg, h, w, net_hw),
            ro.postprocess_latitude(cfg, ll, h, w, net_hw))


_oracle_cache = {}


def _oracle_logits(sd, imgs, net_hw):
    key = (len(imgs), tuple(net_hw))
    if key not in _oracle_cache:
        _oracle_cache[key] = ot.inference_batch(sd, P360, imgs, net_hw)
    return _oracle_cache[key]


_CLS_CASES = [(lg, cf, dec, None) for lg in (True, False) for cf in (False, True) for dec in ("argmax", "subbin")] + \
    [(True, False, "argmax", (320, 448)), (False, True, "subbin", (320, 448))]     # a rectangular working size


@pytest.mark.parametrize("logits,confidence,decode,resize", _CLS_CASES)
def test_classification_variant_matches_the_oracle(logits, confidence, decode, resize):
    """The merged logits against the oracle's at 1e-3; the decode, confidence and post-process against the oracle's on the
    engine's own merged logits (argmax is discontinuous: the decode of the oracle's logits differs where two logits are within
    the logit error); decode_only against the logits path, bit for bit."""
    kw = dict(tta="flip", decode=decode, confidence=confidence, resize=resize)
    lm, sd = _model(P360, **kw)
    sizes = SIZES if resize is None else SIZES[:1]      # (the larger working size: one image keeps the device memory down)
    imgs = _images(sizes)
    ref = lm.inference_batch(imgs)       # logits=True
    net_hw = lm.net_size()
    ora = _oracle_logits(sd, imgs, net_hw)
    for k in ("pred_gravity", "pred_latitude"):
        assert U.rel_err(_stack(ref, k), _stack(ora, k)) < TOL, k
    out = ref if logits else _model(P360, logits=False, **kw)[0].inference_batch(imgs)
    for i, ((h, w), r, o) in enumerate(zip(sizes, ref, out)):
        assert list(o) == list(ref[i]) or not logits
        up, lat, go, lo = _decoded_from_logits(r["pred_gravity"].cpu(), r["pred_latitude"].cpu(), h, w, net_hw, decode)
        if not logits:
            assert (o["pred_gravity"].cpu() - up).abs().max().item() < 2e-6
            assert (o["pred_latitude"].cpu() - lat).abs().max().item() < 1e-4
            for k in ("pred_gravity_original", "pred_latitude_original"):
                assert torch.equal(o[k], r[k]), k
        scale = torch.tensor([[w / net_hw[1]], [h / net_hw[0]]]).unsqueeze(-1)
        ok = ro.pf_postprocess(torch.as_tensor(up, dtype=torch.float32) * scale, h, w, net_hw).norm(dim=0) >= 0.1 * min(scale.min().item(), 1.0)
        assert (o["pred_gravity_original"].cpu() - go).abs().amax(0)[ok].max().item() < 2e-5
        assert (o["pred_latitude_original"].cpu() - lo).abs().max().item() < 1e-4
        if confidence:
            for k, lg in (("gravity", r["pred_gravity"]), ("latitude", r["pred_latitude"])):
                want = torch.from_numpy(ocf.confidence(lg.cpu().numpy())).float()
                assert (o[f"pred_{k}_confidence"].cpu() / want - 1).abs().max().item() < 2e-5, k
                if not logits:
                    assert torch.equal(o[f"pred_{k}_confidence"], ref[i][f"pred_{k}_confidence"]), k


@pytest.mark.parametrize("version", ["Paramnet-360Cities-edina-centered", P360])
def test_bf16_within_the_emulated_bounds(version):
    m, sd = _model(version, tta="flip", precision="bf16")
    imgs = _images()
    out = m.inference_batch(imgs)
    ora = ot.inference_batch(sd, version, imgs)
    table = error_table(out, ora, classification=version == P360)
    print(version, "bf16", {k: round(v, 4) for k, v in table.items()})
    for k, e in table.items():
        assert e < (DEG_BOUND if k in ANGLE_KEYS else REL_BOUND), (version, k, e)


# ------------------------------------------------------------------------------------------------ exact mirror-equivariance
UP_CONF_REL = 1e-5       # the up head's confidence sums its 73 exponentials in class order, which the class map permutes
DECODED_UP, DECODED_LAT = 2e-6, 1e-4         # decoded fields: cos / sin of mirrored bin angles, rounded once each
ORIG_UP, ORIG_LAT = 1e-4, 1e-3               # post-process: the mirrored sample positions round differently
# decoded (piecewise constant) up fields: a sample position's rounding (ulp of the source column, 3e-5 at 320) times the largest
# step between neighbouring decoded vectors (2), over the shortest blend kept (0.1), is 6e-4
ORIG_UP_CLS = 1e-3
# and for decoded latitudes, whose neighbouring columns can differ by up to 180 degrees (synthetic weights): 5.4e-3 degrees
ORIG_LAT_CLS = 1e-2


def _mirror(t):
    return t.flip(-1)


def _blend_ok(lg, decode, h, w, net_hw):
    """Pixels of the [h, w] output whose bilinear blend of decoded up vectors is at least 0.1 long: F.normalize of a near-zero blend
    (bin 72's zero vector, or near-opposite neighbours) has a direction set by the last rounding (as in tests/test_gpu_subbin.py)."""
    up = osb.decode_gravity(lg.numpy(), axis=0) if decode == "subbin" else om.decode_bin(lg.argmax(0), 73).numpy()
    scale = torch.tensor([[w / net_hw[1]], [h / net_hw[0]]]).unsqueeze(-1)
    blend = ro.pf_postprocess(torch.as_tensor(up, dtype=torch.float32) * scale, h, w, net_hw).norm(dim=0)
    return blend >= 0.1 * min(scale.min().item(), 1.0)


def _tie_free(lg):
    """Pixels whose top two merged logits differ: an exact tie resolves to the first index, which the class map can reorder."""
    top = lg.topk(2, dim=0).values
    return top[0] != top[1]


@pytest.mark.parametrize("version,kw", [(v, {}) for v in REGRESSION] + [(P360, {}), (P360, dict(logits=False, confidence=True, decode="subbin"))])
def test_mirrored_image_gives_the_mirrored_fields(version, kw):
    m, _ = _model(version, tta="flip", **kw)
    imgs = _images([(240, 333), (320, 320)], seed=60)
    flipped = [np.ascontiguousarray(im[:, ::-1]) for im in imgs]
    a, b = m.inference_batch(imgs), m.inference_batch(flipped)
    P = torch.from_numpy(ot.class_map(73, True))
    cls = version == P360
    # the classification decodes agree where no two merged logits of a pixel tie (the logits of the same images decide)
    lgs = _model(P360, tta="flip", decode=kw.get("decode", "argmax"))[0].inference_batch(imgs) if cls else None
    for i, (x, y) in enumerate(zip(a, b)):
        assert list(x) == list(y)
        g, gf = x["pred_gravity"].cpu(), y["pred_gravity"].cpu()
        ties = False
        if cls:
            ok_g, ok_l = _tie_free(lgs[i]["pred_gravity"].cpu()), _tie_free(lgs[i]["pred_latitude"].cpu())
            ties = not (ok_g.all() and ok_l.all())
            assert ok_g.float().mean() > 0.999 and ok_l.float().mean() > 0.999
        if not cls:
            assert torch.equal(gf[0], -_mirror(g[0])) and torch.equal(gf[1], _mirror(g[1]))
            assert torch.equal(y["pred_latitude"].cpu(), _mirror(x["pred_latitude"].cpu()))
        elif not kw:    # logits: classes mapped, columns mirrored
            assert torch.equal(gf, _mirror(g)[P])
            assert torch.equal(y["pred_latitude"].cpu(), _mirror(x["pred_latitude"].cpu()))
        else:           # decode_only: the decoded fields and the confidence maps
            mg, ml = _mirror(ok_g), _mirror(ok_l)
            assert (gf[0] + _mirror(g[0]))[mg].abs().max().item() < DECODED_UP and (gf[1] - _mirror(g[1]))[mg].abs().max().item() < DECODED_UP
            assert (y["pred_latitude"].cpu()[0] - _mirror(x["pred_latitude"].cpu()[0]))[ml].abs().max().item() < DECODED_LAT
            assert torch.equal(y["pred_latitude_confidence"].cpu(), _mirror(x["pred_latitude_confidence"].cpu()))
            cg, cgf = x["pred_gravity_confidence"].cpu(), y["pred_gravity_confidence"].cpu()
            assert (cgf / _mirror(cg) - 1).abs().max().item() < UP_CONF_REL
        if ties:
            print(f"image {i}: a tie between two merged logits; the _original fields are not compared")
            continue
        go, gof = x["pred_gravity_original"].cpu(), y["pred_gravity_original"].cpu()
        ok = torch.ones(go.shape[1:], dtype=torch.bool)
        if cls:
            ok = _blend_ok(lgs[i]["pred_gravity"].cpu(), kw.get("decode", "argmax"), go.shape[1], go.shape[2], m.net_size())
            assert ok.float().mean() > 0.95
        mo = _mirror(ok)
        bound = ORIG_UP_CLS if cls else ORIG_UP
        assert (gof[0] + _mirror(go[0]))[mo].abs().max().item() < bound and (gof[1] - _mirror(go[1]))[mo].abs().max().item() < bound
        lo, lof = x["pred_latitude_original"].cpu(), y["pred_latitude_original"].cpu()
        far = lo.abs() < 75           # asin amplifies the rounding near the poles of the regression heads
        assert (lof - _mirror(lo))[_mirror(far)].abs().max().item() < (ORIG_LAT_CLS if cls else ORIG_LAT)


# ------------------------------------------------------------------------------------------------ the mirrored pre-process
def test_mirror_slots_of_the_pre_process():
    # (a small working size: the debug taps keep every intermediate of the forward)
    m, _ = _model("Paramnet-360Cities-edina-centered", tta="flip", resize=(64, 96))
    sizes = [(240, 333), (50, 41), (481, 640)]          # down- and up-sampling, odd widths
    imgs = _images(sizes, seed=80)
    m.debug_taps(True)
    try:
        m.inference_batch(imgs)
        pre = m.read_taps()["pre"]
        h, w = m.net_size()
        pre = pre.view(2 * len(imgs), h, w, 4)
        L = _native.lib()
        mean = (ctypes.c_float * 3)(*m.pixel_mean.flatten().tolist())
        std = (ctypes.c_float * 3)(*m.pixel_std.flatten().tolist())
        for i, im in enumerate(imgs):
            for k, src in ((i, im), (len(imgs) + i, np.ascontiguousarray(im[:, ::-1]))):
                d = torch.from_numpy(src).cuda()
                y = torch.empty(h, w, 4, device="cuda")
                _native.check(L.pf_op_preprocess_sized(d.data_ptr(), src.shape[0], src.shape[1], h, w, mean, std, y.data_ptr(), U.stream_ptr()))
                torch.cuda.synchronize()
                assert torch.equal(pre[k], y), (i, k)
        # the float forward() path: the given [3, H, W] image mirrored
        f = [{"image": ro.preprocess(im, (h, w)), "height": im.shape[0], "width": im.shape[1]} for im in imgs[:2]]
        m.forward(f)
        pre = m.read_taps()["pre"].view(4, h, w, 4)
        for i in range(2):
            assert torch.equal(pre[2 + i], pre[i].flip(1))
    finally:
        m.debug_taps(False)


# ------------------------------------------------------------------------------------------------ equal paths, workspace, options
def _same(a, b):
    for x, y in zip(a, b):
        assert list(x) == list(y)
        for k, v in x.items():
            assert (v == y[k]) if isinstance(v, str) else torch.equal(v.cpu(), y[k].cpu()), k


def test_input_paths_agree():
    m, _ = _model(P360, tta="flip", confidence=True)
    imgs = _images()
    want = m.inference_batch(imgs)
    _same(m.inference_batch([torch.from_numpy(im).cuda() for im in imgs]), want)
    _same([m.inference(imgs[1])], want[1:])
    cv2 = pytest.importorskip("cv2")
    jpegs = [cv2.imencode(".jpg", im)[1].tobytes() for im in imgs]
    blob, offs, hs, ws = m.decode_batch(jpegs)
    decoded = [blob[o:o + h * w * 3].view(h, w, 3) for o, h, w in zip(offs.tolist(), hs, ws)]
    _same(m.inference_batch_encoded(jpegs), m.inference_batch(decoded))


def test_workspace_follows_the_option():
    m, _ = _model("Paramnet-360Cities-edina-centered")
    eng = m._get_engine()
    L = eng.L
    off = L.pf_workspace_bytes(eng.handle, 4, 320)
    _native.check(L.pf_set_option(eng.handle, b"flip_tta", 1))
    try:
        on = L.pf_workspace_bytes(eng.handle, 4, 320)
        assert on > off
        imgs = _images()
        n = len(imgs)
        h = np.array([im.shape[0] for im in imgs], np.int32)
        w = np.array([im.shape[1] for im in imgs], np.int32)
        need = L.pf_workspace_bytes(eng.handle, n, int(h.max())) - 4096     # the dry run's peak (the figure adds 4096 bytes of slack)
        blob = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).cuda()
        offs = np.array([0, imgs[0].size], np.int64)
        hw = (h.astype(np.int64) * w)
        outs = [torch.empty(k, device="cuda") for k in (n * 2 * 320 * 320, n * 320 * 320, int(2 * hw.sum()), int(hw.sum()), n * 8)]
        bt = _native.pf_batch()
        bt.n = n
        i64p, i32p = ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int32)
        g_off, l_off = np.array([0, 2 * hw[0]], np.int64), np.array([0, hw[0]], np.int64)
        bt.images_u8, bt.image_offset = blob.data_ptr(), offs.ctypes.data_as(i64p)
        bt.height, bt.width = h.ctypes.data_as(i32p), w.ctypes.data_as(i32p)
        bt.pred_gravity, bt.pred_latitude = outs[0].data_ptr(), outs[1].data_ptr()
        bt.gravity_original, bt.gravity_original_offset = outs[2].data_ptr(), g_off.ctypes.data_as(i64p)
        bt.latitude_original, bt.latitude_original_offset = outs[3].data_ptr(), l_off.ctypes.data_as(i64p)
        bt.params = outs[4].data_ptr()
        ws = torch.empty(need + 4096, dtype=torch.uint8, device="cuda")
        before = L.pf_kernel_launch_count()
        assert L.pf_forward(eng.handle, ctypes.byref(bt), ws.data_ptr(), need - 1, None) < 0
        assert L.pf_kernel_launch_count() == before
        _native.check(L.pf_forward(eng.handle, ctypes.byref(bt), ws.data_ptr(), need, None))
        torch.cuda.synchronize()
        assert torch.isfinite(outs[0]).all()
    finally:
        _native.check(L.pf_set_option(eng.handle, b"flip_tta", 0))
    assert L.pf_workspace_bytes(eng.handle, 4, 320) == off


def test_option_values_and_persistence():
    for bad in ("rotate", True, 1, "FLIP"):
        with pytest.raises(ValueError):
            PerspectiveFields(P360, tta=bad)
    img = _images([(200, 300)], seed=90)
    plain, _ = _model("PersNet_Paramnet-GSV-centered")
    base, state = plain.inference_batch(img)[0]["pred_gravity"], plain.state_dict()
    m, _ = _model("PersNet_Paramnet-GSV-centered", tta="flip")
    want = m.inference_batch(img)[0]
    assert not torch.equal(want["pred_gravity"], base)
    m2 = m.cpu().cuda()
    m2.load_state_dict(state)
    assert m2._options.get("flip_tta") == 1
    _same([m2.inference_batch(img)[0]], [want])
