"""GPU: the heads' confidence maps (PerspectiveFields(confidence=True), pf_forward_confidence) against the float64 softmax maximum
of the exact logits, F.interpolate of the net-size maps, and a confidence-off model on the same inputs."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import oracle_confidence as ocf
import pf_test_util as U
from oracle import weights_gen as wg
from perspectivefields_b200 import PerspectiveFields, _native, dist

pytestmark = pytest.mark.gpu

VERSION = "PersNet-360Cities"
NC = {"gravity": 73, "latitude": 180}
CONF_KEYS = ("pred_gravity_confidence", "pred_latitude_confidence", "pred_gravity_confidence_original", "pred_latitude_confidence_original")


def _models(**kw):
    off = U.make_model(VERSION, seed=0, device="cuda", model_kwargs=dict(kw))[0]
    on = U.make_model(VERSION, seed=0, device="cuda", model_kwargs=dict(kw, confidence=True))[0]
    return off, on


def _images(sizes, seed=11):
    return [wg.smooth_images(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(sizes)]


def _logits(model, res, imgs, logits):
    """[n, NC, H, W] float64 logits of both heads: the returned ones, or the debug taps of the prediction convs."""
    if logits:
        return {k: torch.stack([r["pred_" + k] for r in res]).double() for k in NC}
    model.debug_taps(True)
    try:
        model.inference_batch(imgs)
        taps = model.read_taps()
    finally:
        model.debug_taps(False)
    h, w = model.net_size()
    return {"gravity": taps["head.raw_g"].view(len(imgs), 73, h, w).double(), "latitude": taps["head.raw_l"].view(len(imgs), 180, h, w).double()}


@pytest.mark.parametrize("logits", [True, False])
@pytest.mark.parametrize("resize", [None, (256, 384)])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_net_size_confidence_matches_softmax_max(logits, resize, precision):
    _, m = _models(logits=logits, precision=precision, resize=resize)
    imgs = _images([(240, 320), (300, 200)])
    res = m.inference_batch(imgs)
    ref = _logits(m, res, imgs, logits)
    h, w = m.net_size()
    for k in NC:
        want = torch.from_numpy(ocf.confidence(ref[k].cpu().numpy(), axis=1))
        got = torch.stack([r[f"pred_{k}_confidence"] for r in res]).double().cpu()
        assert got.shape == (len(imgs), h, w)
        assert (got - want).abs().max().item() < 2e-6, k


def test_original_maps_are_the_bilinear_resample():
    _, m = _models(logits=False)
    sizes = [(240, 320), (97, 130), (31, 3100), (50, 4), (33, 7)]     # W % 4 != 0, W > 3072, W = 4
    res = m.inference_batch(_images(sizes))
    for (h, w), r in zip(sizes, res):
        for k in ("gravity", "latitude"):
            net = r[f"pred_{k}_confidence"]
            want = Fn.interpolate(net[None, None], size=(h, w), mode="bilinear", align_corners=False)[0, 0]
            got = r[f"pred_{k}_confidence_original"]
            assert got.shape == (h, w) and got.is_contiguous()
            assert (got - want).abs().max().item() < 1e-6, (h, w, k)


@pytest.mark.parametrize("logits", [True, False])
def test_other_keys_bit_identical_and_values_in_range(logits):
    off, on = _models(logits=logits)
    imgs = _images([(240, 320), (120, 161)])
    a = off.inference_batch(imgs)
    b = on.inference_batch(imgs)
    c = on.inference_batch(imgs)
    for x, y, z in zip(a, b, c):
        assert list(y)[:len(x)] == list(x) and list(y)[len(x):] == list(CONF_KEYS)
        for k, v in x.items():
            assert (v == y[k]) if isinstance(v, str) else torch.equal(v, y[k]), k
        for k in CONF_KEYS:
            assert torch.equal(y[k], z[k]), k
            t = y[k]
            lo = 1.0 / NC["gravity" if "gravity" in k else "latitude"]
            assert torch.isfinite(t).all() and t.min().item() >= lo * (1 - 1e-6) and t.max().item() <= 1.0, k
    # the device-tensor, encoded-free forward and the float branch carry the keys too
    dev = on.inference_batch([torch.from_numpy(im).cuda() for im in imgs])
    for x, y in zip(b, dev):
        for k in CONF_KEYS:
            assert torch.equal(x[k], y[k])
    h, w = on.net_size()
    fwd = on.forward([{"image": torch.rand(3, h, w) * 255, "height": 100, "width": 150}])
    assert set(CONF_KEYS) <= set(fwd[0]) and fwd[0]["pred_latitude_confidence_original"].shape == (100, 150)


def test_survives_to_and_load_state_dict():
    off, on = _models()
    img = _images([(120, 160)])
    want = on.inference_batch(img)[0]["pred_gravity_confidence"]
    on.load_state_dict(off.state_dict())
    on = on.cpu().cuda()
    got = on.inference_batch(img)[0]
    assert torch.equal(got["pred_gravity_confidence"], want)


def test_regression_variants_and_bad_pointers_are_rejected():
    with pytest.raises(ValueError):
        PerspectiveFields("Paramnet-360Cities-edina-centered", confidence=True)
    with pytest.raises(ValueError):
        PerspectiveFields(VERSION, confidence=1)
    L = _native.lib()
    img = _images([(64, 80)])
    for version in ("Paramnet-360Cities-edina-centered", VERSION):
        m = U.make_model(version, seed=0, device="cuda")[0]
        eng = m._get_engine()
        out = eng.forward(1, [64], [80], blob=torch.from_numpy(img[0]).cuda().reshape(-1), offsets=[0])
        torch.cuda.synchronize()
        h, w = m.net_size()
        bufs = [torch.empty(h * w + 1, device="cuda"), torch.empty(h * w + 1, device="cuda"),
                torch.empty(64 * 80 + 1, device="cuda"), torch.empty(64 * 80 + 1, device="cuda")]
        good = [b.data_ptr() for b in bufs]
        bt = _native.pf_batch()
        i64p, i32p = ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int32)
        hh, ww, off = np.array([64], np.int32), np.array([80], np.int32), np.zeros(1, np.int64)
        blob = torch.from_numpy(img[0]).cuda().reshape(-1)
        bt.n, bt.images_u8, bt.image_offset = 1, blob.data_ptr(), off.ctypes.data_as(i64p)
        bt.height, bt.width = hh.ctypes.data_as(i32p), ww.ctypes.data_as(i32p)
        bt.pred_gravity, bt.pred_latitude = out["pred_gravity"].data_ptr(), out["pred_latitude"].data_ptr()
        bt.gravity_original, bt.gravity_original_offset = out["gravity_original"].data_ptr(), off.ctypes.data_as(i64p)
        bt.latitude_original, bt.latitude_original_offset = out["latitude_original"].data_ptr(), off.ctypes.data_as(i64p)
        bt.params = out["params"].data_ptr()
        ws = eng._workspace(L.pf_workspace_bytes(eng.handle, 1, 64), torch.cuda.current_stream())
        cases = [good] if version != VERSION else []
        for j in range(4):
            cases += [good[:j] + [None] + good[j + 1:], good[:j] + [good[j] + 2] + good[j + 1:]]
        before = L.pf_kernel_launch_count()
        for ptrs in cases:
            cf = _native.pf_confidence(*ptrs)
            rc = L.pf_forward_confidence(eng.handle, ctypes.byref(bt), ctypes.byref(cf), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
            assert rc == -1, (version, ptrs)
        assert L.pf_forward_confidence(eng.handle, ctypes.byref(bt), None, ws.data_ptr(), ws.numel(), 0) == -1
        assert L.pf_kernel_launch_count() == before
        if version == VERSION:   # the good pointers run
            cf = _native.pf_confidence(*good)
            assert L.pf_forward_confidence(eng.handle, ctypes.byref(bt), ctypes.byref(cf), ws.data_ptr(), ws.numel(),
                                           torch.cuda.current_stream().cuda_stream) == 0
            torch.cuda.synchronize()


def test_sharded_inference_refuses_confidence():
    _, on = _models()
    with pytest.raises(ValueError):
        dist.inference_batch_sharded(on, _images([(64, 64)]))
