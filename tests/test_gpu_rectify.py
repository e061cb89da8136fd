"""GPU: the upright warp (csrc/rectify.cuh) through rectify.upright and pf_rectify_views, against the CPU oracle
(tests/oracle_rectify.py), on inference_batch and fit_camera results, and without synchronisation."""
import ctypes
import math

import numpy as np
import pytest
import torch

import oracle_rectify as orr
import pf_test_util as U
from oracle import weights_gen as wg
from perspectivefields_b200 import _native, calibrate, rectify

pytestmark = pytest.mark.gpu

CAMERAS = [(14.0, -9.0, 63.0, 0.0, 0.0), (-27.0, 22.0, 78.0, 0.05, -0.04), (4.0, 31.0, 96.0, -0.08, 0.07), (-160.0, -12.0, 52.0, 0.02, 0.03),
           (0.0, 48.0, 70.0, 0.0, 0.0)]
SIZES = [(48, 64), (61, 45), (40, 90), (72, 72), (37, 53)]
OUT_SIZES = [None, (50, 70), None, (64, 96), (37, 53)]


def _images(channels, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for h, w in SIZES:
        base = wg.smooth_images(1, h, w, seed=int(rng.integers(1000)))[0]
        out.append(base if channels == 3 else np.ascontiguousarray(base[..., 1]))
    return out


def _cams(params):
    return [dict(zip(rectify.CAMERA_KEYS, p)) for p in params]


def _near_edge(u, v, H, W, eps=1e-7):
    return (np.abs(u) < eps) | (np.abs(u - W) < eps) | (np.abs(v) < eps) | (np.abs(v - H) < eps)


def _check(imgs, params, out, keep_pitch, focal, sizes, mode, fill):
    status = out["status"].cpu().numpy()
    for i, img in enumerate(imgs):
        want = orr.upright(img, params[i], keep_pitch, focal, sizes[i], mode, fill)
        assert status[i] == want["status"], (i, status[i], want["status"])
        cam = [float(out["camera"][i][k]) for k in ("pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy")]
        np.testing.assert_allclose(cam, want["camera"], rtol=1e-12, atol=1e-12, equal_nan=True)
        if want["status"] != 2:
            f_rel = want["Fo"] / out["im"][i].shape[0]
            assert abs(float(out["camera"][i]["pred_rel_focal"]) - f_rel) <= 1e-12 * f_rel
            assert float(out["camera"][i]["pred_vfov"]) == float(out["camera"][i]["pred_general_vfov"])
        H, W = img.shape[:2]
        got_im = out["im"][i].cpu().numpy()
        got_mask = out["mask"][i].cpu().numpy()
        got_map = out["map"][i].cpu().numpy()
        assert got_im.shape == want["im"].shape and got_mask.dtype == np.bool_
        edge = _near_edge(want["u"], want["v"], H, W) if want["status"] != 2 else np.zeros_like(want["mask"])
        assert np.array_equal(got_mask[~edge], want["mask"][~edge]), i
        both = got_mask & want["mask"]
        d = np.abs(got_im.astype(np.int32) - want["im"].astype(np.int32))
        d = d if d.ndim == 2 else d.max(axis=2)
        if mode == "bilinear":
            assert d[both].max(initial=0) <= 1 and (d[both] > 0).mean() < 1e-2, (i, d[both].max(initial=0), (d[both] > 0).mean())
        else:
            # a nearest tap flips only where an index + 1/2 lies within rounding of an integer
            s = np.stack([want["u"], want["v"]])
            tie = np.any(np.abs(s - np.round(s)) < 1e-9, axis=0)
            assert np.all(d[both & ~tie] == 0), i
        neither = ~got_mask & ~want["mask"]
        fv = np.asarray([fill] * (1 if img.ndim == 2 else 3) if np.isscalar(fill) else fill, np.uint8)
        g3 = got_im.reshape(got_im.shape[0], got_im.shape[1], -1)
        assert np.all(g3[neither] == fv), i
        assert np.isnan(got_map[~got_mask]).all()
        assert np.max(np.abs(got_map[both] - want["map"][both]), initial=0.0) <= 1e-4


@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
@pytest.mark.parametrize("focal", ["same", "fill", 55.0])
@pytest.mark.parametrize("keep_pitch", [False, True])
def test_against_the_oracle(channels, mode, focal, keep_pitch):
    imgs = _images(channels)
    fill = 17 if channels == 1 else (5, 200, 90)
    dev_imgs = [torch.from_numpy(im).cuda() for im in imgs]
    out = rectify.upright(dev_imgs, _cams(CAMERAS), keep_pitch=keep_pitch, focal=focal, size=OUT_SIZES, mode=mode, fill=fill,
                          outputs=("mask", "map"))
    sizes = [s if s is not None else im.shape[:2] for s, im in zip(OUT_SIZES, imgs)]
    _check(imgs, CAMERAS, out, keep_pitch, focal, sizes, mode, fill)
    if focal == "fill" and not keep_pitch:
        assert int(out["status"][4]) == 1      # pitch 48 > vfov / 2: no zoom fills the canvas
    # host images and numbers give the same bytes
    host = rectify.upright(imgs, _cams(CAMERAS), keep_pitch=keep_pitch, focal=focal, size=OUT_SIZES, mode=mode, fill=fill,
                           outputs=("mask", "map"))
    for a, b in zip(out["im"] + out["mask"], host["im"] + host["mask"]):
        assert torch.equal(a, b)


def test_status_2_for_unusable_parameters():
    bad_fit = calibrate.fit_camera([{"pred_gravity_original": torch.full((2, 16, 16), math.nan, device="cuda"),
                                     "pred_latitude_original": torch.full((16, 16), math.nan, device="cuda")}])[0]
    assert int(bad_fit["fit_status"]) == 2
    imgs = [torch.full((20, 30, 3), 99, dtype=torch.uint8, device="cuda") for _ in range(4)]
    cams = [bad_fit, dict(zip(rectify.CAMERA_KEYS, (0.0, 0.0, -10.0, 0.0, 0.0))), dict(zip(rectify.CAMERA_KEYS, (math.inf, 0.0, 60.0, 0.0, 0.0))),
            dict(zip(rectify.CAMERA_KEYS, (5.0, 3.0, 60.0, 0.0, 0.0)))]
    out = rectify.upright(imgs, cams, fill=(1, 2, 3), outputs=("mask", "map"))
    assert out["status"].tolist() == [2, 2, 2, 0]
    for i in range(3):
        assert (out["im"][i] == torch.tensor([1, 2, 3], dtype=torch.uint8, device="cuda")).all()
        assert not out["mask"][i].any() and torch.isnan(out["map"][i]).all()
        assert all(math.isnan(float(v)) for v in out["camera"][i].values())
    assert out["mask"][3].float().mean() > 0.5


def test_repeated_calls_are_bit_identical_and_do_not_synchronise():
    imgs = [torch.from_numpy(im).cuda() for im in _images(3, seed=4)]
    cams = [{k: torch.tensor(v, dtype=torch.float64, device="cuda") for k, v in c.items()} for c in _cams(CAMERAS)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = rectify.upright(imgs, cams, focal="fill", outputs=("mask", "map"))
        b = rectify.upright(imgs, cams, focal="fill", outputs=("mask", "map"))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in ("im", "mask", "map"):
        for x, y in zip(a[k], b[k]):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    assert torch.equal(a["status"], b["status"])
    for x, y in zip(a["camera"], b["camera"]):
        assert all(torch.equal(x[k], y[k]) for k in x)
    for t in a["im"]:
        assert t.data_ptr() % 16 == 0


def test_inference_results_round_trip():
    version = "Paramnet-360Cities-edina-centered"
    model = U.make_model(version, seed=0, device="cuda")[0]
    host = wg.smooth_images(3, 96, 128, seed=2) + wg.smooth_images(1, 80, 60, seed=3)
    imgs = [torch.from_numpy(im).cuda() for im in host]
    results = model.inference_batch(imgs)
    out = rectify.upright(imgs, results, outputs=("mask", "map"))
    params = [[float(r[k]) for k in rectify.CAMERA_KEYS] for r in results]
    _check(host, params, out, False, "same", [None] * len(host), "bilinear", 0)
    for k in rectify.OUTPUT_KEYS:
        assert out["camera"][0][k].dtype == torch.float64 and out["camera"][0][k].dim() == 0
    fitted = calibrate.fit_camera(results)
    out2 = rectify.upright(imgs, fitted, focal="fill")
    assert out2["status"].shape == (len(imgs),)
    again = model.inference_batch(out["im"])
    assert len(again) == len(imgs) and all("pred_roll" in r for r in again)
    uncentred = U.make_model("Paramnet-360Cities-edina-uncentered", seed=0, device="cuda")[0].inference_batch(imgs)
    out3 = rectify.upright(imgs, uncentred, keep_pitch=True)
    params3 = [[float(r[k]) for k in rectify.CAMERA_KEYS] for r in uncentred]
    for i in range(len(imgs)):
        want = orr.upright(host[i], params3[i], True)
        assert int(out3["status"][i]) == want["status"]


def test_invalid_arguments_raise_before_any_launch():
    L = _native.lib()
    img = torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda")
    cam = dict(zip(rectify.CAMERA_KEYS, (0.0, 0.0, 60.0, 0.0, 0.0)))
    before = L.pf_kernel_launch_count()
    cases = [(ValueError, dict(focal="zoom")), (ValueError, dict(focal=180.0)), (ValueError, dict(focal=True)), (ValueError, dict(mode="cubic")),
             (ValueError, dict(outputs=("depth",))), (ValueError, dict(fill=256)), (ValueError, dict(fill=(1, 2))), (ValueError, dict(fill=1.5)),
             (TypeError, dict(keep_pitch=1)), (ValueError, dict(size=(0, 4))), (ValueError, dict(size=[(4, 4), (4, 4)]))]
    for exc, kw in cases:
        with pytest.raises(exc):
            rectify.upright([img], [cam], **kw)
    with pytest.raises(ValueError):
        rectify.upright([], [])
    with pytest.raises(ValueError):
        rectify.upright([img], [cam, cam])
    with pytest.raises(ValueError):
        rectify.upright([img], [{"pred_roll": 0.0}])
    with pytest.raises(TypeError):
        rectify.upright([img, np.zeros((8, 8, 3), np.uint8)], [cam, cam])
    with pytest.raises(TypeError):
        rectify.upright([img, img[..., 0].contiguous()], [cam, cam])
    with pytest.raises(TypeError):
        rectify.upright([img.float()], [cam])
    with pytest.raises(TypeError):
        rectify.upright([img], [dict(cam, pred_roll="0")])
    # the C ABI checks every argument before its first launch
    d = (_native.pf_rectify_image * 1)()
    d[0].height = d[0].width = d[0].out_height = d[0].out_width = 8
    d[0].mask_offset = d[0].map_offset = -1
    need = L.pf_rectify_workspace(d, 1)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(8 * 8 * 3, dtype=torch.uint8, device="cuda")
    par = torch.zeros((1, 5), dtype=torch.float64, device="cuda")
    cam_o = torch.empty((1, 5), dtype=torch.float64, device="cuda")
    st = torch.empty(1, dtype=torch.int32, device="cuda")
    fill = (ctypes.c_int32 * 3)(0, 0, 0)

    def call(**kw):
        a = dict(channels=3, keep_pitch=0, focal_mode=0, vfov=0.0, sampler=0, ws_bytes=need, n=1, mask=None)
        a.update(kw)
        return L.pf_rectify_views(0, d, a["n"], img.data_ptr(), out.data_ptr(), a["mask"], None, a["channels"], par.data_ptr(), a["keep_pitch"],
                                  a["focal_mode"], a["vfov"], a["sampler"], fill, cam_o.data_ptr(), st.data_ptr(), ws.data_ptr(),
                                  a["ws_bytes"], torch.cuda.current_stream().cuda_stream)

    for kw in (dict(channels=2), dict(keep_pitch=2), dict(focal_mode=3), dict(focal_mode=1, vfov=0.0), dict(sampler=2),
               dict(ws_bytes=need - 1), dict(n=0)):
        assert call(**kw) < 0, kw
    d[0].mask_offset = 0
    assert call() < 0          # a mask offset without mask_base
    d[0].mask_offset = -1
    fill[1] = 256
    assert call() < 0
    assert L.pf_kernel_launch_count() == before
