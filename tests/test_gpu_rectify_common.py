"""GPU: rectify.upright(focal="fill_common") (csrc/rectify.cuh, rectify_setup_common_kernel): one zoom for the whole call, the
largest "fill" focal length per output height of the usable images, against the CPU oracle (tests/oracle_rectify.py)."""
import math

import numpy as np
import pytest
import torch

import oracle_rectify as orr
from oracle import weights_gen as wg
from perspectivefields_b200 import _native, calibrate, panocam, rectify

pytestmark = pytest.mark.gpu

# the fourth camera's pitch exceeds half its vfov (no zoom fills its canvas: status 1); the sixth is unusable (status 2)
CAMERAS = [(14.0, -9.0, 63.0, 0.0, 0.0), (-27.0, 22.0, 78.0, 0.05, -0.04), (4.0, 11.0, 96.0, -0.08, 0.07), (0.0, 48.0, 70.0, 0.0, 0.0),
           (-6.0, 3.0, 52.0, 0.02, 0.03), (1.0, 2.0, math.nan, 0.0, 0.0)]
SIZES = [(48, 64), (61, 45), (40, 90), (37, 53), (72, 72), (30, 40)]
OUT_SIZES = [None, (50, 70), None, (37, 53), (64, 96), None]


def _cams(params):
    return [dict(zip(rectify.CAMERA_KEYS, p)) for p in params]


def _common_fo(params, sizes, outs):
    """The oracle's common f_o: the largest "fill" F_o / H_o over the images with usable parameters."""
    f = [orr.setup(p, h, w, ho, wo, False, "fill") for p, (h, w), (ho, wo) in zip(params, sizes, outs)]
    return max(s["Fo"] / ho for s, (ho, _) in zip(f, outs) if s["status"] != 2), f


def _at(params, H, W, Ho, Wo, Fo):
    """oracle_rectify.setup's map and camera at the output focal length Fo."""
    r, e, f, F, cx, cy = orr.input_camera(params, H, W)
    R = orr.rz(-r) @ orr.rx(-e)
    K = np.array([[F, 0.0, cx], [0.0, F, cy], [0.0, 0.0, 1.0]])
    Koi = np.array([[1.0 / Fo, 0.0, -(Wo / 2.0) / Fo], [0.0, 1.0 / Fo, -(Ho / 2.0) / Fo], [0.0, 0.0, 1.0]])
    return K @ R @ Koi, [0.0, 0.0, 2.0 * math.atan(Ho / (2.0 * Fo)) * orr.R2D, 0.0, 0.0]


@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
def test_against_the_oracle(channels, mode):
    rng = np.random.default_rng(1)
    imgs = []
    for h, w in SIZES:
        base = wg.smooth_images(1, h, w, seed=int(rng.integers(1000)))[0]
        imgs.append(base if channels == 3 else np.ascontiguousarray(base[..., 1]))
    outs = [s if s is not None else im.shape[:2] for s, im in zip(OUT_SIZES, imgs)]
    out = rectify.upright([torch.from_numpy(im).cuda() for im in imgs], _cams(CAMERAS), focal="fill_common", size=OUT_SIZES, mode=mode,
                          fill=9, outputs=("mask", "map"))
    fo, fills = _common_fo(CAMERAS, SIZES, outs)
    status = out["status"].cpu().numpy()
    assert list(status) == [s["status"] for s in fills] == [0, 0, 0, 1, 0, 2]
    for i, img in enumerate(imgs):
        H, W = img.shape[:2]
        Ho, Wo = outs[i]
        got_mask = out["mask"][i].cpu().numpy()
        if status[i] == 2:
            assert not got_mask.any() and math.isnan(float(out["camera"][i]["pred_roll"]))
            assert (out["im"][i].cpu().numpy() == 9).all()
            continue
        rel = float(out["camera"][i]["pred_rel_focal"])
        assert abs(rel - fo) <= 1e-12 * fo, (i, rel, fo)
        assert fo * Ho >= fills[i]["Fo"] * (1 - 1e-15)
        M, cam = _at(CAMERAS[i], H, W, Ho, Wo, fo * Ho)
        got_cam = [float(out["camera"][i][k]) for k in ("pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy")]
        np.testing.assert_allclose(got_cam, cam, rtol=1e-12, atol=1e-12)
        u, v, valid = orr.positions(M, Ho, Wo, H, W)
        want = orr.sample(img[..., None] if img.ndim == 2 else img, u, v, valid, mode, [9] * (1 if img.ndim == 2 else 3))
        if status[i] == 0:
            assert got_mask.all(), i          # the common zoom keeps every filled canvas filled
        edge = (np.abs(u) < 1e-7) | (np.abs(u - W) < 1e-7) | (np.abs(v) < 1e-7) | (np.abs(v - H) < 1e-7)
        assert np.array_equal(got_mask[~edge], valid[~edge]), i
        both = got_mask & valid
        got_im = out["im"][i].cpu().numpy().reshape(Ho, Wo, -1).astype(np.int32)
        d = np.abs(got_im - want.astype(np.int32)).max(axis=2)
        if mode == "bilinear":
            assert d[both].max(initial=0) <= 1 and (d[both] > 0).sum() <= 1e-2 * both.sum(), i
        else:
            s = np.stack([u, v])
            tie = np.any(np.abs(s - np.round(s)) < 1e-9, axis=0)
            assert np.all(d[both & ~tie] == 0), i
        got_map = out["map"][i].cpu().numpy()
        assert np.max(np.abs(got_map[both] - np.stack([u, v], axis=2)[both]), initial=0.0) <= 1e-4


def test_one_image_is_the_fill_output():
    img = torch.from_numpy(wg.smooth_images(1, 48, 64, seed=3)[0]).cuda()
    for cam in CAMERAS[:3]:
        a = rectify.upright([img], _cams([cam]), focal="fill", outputs=("mask", "map"))
        b = rectify.upright([img], _cams([cam]), focal="fill_common", outputs=("mask", "map"))
        assert int(a["status"][0]) == int(b["status"][0]) == 0
        for k in rectify.OUTPUT_KEYS:
            x, y = float(a["camera"][0][k]), float(b["camera"][0][k])
            assert abs(x - y) <= 1e-12 * max(abs(x), 1.0), (k, x, y)
        assert torch.equal(a["mask"][0], b["mask"][0])


def test_fit_then_one_zoom_without_synchronising():
    n = 6
    rolls, pitches = [3.0 + 0.5 * t for t in range(n)], [-4.0 + 0.3 * t for t in range(n)]
    ups, lats = panocam.camera_fields([0.8] * n, [48] * n, [64] * n, [math.radians(p) for p in pitches], [math.radians(r) for r in rolls],
                                      [0.0] * n, [0.0] * n)
    res = [{"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l} for u, l in zip(ups, lats)]
    cams = calibrate.fit_camera(res, groups=[0] * n, smoothness=1.0)
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(n, 48, 64, seed=5)]
    out = rectify.upright(imgs, cams, focal="fill_common")
    assert (out["status"] == 0).all() and all(m.all() for m in out["mask"])
    f = torch.stack([c["pred_rel_focal"] for c in out["camera"]])
    assert float((f.max() - f.min()) / f.max()) < 1e-15
    each = rectify.upright(imgs, cams, focal="fill")
    fe = torch.stack([c["pred_rel_focal"] for c in each["camera"]])
    assert abs(float(f[0]) - float(fe.max())) <= 1e-12 * float(fe.max())


def test_invalid_focal():
    img = torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda")
    for bad in ("fill_Common", "common", None):
        with pytest.raises((ValueError, TypeError)):
            rectify.upright([img], _cams(CAMERAS[:1]), focal=bad)
    assert _native.PF_RECTIFY_FILL_COMMON == 4
