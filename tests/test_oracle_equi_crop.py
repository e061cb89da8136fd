"""CPU: the oracle's pinhole crop (tests/oracle_equi.py, the rule of DESIGN.md section 1) against golden outputs of the unmodified
reference (tests/golden/equi.npz, make_golden_equi.py): the wrapper's arithmetic, dtype handling and get_image's ToTensor /
ToPILImage chain; the horizon / vertical-vanishing-point helpers of perspectivefields_b200.panocam; the rule's geometry against
the ground truth the reference pairs with the crop (get_lat / get_up) and against crop_distortion (tests/oracle_pano.py); and
the argument checks of the Python API, which run before any GPU work."""
import ctypes
import math
import os
import warnings

import numpy as np
import pytest

import oracle_equi as oe
import oracle_pano as op
from perspectivefields_b200 import panocam as pc

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "equi.npz"))
PANO = op.make_panorama(*[int(x) for x in GOLD["pano"]])
CASES = [tuple(c) for c in GOLD["crop_cases"]]
IMAGE_CASES = [tuple(c) for c in GOLD["image_cases"]]
VARIANTS = {"u8": (PANO, "bilinear"), "gray": (np.ascontiguousarray(PANO[:, :, 1]), "bilinear"),
            "f32": ((PANO.astype(np.float32) * np.float32(1.0 / 64)) - np.float32(1.5), "bilinear"), "near": (PANO, "nearest")}


def _view(c):
    vfov, w, h, az, el, roll, ar = c
    return vfov, int(w), int(h), az, el, roll, ar


def _strict(sample):
    return np.abs(sample - np.round(sample)) >= 1e-3


@pytest.mark.parametrize("i", range(len(CASES)))
def test_oracle_matches_reference_crop_equi(i):
    view = _view(CASES[i])
    fov_x, rot = oe.wrapper_args(*view)
    assert [fov_x, rot["roll"], rot["pitch"], rot["yaw"]] == GOLD["wrapper"][i].tolist()
    for key, (img, mode) in VARIANTS.items():
        o = oe.crop_equi_full(img, *view, mode=mode)
        g = GOLD[f"{key}{i}"]
        assert g.dtype == img.dtype, key
        got = o["im"].reshape(g.shape)             # the reference returns a 2-D panorama's crop as [H, W, 1]
        if img.dtype == np.float32:
            assert np.array_equal(got, g), key
        else:
            strict = _strict(o["sample"]).reshape(g.shape) | (mode == "nearest")
            d = np.abs(got.astype(np.int32) - g.astype(np.int32))
            assert (d[strict] == 0).all() and d.max() <= 1, key


@pytest.mark.parametrize("k", range(len(IMAGE_CASES)))
def test_oracle_matches_reference_get_image(k):
    view = _view(IMAGE_CASES[k])
    for fmt in ("RGB", "BGR"):
        o = oe.crop_equi_full(PANO, *view, unit=True, swap_rb=fmt == "BGR")
        g = GOLD[f"image_{fmt}{k}"]
        s = o["sample"].astype(np.float32).astype(np.float64) * 255       # what the final truncation sees
        d = np.abs(o["im"].astype(np.int32) - g.astype(np.int32))
        assert (d[_strict(s)] == 0).all() and d.max() <= 1, fmt
    vfov, w, h, az, el, roll, ar = view
    horizon, vvp = pc.horizon_vvp(vfov, w, h, el, roll)
    assert list(horizon) == GOLD[f"image_horizon{k}"].tolist() and list(vvp) == GOLD[f"image_vvp{k}"].tolist()


def test_horizon_and_vvp_helpers_match_reference():
    for (vfov, w, h, el, roll), g in zip(GOLD["hv_cases"], GOLD["hv"]):
        args = (el / 180 * np.pi, roll / 180 * np.pi, vfov / 180 * np.pi, int(h), int(w))
        with np.errstate(invalid="ignore", divide="ignore"):
            horizon = pc.PanoCam.getRelativeHorizonLineFromAngles(*args)
            vvp = pc.PanoCam.getRelativeVVP(*args)
            mid = pc.PanoCam.getMidpointFromAngle(*args[:3])
        dh = pc.PanoCam.getDeltaHeightFromRoll(args[1], int(h), int(w))
        assert len(vvp) == int(g[5])
        got = np.array([*horizon, *vvp, *([np.nan] * (3 - len(vvp))), mid, dh])
        want = np.concatenate([g[:5], g[6:]])
        assert np.array_equal(got, want, equal_nan=True), (vfov, w, h, el, roll)
    hv = GOLD["hv_cases"]
    assert {0.0, 90.0, -90.0}.issubset(set(hv[:, 3])) and {90.0, -90.0, 180.0}.issubset(set(hv[:, 4]))


def _rule_rotation(view):
    fov_x, rot = oe.wrapper_args(*view)
    roll, el, az = rot["roll"], -rot["pitch"], -rot["yaw"]
    rr = np.array([[math.cos(roll), -math.sin(roll), 0], [math.sin(roll), math.cos(roll), 0], [0, 0, 1]])
    re = np.array([[1, 0, 0], [0, math.cos(el), -math.sin(el)], [0, math.sin(el), math.cos(el)]])
    ra = np.array([[math.cos(az), 0, math.sin(az)], [0, 1, 0], [-math.sin(az), 0, math.cos(az)]])
    return ra @ re @ rr, view[1] / (2 * math.tan(fov_x * math.pi / 180 / 2))


@pytest.mark.parametrize("i", range(len(CASES)))
def test_rule_latitude_and_up_match_reference_ground_truth(i):
    view = _view(CASES[i])
    vfov, w, h, az, el, roll, ar = view
    if abs(ar - w / h) > 1e-12:
        pytest.skip("ar != W / H: the crop's vertical field of view is not the vfov get_lat / get_up describe")
    o = oe.crop_equi_full(PANO, *view)
    lat = np.degrees(o["phi"])
    R, f = _rule_rotation(view)
    # the reference's linspace(-h/2, h/2, h) x linspace(-w/2, w/2, w) grid lies within one pixel of j - w/2, i - h/2 in each axis,
    # and a pixel step turns the ray by at most 1 / f rad
    assert np.abs(lat - GOLD[f"lat{i}"]).max() <= math.degrees(math.sqrt(2) / f)
    assert np.abs(lat - GOLD[f"lat{i}"]).max() <= vfov / h or el > 80   # one pixel's angle, except looking near the pole
    # the rule's up direction: the image of a small step towards world up (-y) from each pixel's ray
    j, ii = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    ray = np.stack(((j - w / 2) / f, (ii - h / 2) / f, np.ones_like(j)), -1)
    world = ray @ R.T
    cam = (world + np.array([0.0, -1e-6, 0.0])) @ R
    q = np.stack((f * cam[..., 0] / cam[..., 2] + w / 2, f * cam[..., 1] / cam[..., 2] + h / 2), -1)
    up = q - np.stack((j, ii), -1)
    up /= np.linalg.norm(up, axis=-1, keepdims=True)
    g = GOLD[f"up{i}"]
    c = np.array([0.0, -1.0, 0.0]) @ R                                # world up in the camera frame -> the VVP
    if abs(c[2]) > 1e-12:
        vvp = np.array([f * c[0] / c[2] + w / 2, f * c[1] / c[2] + h / 2])
        d = np.linalg.norm(vvp - np.stack((j, ii), -1), axis=-1)
    else:
        d = np.full(j.shape, np.inf)
    keep = d > 2
    err = np.linalg.norm(up - g, axis=-1)
    assert (err[keep] <= 0.75 / d[keep] + 1e-6).all(), float(err[keep].max())


@pytest.mark.parametrize("i", [i for i, c in enumerate(CASES) if c[5] == 0 and abs(c[6] - c[1] / c[2]) < 1e-12])
def test_rule_matches_crop_distortion_at_zero_roll(i):
    vfov, w, h, az, el, roll, ar = _view(CASES[i])
    o = oe.crop_equi_full(PANO, vfov, w, h, az, el, roll, ar)
    f = h / (2 * math.tan(math.radians(vfov) / 2))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)      # crop_distortion's minfocal: sqrt of a negative number at xi = 0
        cd = op.crop_distortion_full(PANO, f, 0.0, h, w, az, -el, 0.0)
        flipped = op.crop_distortion_full(PANO, f, 0.0, h, w, -az, -el, 0.0)
    assert np.abs(o["theta"] - cd["ntheta"]).max() <= 1e-12 and np.abs(o["phi"] - cd["nphi"]).max() <= 1e-12
    if az != 0:      # the azimuth's direction is pinned: the opposite sign is far off
        assert np.abs(o["theta"] - flipped["ntheta"]).max() > 0.1


def test_unit_path_matches_torchvision_at_exact_pixels():
    from PIL import Image
    from torchvision import transforms
    p = np.arange(256, dtype=np.uint8).reshape(16, 16)
    img = np.stack((p, p[::-1], p.T), -1)
    ref = np.array(transforms.ToPILImage()(transforms.ToTensor()(Image.fromarray(img))))
    chw = img.transpose(2, 0, 1).astype(np.float32) / np.float32(255)
    j, i = np.meshgrid(np.arange(16, dtype=np.float64), np.arange(16, dtype=np.float64))
    for mode in ("bilinear", "nearest"):
        got = oe.to_output(oe.sample(chw, j, i, mode), np.uint8, unit=True).transpose(1, 2, 0)
        assert np.array_equal(got, ref) and np.array_equal(got, img), mode     # every value survives p / 255 * 255 at a pixel


def test_python_api_checks_arguments_before_gpu_work():
    pano = np.zeros((16, 32, 3), np.uint8)
    good = (60.0, 8, 6, 0.0, 0.0, 0.0, 4 / 3)
    bad_views = [(0.0, 8, 6, 0, 0, 0, 1.0), (180.0, 8, 6, 0, 0, 0, 1.0), (-10.0, 8, 6, 0, 0, 0, 1.0), (float("nan"), 8, 6, 0, 0, 0, 1.0),
                 (60.0, 0, 6, 0, 0, 0, 1.0), (60.0, 8, 0, 0, 0, 0, 1.0), (60.0, 8.5, 6, 0, 0, 0, 1.0), (60.0, 8, 6, float("inf"), 0, 0, 1.0),
                 (60.0, 8, 6, 0, float("nan"), 0, 1.0), (60.0, 8, 6, 0, 0, float("-inf"), 1.0), (60.0, 8, 6, 0, 0, 0, 0.0),
                 (60.0, 8, 6, 0, 0, 0, float("nan")), (170.0, 8, 6, 0, 0, 0, 1e20), (60.0, 8, 6, 0, 0, 0), {"vfov": 60.0, "im_w": 8}]
    for v in bad_views:
        with pytest.raises(ValueError):
            pc.crop_equi_views(pano, [good, v])
    for kw in ({"mode": "bicubic"}, {"img_format": "HSV"}, {"outputs": ("up", "ntheta")}):
        with pytest.raises(ValueError):
            pc.crop_equi_views(pano, [good], **kw)
    with pytest.raises(ValueError):
        pc.crop_equi_views(pano, [])
    with pytest.raises(ValueError):
        pc.crop_equi_views(pano[:, :, 0], [good], img_format="BGR")
    for p in (pano.astype(np.float64), pano.astype(np.int32), pano[:, :, :2], pano[None], pano[:, :, :1]):
        with pytest.raises(TypeError):
            pc.crop_equi_views(p, [good])
    with pytest.raises(ValueError):
        pc.crop_equi_views(pano[:0], [good])
    with pytest.raises(ValueError):
        pc.PanoCam.crop_equi(pano, 60.0, 8, 6, 0.0, 0.0, 0.0, 4 / 3, "area")


def test_pf_equi_view_struct_layout():
    from perspectivefields_b200 import _native
    assert ctypes.sizeof(_native.pf_equi_view) == 56          # include/pf_b200.h: 2 x int32, 5 x double, int64
    assert _native.pf_equi_view.vfov.offset == 8 and _native.pf_equi_view.ar.offset == 40 and _native.pf_equi_view.offset.offset == 48
