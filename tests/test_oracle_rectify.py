"""CPU: the upright warp's rule (tests/oracle_rectify.py) against the camera model pinned to the reference (tests/oracle_calib.py),
the "fill" focal length's definition, and a closed loop through the pinhole crop of a panorama (tests/oracle_equi.py)."""
import math

import numpy as np
import pytest
from scipy import ndimage

import oracle_calib as oc
import oracle_equi as oe
import oracle_rectify as orr
from perspectivefields_b200.panocam import general_vfov

# (roll, pitch, general vfov) in degrees, (cx_rel, cy_rel), (H, W): mixed sizes and off-centre principal points
CAMS = [((12.0, -8.0, 62.0), (0.0, 0.0), (48, 64)), ((-25.0, 20.0, 75.0), (0.06, -0.04), (61, 45)),
        ((3.0, 35.0, 95.0), (-0.1, 0.08), (40, 90)), ((-170.0, -15.0, 50.0), (0.02, 0.03), (72, 72)),
        ((0.0, 0.0, 60.0), (0.0, 0.0), (33, 57))]


def _params(c):
    (roll, pitch, gv), (cx, cy), _ = c
    return (roll, pitch, gv, cx, cy)


def _theta(r, e, f, cxr, cyr):
    return [r, e, math.log(f), cxr, cyr]


@pytest.mark.parametrize("cam", CAMS)
def test_continuous_form_matches_the_pinned_model(cam):
    H, W = cam[2]
    r, e, f, F, cx, cy = orr.input_camera(_params(cam), H, W)
    u, lat = oc.model(_theta(r, e, f, *cam[1]), H, W)
    y, x = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
    ux, uy = orr.up_vector(x, y, r, e, F, cx, cy)
    scale = np.max(np.abs(u))
    assert np.max(np.abs(ux - u[..., 0])) <= 1e-12 * scale and np.max(np.abs(uy - u[..., 1])) <= 1e-12 * scale
    gy, gx = np.meshgrid(cy + oc.lat_grid(H, cy), cx + oc.lat_grid(W, cx), indexing="ij")
    assert np.max(np.abs(orr.latitude(gx, gy, r, e, F, cx, cy) - lat)) < 1e-12


@pytest.mark.parametrize("keep_pitch", [False, True])
@pytest.mark.parametrize("focal", ["same", "fill", 70.0])
@pytest.mark.parametrize("cam", CAMS)
def test_output_camera_sees_what_the_input_saw(cam, keep_pitch, focal):
    """At every output pixel the output camera's latitude equals the input camera's at the mapped position, and the input's up
    direction carried through the map is the output camera's up field: (0, -1) at pitch 0, get_up_general at (0, e) otherwise."""
    H, W = cam[2]
    Ho, Wo = (H, W) if cam[2][0] % 2 else (H + 7, W - 5)
    st = orr.setup(_params(cam), H, W, Ho, Wo, keep_pitch, focal)
    assert st["status"] in (0, 1)
    r, e, f, F, cx, cy = st["input"]
    eo, Fo = (e if keep_pitch else 0.0), st["Fo"]
    assert st["camera"][1] == eo * orr.R2D
    y, x = np.meshgrid(np.arange(Ho) + 0.5, np.arange(Wo) + 0.5, indexing="ij")
    M = st["M"]
    Z = M[2, 0] * x + M[2, 1] * y + M[2, 2]
    u, v, _ = orr.positions(M, Ho, Wo, H, W)
    front = Z > 0
    assert front.any()
    lat_out = orr.latitude(x, y, 0.0, eo, Fo, Wo / 2.0, Ho / 2.0)
    lat_in = orr.latitude(u, v, r, e, F, cx, cy)
    assert np.max(np.abs(lat_out - lat_in)[front]) * orr.R2D < 1e-9
    dx, dy = orr.up_vector(u, v, r, e, F, cx, cy)
    ox, oy = orr.push_direction(np.linalg.inv(M), u, v, dx, dy)
    want, _ = oc.model([0.0, eo, math.log(Fo / Ho), 0.0, 0.0], Ho, Wo)
    if not keep_pitch:
        assert np.all(want[..., 0] == 0.0) and np.all(want[..., 1] < 0.0)
    ok = front & (np.hypot(want[..., 0], want[..., 1]) > 1e-6 * Fo) & (np.hypot(ox, oy) > 1e-12)
    ang = np.arctan2(ox * want[..., 1] - oy * want[..., 0], ox * want[..., 0] + oy * want[..., 1])
    assert ok.any() and np.max(np.abs(ang[ok])) < 1e-9


def _corners_inside(M, Ho, Wo, H, W, tol):
    for X in (0.0, Wo):
        for Y in (0.0, Ho):
            p = M @ np.array([X, Y, 1.0])
            if not (p[2] > 0 and -tol <= p[0] / p[2] <= W + tol and -tol <= p[1] / p[2] <= H + tol):
                return False
    return True


@pytest.mark.parametrize("keep_pitch", [False, True])
@pytest.mark.parametrize("cam", CAMS[:4])
def test_fill_is_the_least_zoom_that_fills(cam, keep_pitch):
    H, W = cam[2]
    st = orr.setup(_params(cam), H, W, H, W, keep_pitch, "fill")
    assert st["status"] == 0
    same = orr.setup(_params(cam), H, W, H, W, keep_pitch, "same")
    f_same = same["Fo"]
    assert st["Fo"] >= f_same
    assert _corners_inside(st["M"], H, W, H, W, 1e-9 * max(H, W))
    assert st["Fo"] > f_same * (1 + 1e-6), "these cameras need a zoom to fill"
    smaller = 2.0 * math.atan(H / (2.0 * st["Fo"] * (1 - 1e-9))) * orr.R2D
    assert not _corners_inside(orr.setup(_params(cam), H, W, H, W, keep_pitch, smaller)["M"], H, W, H, W, 0.0)
    u, v, valid = orr.positions(st["M"], H, W, H, W)
    assert valid.all()


def test_fill_is_the_same_focal_when_it_already_fills():
    st = orr.setup((0.0, 0.0, 60.0, 0.0, 0.0), 48, 64, 48, 64, False, "fill")
    assert st["status"] == 0 and st["Fo"] == orr.setup((0.0, 0.0, 60.0, 0.0, 0.0), 48, 64, 48, 64, False, "same")["Fo"]


@pytest.mark.parametrize("params,keep_pitch", [((0.0, 40.0, 60.0, 0.0, 0.0), False),      # pitch > vfov / 2: the horizon is off the image
                                               ((10.0, -70.0, 90.0, 0.0, 0.0), False),
                                               ((5.0, 0.0, 60.0, 0.7, 0.0), True)])        # principal point outside the image
def test_fill_impossible_gives_status_1_and_the_same_focal(params, keep_pitch):
    st = orr.setup(params, 48, 64, 48, 64, keep_pitch, "fill")
    assert st["status"] == 1
    assert st["Fo"] == orr.setup(params, 48, 64, 48, 64, keep_pitch, "same")["Fo"]


@pytest.mark.parametrize("params", [(math.nan, 0.0, 60.0, 0.0, 0.0), (0.0, 0.0, 0.0, 0.0, 0.0), (0.0, 0.0, -30.0, 0.0, 0.0),
                                    (0.0, math.inf, 60.0, 0.0, 0.0), (0.0, 0.0, 180.0, 0.0, 0.0), (0.0, 0.0, 170.0, 3.0, 0.0)])
def test_unusable_parameters_give_status_2(params):
    img = np.full((8, 10, 3), 77, np.uint8)
    o = orr.upright(img, params, fill=(1, 2, 3))
    assert o["status"] == 2 and not o["mask"].any() and np.isnan(o["map"]).all() and all(math.isnan(c) for c in o["camera"])
    assert (o["im"] == np.array([1, 2, 3], np.uint8)).all()


@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
@pytest.mark.parametrize("shape", [(9, 13, 3), (10, 7)])
def test_identity_camera_returns_the_image(mode, shape):
    img = np.random.default_rng(1).integers(0, 256, shape, dtype=np.uint8)
    o = orr.upright(img, (0.0, 17.0, 70.0, 0.0, 0.0), keep_pitch=True, mode=mode)
    assert o["status"] == 0 and o["mask"].all() and np.array_equal(o["im"], img)
    y, x = np.meshgrid(np.arange(shape[0]) + 0.5, np.arange(shape[1]) + 0.5, indexing="ij")
    assert np.max(np.abs(o["map"][..., 0] - x)) < 1e-5 and np.max(np.abs(o["map"][..., 1] - y)) < 1e-5


def test_bilinear_rounds_half_to_even():
    img = np.array([[[10], [11]], [[12], [13]]], np.uint8)
    # the pixel centre halfway between columns 0 and 1 of row 0: (10 + 11) / 2 = 10.5 -> 10; (12 + 13) / 2 -> 12
    M = np.array([[1.0, 0.0, 0.5], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    u, v, valid = orr.positions(M, 2, 1, 2, 2)
    out = orr.sample(img, u, v, valid, "bilinear", [0])
    assert out[0, 0, 0] == 10 and out[1, 0, 0] == 12


# ---------------------------------------------------------------- closed loop through the pinhole crop of a panorama
def smooth_panorama(seed, hp=256, wp=512):
    """uint8 [hp, wp, 3]: a few seeded low-frequency waves, periodic in azimuth."""
    rng = np.random.default_rng(seed)
    y, x = np.meshgrid((np.arange(hp) + 0.5) / hp * math.pi, np.arange(wp) / wp * 2 * math.pi, indexing="ij")
    ch = []
    for _ in range(3):
        a = np.zeros_like(x)
        for _ in range(3):
            a += rng.uniform(20, 40) * np.sin(rng.integers(1, 4) * x + rng.uniform(0, 6)) * np.cos(rng.integers(1, 4) * y + rng.uniform(0, 6))
        ch.append(128 + a)
    return np.clip(np.stack(ch, axis=2), 0, 255).astype(np.uint8)


def direct_view(pano, Ho, Wo, Fo, az, el):
    """The panorama sampled (oracle_equi's bilinear sampler, float64) along the rays of a pinhole camera at (az, el), roll 0,
    centred, focal Fo, at its pixel centres."""
    y, x = np.meshgrid((np.arange(Ho) + 0.5 - Ho / 2.0) / Fo, (np.arange(Wo) + 0.5 - Wo / 2.0) / Fo, indexing="ij")
    ce, se, ca, sa = math.cos(el), math.sin(el), math.cos(az), math.sin(az)
    ye, ze = y * ce - se, y * se + ce
    xa, za = x * ca + ze * sa, -(x * sa) + ze * ca
    n = np.sqrt((xa * xa + ye * ye) + za * za)
    hp, wp = pano.shape[:2]
    u = (np.arctan2(xa, za) + np.pi) * (wp / (2 * np.pi))
    v = (np.pi / 2 + np.arcsin(ye / n)) * (hp / np.pi)
    return oe.sample(pano.transpose(2, 0, 1), u, v, "bilinear").transpose(1, 2, 0)


# Worst |straightened - direct| over the masked interior (>= 2 px from the mask border), measured on the CPU for the four cases
# below: 1.42 - 1.48 levels (mean 0.35 - 0.39).  The straightened image interpolates twice (the crop, truncated to uint8, then
# the warp, rounded) where the direct view interpolates once: up to 1 level from the truncation, 0.5 from the rounding, plus the
# difference of two interpolants of a smooth panorama.  The same loop with the principal point half a pixel off (cx_rel =
# cy_rel = 0, see below) measures 1.89 - 2.21 levels, so this bound also catches a half-pixel error in the camera convention.
LOOP_TOL = 1.6


@pytest.mark.parametrize("az,el,roll,keep_pitch", [(30.0, 0.0, 20.0, False), (-50.0, 15.0, -10.0, False), (100.0, -25.0, 35.0, False),
                                                   (10.0, 20.0, 15.0, True)])
def test_closed_loop_through_the_pinhole_crop(az, el, roll, keep_pitch):
    pano = smooth_panorama(3)
    H, W, vfov = 120, 160, 60.0
    crop = oe.crop_equi_full(pano, vfov, W, H, az, el, roll, W / H, "bilinear")["im"]
    f = 1.0 / (2.0 * math.tan(math.radians(vfov) / 2.0))
    # the crop samples pixel k at k - W/2 from its centre ray, i.e. its principal point is the pixel-centre position W/2 + 1/2
    cxr, cyr = 0.5 / W, 0.5 / H
    gv = float(general_vfov(cxr, cyr, 1, f, True))
    o = orr.upright(crop, (roll, el, gv, cxr, cyr), keep_pitch=keep_pitch)
    assert o["status"] == 0 and o["camera"][1] == (el if keep_pitch else 0.0)
    ref = direct_view(pano, H, W, o["Fo"], math.radians(az), math.radians(el) if keep_pitch else 0.0)
    inner = ndimage.binary_erosion(o["mask"], iterations=2)
    assert inner.sum() > 0.3 * H * W
    err = np.abs(o["im"].astype(np.float64) - ref)[inner]
    assert err.max() <= LOOP_TOL, err.max()
