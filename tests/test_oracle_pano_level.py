"""CPU: the panorama-levelling oracle (tests/oracle_pano_level.py) against the camera-fit oracle it restates in terms of v, an
independent solver (scipy.optimize.least_squares) and the rotation and normalisation rules."""
import math

import numpy as np
import pytest
from scipy.optimize import least_squares

import oracle_calib as oc
import oracle_pano_level as opl

# (vfov, im_w, im_h, azimuth, elevation, roll, ar): mixed sizes and aspect ratios, elevations of +-30 degrees
VIEWS = [(70.0, 32, 24, 0.0, 0.0, 0.0, 32 / 24), (60.0, 20, 30, 90.0, 30.0, 5.0, 0.8), (80.0, 28, 28, 200.0, -30.0, -10.0, 1.0),
         (65.0, 36, 24, 300.0, 10.0, 0.0, 1.2)]
TILTS = [(0.0, 0.0), (5.0, -3.0), (-12.0, 20.0), (25.0, 8.0)]


def _view_geometry(view):
    vfov, w, h, az, el, roll, ar = view
    return opl.crop_rotation(az, el, roll), opl.crop_focal(vfov, w, ar), h, w


def _compare(v, H, W, F, cam):
    u, l, _ = opl.model(v, H, W, F)
    uc, lc = oc.model(cam, H, W)
    assert np.max(np.abs(u - uc)) <= 1e-12 * F
    assert np.max(np.abs(l - lc)) <= 1e-12


@pytest.mark.parametrize("view", VIEWS)
def test_v_model_is_the_camera_model_for_a_level_panorama(view):
    A, F, H, W = _view_geometry(view)
    _, _, _, _, el, roll, _ = view
    v = A.T @ opl.N
    assert np.allclose(v, opl.level_up(math.radians(el), math.radians(roll)), atol=1e-15)
    _compare(v, H, W, F, (math.radians(roll), math.radians(el), math.log(F / H)))


@pytest.mark.parametrize("tilt", TILTS)
@pytest.mark.parametrize("view", VIEWS)
def test_v_model_is_the_effective_camera_for_a_tilted_panorama(tilt, view):
    A, F, H, W = _view_geometry(view)
    T = opl.tilt(math.radians(tilt[0]), math.radians(tilt[1]))
    a2, e2, r2 = opl.decompose(T @ A)
    assert np.allclose(opl.crop_rotation(a2, e2, r2), T @ A, atol=1e-14)
    g, _ = opl.gravity((math.radians(tilt[0]), math.radians(tilt[1])))
    assert np.allclose(g, T.T @ opl.N, atol=1e-15)
    _compare(A.T @ g, H, W, F, (math.radians(r2), math.radians(e2), math.log(F / H)))


def _panorama(rng, tilt, noise=True, weights=False):
    """Noisy fields of VIEWS' effective cameras under the tilt -> list of oracle view dicts."""
    T = opl.tilt(math.radians(tilt[0]), math.radians(tilt[1]))
    out = []
    for view in VIEWS:
        A, F, H, W = _view_geometry(view)
        _, e2, r2 = opl.decompose(T @ A)
        cam = (math.radians(r2), math.radians(e2), math.log(F / H))
        if noise:
            up, lat = oc.noisy_fields(rng, cam, H, W, holes=False)
        else:
            u, l = oc.model(cam, H, W)
            up, lat = (u / np.linalg.norm(u, axis=2, keepdims=True)).astype(np.float32), np.degrees(l).astype(np.float32)
        d = {"A": A, "F": F, "up": up, "lat": lat, "mask": rng.random((H, W)) > 0.1}
        if weights:
            d["weights"] = (rng.uniform(0.1, 1.0, (H, W)).astype(np.float32), rng.uniform(0.1, 1.0, (H, W)).astype(np.float32))
        out.append(d)
    return out


def _stacked_residuals(theta, views, sqrt_w):
    g, _ = opl.gravity(theta)
    rs = []
    for vw in views:
        r, _, w = opl.residuals(vw["A"].T @ g, vw["F"], vw["up"], vw["lat"], vw["mask"], vw.get("weights", (None, None)))
        rs.append(r * np.sqrt(w) if sqrt_w else r)
    return np.concatenate(rs)


@pytest.mark.parametrize("kind", ["least_squares", "huber", "weighted"])
def test_lm_agrees_with_least_squares(kind):
    rng = np.random.default_rng(3)
    views = _panorama(rng, (-12.0, 20.0), weights=kind == "weighted")
    huber = math.radians(2.0) if kind == "huber" else None
    got = opl.fit(views, huber=huber, max_iterations=200)
    assert got["status"] == 0
    ref = least_squares(lambda t: _stacked_residuals(t, views, kind == "weighted"), np.zeros(2), method="lm" if huber is None else "trf",
                        loss="linear" if huber is None else "huber", f_scale=huber or 1.0, xtol=1e-15, ftol=1e-15, gtol=1e-15)
    th = opl.normalise(ref.x)
    assert np.allclose(got["theta"], th, atol=1e-8), (got["theta"], th)
    assert abs(got["cost"] - ref.cost) <= 1e-9 * ref.cost


def test_exact_fields_give_the_tilt_back():
    rng = np.random.default_rng(1)
    for tilt in TILTS:
        got = opl.fit(_panorama(rng, tilt, noise=False), max_iterations=100)
        assert got["status"] == 0
        assert np.allclose(got["angles"], tilt, atol=1e-6), (got["angles"], tilt)


@pytest.mark.parametrize("theta", [(0.3, -0.2), (-1.2, 2.9), (1.5, 0.0), (0.0, math.pi), (-0.4, -3.0)])
def test_rotation_is_the_smallest_one_to_the_up_direction(theta):
    g, _ = opl.gravity(theta)
    R = opl.rotation_to(g)
    assert np.allclose(R @ opl.N, g, atol=1e-14)
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-14) and abs(np.linalg.det(R) - 1.0) < 1e-14
    angle = math.acos(max(-1.0, min(1.0, (np.trace(R) - 1.0) / 2.0)))
    assert abs(angle - math.acos(float(opl.N @ g))) < 1e-7
    axis = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    assert abs(axis @ opl.N) < 1e-14            # about a horizontal axis: no yaw
    # the device's closed form: R = c I + [w]x + w w^T / (1 + c), w = n x g, c = n . g (180 degrees about x where 1 + c = 0)
    w, c = np.cross(opl.N, g), float(opl.N @ g)
    if not 1.0 + c > 0.0:
        return
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    assert np.allclose(c * np.eye(3) + K + np.outer(w, w) / (1.0 + c), R, atol=1e-13)


def test_upside_down_rotation():
    assert np.array_equal(opl.rotation_to(-opl.N), np.diag([1.0, -1.0, -1.0]))


@pytest.mark.parametrize("theta", [(0.3, -0.2), (2.0, 0.5), (-2.5, -2.0), (1.0, 3.0)])
def test_normalisation_keeps_the_up_direction(theta):
    psi, phi = opl.normalise(theta)
    assert abs(psi) <= math.pi / 2 and -math.pi < phi <= math.pi
    assert np.allclose(opl.gravity((psi, phi))[0], opl.gravity(theta)[0], atol=1e-14)
    assert np.allclose(opl.gravity((math.pi - psi, phi + math.pi))[0], opl.gravity(theta)[0], atol=1e-14)


def test_identity_warp_keeps_rows_below_the_pole():
    rng = np.random.default_rng(0)
    pano = rng.integers(0, 256, (25, 50, 3), dtype=np.uint8)
    out, _, u, v = opl.rotate(pano, np.eye(3))
    assert np.array_equal(out[1:], pano[1:])
    assert np.allclose(u[1:], np.arange(50)[None, :], atol=1e-9) and np.allclose(v[1:], np.arange(1, 25)[:, None], atol=1e-9)
