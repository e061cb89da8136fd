"""CPU: the camera fit's rule (tests/oracle_calib.py) against the reference's field functions (oracle/panocam.py), central
differences, and scipy.optimize.least_squares as an independent solver; panocam.general_vfov against the reference formula."""
import math

import numpy as np
import pytest
import scipy.optimize

import oracle_calib as oc
from oracle import panocam as op
from perspectivefields_b200 import panocam

THETAS = [(0.3, 0.0, 0.1, 0.0, 0.0), (-0.7, 0.4, -0.2, 0.08, -0.05), (2.0, -1.1, 0.4, -0.2, 0.15), (0.0, 1.2, -0.5, 0.0, 0.0),
          (-3.0, -0.05, 0.0, 0.3, 0.3)]


@pytest.mark.parametrize("theta", THETAS)
@pytest.mark.parametrize("hw", [(30, 40), (33, 17)])
def test_model_is_the_reference_field(theta, hw):
    H, W = hw
    r, e, s, cx, cy = theta
    u, l = oc.model(theta, H, W)
    ref_up = op.get_up_general(math.exp(s), W, H, e, r, cx, cy)
    ref_lat = op.get_lat_general(math.exp(s), W, H, e, r, cx, cy)
    un = u / np.linalg.norm(u, axis=2)[..., None]
    if e == 0:
        assert np.allclose(u / np.linalg.norm(u, axis=2)[..., None], [-math.sin(r), -math.cos(r)], atol=1e-15, rtol=0)
    assert np.max(np.abs(un - ref_up)) < 1e-12
    assert np.max(np.abs(np.degrees(l) - ref_lat)) < 1e-12


@pytest.mark.parametrize("theta", THETAS)
@pytest.mark.parametrize("P", [3, 5])
def test_jacobian_matches_central_differences(theta, P):
    H, W = 21, 26
    du, dl = oc.jacobians(theta, H, W, P)
    for k in range(P):
        h = 1e-6
        tp, tm = list(theta), list(theta)
        tp[k] += h
        tm[k] -= h
        (up, lp), (um, lm) = oc.model(tp, H, W), oc.model(tm, H, W)
        nu, nl = (up - um) / (2 * h), (lp - lm) / (2 * h)
        assert np.max(np.abs(du[..., k] - nu)) <= 1e-6 * max(np.max(np.abs(nu)), 1.0)
        assert np.max(np.abs(dl[..., k] - nl)) <= 1e-6 * max(np.max(np.abs(nl)), 1.0)
    # the residual Jacobians, through the atan2 of the up residual
    rng = np.random.default_rng(3)
    upf, lat = oc.noisy_fields(rng, theta, H, W)
    _, Ju, _, Jl = oc.residuals(theta, upf, lat, None, P)
    for k in range(P):
        h = 1e-6
        tp, tm = list(theta), list(theta)
        tp[k] += h
        tm[k] -= h
        (rup, _, rlp, _), (rum, _, rlm, _) = oc.residuals(tp, upf, lat, None, P), oc.residuals(tm, upf, lat, None, P)
        d = np.angle(np.exp(1j * (rup - rum))) / (2 * h)
        assert np.max(np.abs(Ju[:, k] - d)) <= 1e-6 * max(np.max(np.abs(d)), 1.0)
        assert np.max(np.abs(Jl[:, k] - (rlp - rlm) / (2 * h))) <= 1e-6 * max(np.max(np.abs(Jl[:, k])), 1.0)


CAMS = [(0.2, -0.3, math.log(0.9), 0.0, 0.0), (-0.6, 0.9, math.log(0.6), 0.08, -0.05), (0.05, 0.15, math.log(1.4), -0.1, 0.04)]


@pytest.mark.parametrize("cam", CAMS)
@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(3.0)])
def test_fit_agrees_with_scipy(cam, principal_point, huber):
    H, W = 36, 48
    P = 5 if principal_point else 3
    rng = np.random.default_rng(11)
    cam = cam if principal_point else cam[:3] + (0.0, 0.0)
    up, lat = oc.noisy_fields(rng, cam, H, W)
    mask = rng.random((H, W)) > 0.1
    res = oc.fit(up, lat, mask, principal_point, huber, max_iterations=200)
    assert res["status"] == 0 and res["iterations"] < 200

    def fun(t):
        ru, _, rl, _ = oc.residuals(t, up, lat, mask, P)
        return np.concatenate([ru, rl])

    def jac(t):
        _, Ju, _, Jl = oc.residuals(t, up, lat, mask, P)
        return np.concatenate([Ju, Jl])

    kw = dict(loss="linear") if huber is None else dict(loss="huber", f_scale=huber)
    sp = scipy.optimize.least_squares(fun, np.asarray(res["start"]), jac=jac, method="trf", x_scale="jac", ftol=1e-15, xtol=1e-15,
                                      gtol=1e-15, max_nfev=1000, **kw)
    assert res["cost"] <= sp.cost * (1 + 1e-9)
    t = np.asarray(oc.normalise(list(sp.x) + [0.0] * (5 - P)))
    assert np.max(np.abs(np.asarray(res["theta"]) - t)) < 1e-6
    # and the fit lands near the true camera (plain least squares is pulled by the outliers: a looser bound)
    tol = 0.05 if huber is None else 0.02
    assert abs(res["theta"][0] - cam[0]) < tol and abs(res["theta"][1] - cam[1]) < tol


@pytest.mark.parametrize("cam", CAMS)
@pytest.mark.parametrize("principal_point", [False, True])
def test_exact_fields_recover_the_camera(cam, principal_point):
    H, W = 40, 60
    cam = cam if principal_point else cam[:3] + (0.0, 0.0)
    u, l = oc.model(cam, H, W)
    res = oc.fit(u, np.degrees(l), None, principal_point)
    assert res["status"] == 0
    assert np.max(np.abs(np.asarray(res["theta"]) - np.asarray(cam))) < 1e-9


def test_start_and_normalisation():
    H, W = 48, 64
    cam = (0.4, -0.3, math.log(0.8), 0.0, 0.0)
    u, l = oc.model(cam, H, W)
    r, e, s = oc.start(u, np.degrees(l), None)
    assert abs(r - cam[0]) < 0.05 and abs(e - cam[1]) < 0.05 and abs(s - cam[2]) < 0.1
    empty = np.full((H, W, 2), np.nan), np.full((H, W), np.nan)
    assert oc.start(*empty, None) == (0.0, 0.0, math.log(oc.F_DEFAULT))
    for th in ([0.3, 2.0, 0.1], [-3.0, -1.9, 0.0], [7.0, 4.0, 0.2]):
        n = oc.normalise(th + [0.0, 0.0])
        assert abs(n[1]) <= math.pi / 2 and -math.pi < n[0] <= math.pi
        (ua, la), (ub, lb) = oc.model(th, 9, 11), oc.model(n, 9, 11)
        assert np.allclose(ua, ub, atol=1e-12) and np.allclose(la, lb, atol=1e-12)
    res = oc.fit(*empty, None)
    assert res["status"] == 2 and all(math.isnan(v) for v in res["params"])
    assert oc.fit(u, np.degrees(l), None, max_iterations=1)["status"] == 1


def _reference_general_vfov(d_cx, d_cy, h, focal, degree):
    """utils/utils.py:13-44, restated."""
    p_sqr = focal ** 2 + d_cx ** 2 + (d_cy + 0.5 * h) ** 2
    q_sqr = focal ** 2 + d_cx ** 2 + (d_cy - 0.5 * h) ** 2
    cos_fov = (p_sqr + q_sqr - h ** 2) / 2 / np.sqrt(p_sqr) / np.sqrt(q_sqr)
    fov = np.arccos(cos_fov)
    return np.degrees(fov) if degree else fov


def test_general_vfov():
    rng = np.random.default_rng(5)
    cx, cy, f = rng.uniform(-0.3, 0.3, 50), rng.uniform(-0.3, 0.3, 50), rng.uniform(0.3, 3.0, 50)
    for degree in (True, False):
        g = panocam.general_vfov(cx, cy, 1, f, degree)
        assert np.array_equal(g, _reference_general_vfov(cx, cy, 1, f, degree))
        assert np.max(np.abs(panocam.general_vfov_to_focal(cx, cy, 1, g, degree) - f)) < 1e-12
    assert panocam.general_vfov(0.0, 0.0, 480, 415.0, True) == _reference_general_vfov(0.0, 0.0, 480, 415.0, True)
    assert abs(panocam.general_vfov(0.0, 0.0, 1, 1 / (2 * math.tan(0.5)), False) - 1.0) < 1e-15
