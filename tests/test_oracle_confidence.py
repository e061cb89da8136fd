"""CPU: the float64 oracle of the head confidence and of the weighted camera fit (tests/oracle_confidence.py) against torch's
softmax, the unweighted oracle and scipy."""
import math

import numpy as np
import pytest
import torch
from scipy.optimize import approx_fprime, least_squares

import oracle_calib as oc
import oracle_calib_shared as ocs
import oracle_confidence as ocf

CAM = (0.3, -0.4, math.log(0.9), 0.05, -0.03)


def _case(seed=3, h=40, w=52):
    rng = np.random.default_rng(seed)
    up, lat = oc.noisy_fields(rng, CAM, h, w)
    wu = rng.uniform(0.2, 3.0, (h, w)).astype(np.float32)
    wl = rng.uniform(0.2, 3.0, (h, w)).astype(np.float32)
    return rng, up, lat, wu, wl


def test_confidence_matches_torch_softmax():
    rng = np.random.default_rng(0)
    for nc in (73, 180):
        logits = rng.standard_normal((nc, 9, 11)) * rng.uniform(0.1, 20.0)
        want = torch.softmax(torch.from_numpy(logits), dim=0).amax(dim=0).numpy()
        got = ocf.confidence(logits)
        assert np.max(np.abs(got - want)) < 1e-15
        assert np.all(got >= 1.0 / nc - 1e-15) and np.all(got <= 1.0)


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_unit_weights_are_the_unweighted_fit(principal_point, huber):
    _, up, lat, _, _ = _case()
    h, w = lat.shape
    ones = np.ones((h, w), np.float32)
    a = oc.fit(up, lat, None, principal_point, huber)
    b = ocf.fit(up, lat, None, principal_point, huber, wu=ones, wl=ones)
    assert a["status"] == b["status"] == 0
    assert a["params"] == b["params"] and a["cost"] == b["cost"] and a["iterations"] == b["iterations"]


@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_zero_weights_are_the_masked_fit(huber):
    rng, up, lat, _, _ = _case()
    h, w = lat.shape
    region = np.zeros((h, w), bool)
    region[5:20, 10:40] = True
    region |= rng.random((h, w)) < 0.1
    wts = np.where(region, 0.0, 1.0).astype(np.float32)
    a = oc.fit(up, lat, ~region, True, huber)
    b = ocf.fit(up, lat, None, True, huber, wu=wts, wl=wts)
    assert a["params"] == b["params"] and a["cost"] == b["cost"] and a["iterations"] == b["iterations"]


def test_least_squares_matches_scipy_on_scaled_residuals():
    _, up, lat, wu, wl = _case()
    P = 5
    got = ocf.fit(up, lat, None, True, None, wu=wu, wl=wl)
    assert got["status"] == 0

    def fun(th):
        ru, _, vu, rl, _, vl = ocf.residuals(th, up, lat, None, P, wu, wl)
        return np.concatenate([np.sqrt(vu) * ru, np.sqrt(vl) * rl])

    x0 = np.array(ocf.start(up, lat, None, wu, wl) + (0.0, 0.0))
    ref = least_squares(fun, x0, xtol=1e-15, ftol=1e-15, gtol=1e-15, method="lm")
    th = np.array(oc.normalise(list(ref.x)))
    assert np.max(np.abs(np.array(got["theta"]) - th)) < 1e-7, (got["theta"], th)
    assert abs(got["cost"] - ref.cost) <= 1e-9 * ref.cost


def test_huber_gradient_vanishes_at_the_solution():
    _, up, lat, wu, wl = _case(seed=5)
    huber = math.radians(2.5)
    got = ocf.fit(up, lat, None, True, huber, wu=wu, wl=wl)
    assert got["status"] == 0
    th = np.array(got["theta"])
    f = lambda t: ocf.cost(t, up, lat, None, 5, huber, wu, wl)
    grad = approx_fprime(th, f, 1e-7)                  # forward differences: step error ~ 1e-7 x the Hessian
    hess = np.abs(np.diag(ocf.evaluate(th, up, lat, None, 5, huber, wu, wl)[1]))
    assert np.all(np.abs(grad) < 1e-6 * hess), (grad, hess)
    central = np.array([(f(th + e) - f(th - e)) / 2e-6 for e in np.eye(5) * 1e-6])
    assert np.max(np.abs(central)) < 1e-6 * max(1.0, got["cost"]), central
    _, _, g, _ = ocf.evaluate(th, up, lat, None, 5, huber, wu, wl)
    assert np.max(np.abs(g)) < 1e-6 * max(1.0, got["cost"]), g


def test_start_uses_only_weighted_pixels():
    _, up, lat, _, _ = _case()
    h, w = lat.shape
    wu = np.ones((h, w), np.float32)
    wl = np.ones((h, w), np.float32)
    wu[h // 2 - 4:h // 2 + 4, w // 2 - 4:w // 2 + 4] = np.nan       # no usable up weight in the start window: roll falls back to 0
    wl[h // 2 - 4:h // 2 + 4, w // 2 - 4:w // 2 + 4] = -1.0
    r, e, s = ocf.start(up, lat, None, wu, wl)
    assert (r, e, s) == (0.0, 0.0, math.log(oc.F_DEFAULT))


@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_grouped_unit_weights_are_the_unweighted_grouped_fit(huber):
    rng = np.random.default_rng(8)
    cams = [CAM, (-0.2, 0.3, math.log(0.9), 0.05, -0.03), (0.1, -0.1, math.log(1.2), 0.0, 0.0)]
    ups, lats, ones, wts = [], [], [], []
    for cam in cams:
        u, l = oc.noisy_fields(rng, cam, 36, 44)
        ups.append(u)
        lats.append(l)
        ones.append((np.ones((36, 44), np.float32), np.ones((36, 44), np.float32)))
        wts.append((rng.uniform(0.2, 3.0, (36, 44)).astype(np.float32), None))
    a = ocs.fit_groups(ups, lats, None, [0, 0, 1], True, huber)
    b = ocf.fit_groups(ups, lats, None, ones, [0, 0, 1], True, huber)
    for x, y in zip(a, b):
        assert x["params"] == y["params"] and x["cost"] == y["cost"] and x["iterations"] == y["iterations"]
    # a group of one image is that image's weighted fit
    c = ocf.fit_groups(ups[2:], lats[2:], None, wts[2:], [0], True, huber, max_iterations=300)[0]
    d = ocf.fit(ups[2], lats[2], None, True, huber, max_iterations=300, wu=wts[2][0], wl=wts[2][1])
    assert np.max(np.abs(np.array(c["theta"]) - np.array(d["theta"]))) < 1e-8
