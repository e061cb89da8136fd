"""CPU: the camera-track fit's rule (tests/oracle_calib_sequence.py) against scipy.optimize.least_squares on the stacked
residuals, the per-image and grouped fits at its limits, a frame without data, and the jitter it removes."""
import math

import numpy as np
import pytest
import scipy.optimize

import oracle_calib as oc
import oracle_calib_sequence as oseq
import oracle_calib_shared as ocs

H, W = 24, 32


def _track(m, rng, jitter_deg=1.0, principal_point=False, noisy=True, period=40.0):
    """m frames of one camera on a slow sinusoidal roll / pitch track, each jittered by N(0, jitter) degrees.  Returns (ups,
    lats, the true track (roll, pitch) in radians [m, 2], the jittered cameras)."""
    t = np.arange(m)
    track = np.radians(np.stack([8.0 * np.sin(2 * np.pi * t / period) + 3.0, 5.0 * np.cos(2 * np.pi * t / (1.4 * period)) - 4.0], axis=1))
    cams = []
    ups, lats = [], []
    for k in range(m):
        r, e = track[k] + np.radians(jitter_deg) * rng.standard_normal(2)
        cam = (r, e, math.log(0.8)) + ((0.04, -0.03) if principal_point else (0.0, 0.0))
        if noisy:
            u, l = oc.noisy_fields(rng, cam, H, W, holes=False)
        else:
            u, l = oc.model(cam, H, W)
            u, l = u.astype(np.float32), np.degrees(l).astype(np.float32)
        ups.append(u)
        lats.append(l)
        cams.append(cam)
    return ups, lats, track, cams


def _huber_loss(M, huber):
    """scipy's callable loss for the stacked residuals: Huber on the unscaled pixel residual r = f sqrt(M) (entries with M > 0),
    quadratic on the prior's entries; rho in terms of z = f^2 with the 1 / M scaling kept."""
    pix = M > 0
    Ms = np.where(pix, M, 1.0)

    def loss(z):
        r2 = z * Ms
        lin = pix & (r2 > huber * huber)
        a = np.sqrt(np.where(lin, r2, 1.0))
        rho = np.where(lin, (2.0 * huber * a - huber * huber) / Ms, z)
        d1 = np.where(lin, huber / a, 1.0)
        d2 = np.where(lin, -0.5 * huber * Ms / np.where(lin, a ** 3, 1.0), 0.0)
        return np.stack([rho, d1, d2])

    return loss


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(3.0)])
def test_sequence_fit_agrees_with_scipy(principal_point, huber):
    P = 5 if principal_point else 3
    K = P - 2
    rng = np.random.default_rng(3)
    ups, lats, _, _ = _track(6, rng, principal_point=principal_point)
    masks = [rng.random((H, W)) > 0.1 for _ in ups]
    sigma = (0.5, 0.8)
    mem = list(range(len(ups)))
    fields = list(zip(ups, lats, masks))
    out = oseq.fit_sequence(fields, mem, sigma, principal_point, huber, max_iterations=300)
    assert all(out[i]["status"] == 0 and out[i]["iterations"] < 300 for i in mem)
    x0 = oseq.sequence_start(fields, mem, principal_point)[:2 * len(mem) + K]
    M = oseq.stacked_residuals(x0, mem, fields, P, sigma)[2]
    kw = dict(loss="linear") if huber is None else dict(loss=_huber_loss(M, huber))
    sp = scipy.optimize.least_squares(lambda x: oseq.stacked_residuals(x, mem, fields, P, sigma)[0], x0,
                                      jac=lambda x: oseq.stacked_residuals(x, mem, fields, P, sigma)[1], method="trf", x_scale="jac",
                                      ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=1000, **kw)
    x = out[0]["x"]
    C = oseq.evaluate(x, mem, fields, P, huber, 1 / sigma[0] ** 2, 1 / sigma[1] ** 2)[0]
    assert C <= sp.cost * (1 + 1e-9), (C, sp.cost)
    assert np.max(np.abs(x - sp.x)) < 1e-6, np.max(np.abs(x - sp.x))


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(3.0)])
def test_a_single_frame_is_the_per_image_fit(principal_point, huber):
    rng = np.random.default_rng(5)
    ups, lats, _, _ = _track(1, rng, principal_point=principal_point)
    mask = rng.random((H, W)) > 0.1
    got = oseq.fit_sequence([(ups[0], lats[0], mask)], [0], (1.0, 1.0), principal_point, huber, 300)[0]
    want = oc.fit(ups[0], lats[0], mask, principal_point, huber, 300)
    assert got["status"] == want["status"] == 0
    assert np.max(np.abs(np.array(got["theta"]) - np.array(want["theta"]))) < 1e-9
    assert abs(got["cost"] - want["cost"]) <= 1e-9 * want["cost"]


@pytest.mark.parametrize("principal_point", [False, True])
def test_a_loose_prior_is_the_grouped_fit(principal_point):
    rng = np.random.default_rng(7)
    ups, lats, _, _ = _track(5, rng, jitter_deg=3.0, principal_point=principal_point)
    mem = list(range(5))
    got = oseq.fit_sequences(ups, lats, None, [0] * 5, 1e12, principal_point, None, 300)
    want = ocs.fit_groups(ups, lats, None, [0] * 5, principal_point, None, 300)
    for i in mem:
        assert got[i]["status"] == want[i]["status"] == 0
        assert np.max(np.abs(np.array(got[i]["theta"]) - np.array(want[i]["theta"]))) < 1e-7, i
        assert abs(got[i]["cost"] - want[i]["cost"]) <= 1e-7 * want[i]["cost"]


def test_a_tight_prior_gives_one_angle_pair():
    rng = np.random.default_rng(9)
    ups, lats, _, _ = _track(5, rng, jitter_deg=2.0)
    out = oseq.fit_sequences(ups, lats, None, [0] * 5, 1e-6, False, None, 300)
    th = np.array([o["theta"][:2] for o in out])
    assert all(o["status"] == 0 for o in out)
    assert np.max(np.abs(th - th[0])) < 1e-9, th


def test_a_fully_masked_frame_sits_at_its_neighbours_mean():
    rng = np.random.default_rng(11)
    ups, lats, _, _ = _track(5, rng, jitter_deg=2.0)
    masks = [None] * 5
    masks[2] = np.zeros((H, W), bool)
    out = oseq.fit_sequences(ups, lats, masks, [0] * 5, 0.5, True, None, 300)
    assert all(o["status"] == 0 for o in out)
    assert out[2]["cost"] == 0.0
    x = out[2]["x"]
    assert abs(x[4] - 0.5 * (x[2] + x[6])) < 1e-9 and abs(x[5] - 0.5 * (x[3] + x[7])) < 1e-9


def test_unwrapped_roll_starts():
    rng = np.random.default_rng(13)
    ups, lats, _, _ = _track(3, rng)
    fields = [(u, l, None) for u, l in zip(ups, lats)]
    inits = [(math.pi - 0.05, 0.0, 0.8, 0, 0), (-math.pi + 0.05, 0.0, 0.8, 0, 0), (math.pi - 0.1 + 4 * math.pi, 0.0, 0.8, 0, 0)]
    x = oseq.sequence_start(fields, [0, 1, 2], False, inits)
    assert abs(x[2] - (math.pi + 0.05)) < 1e-12 and abs(x[4] - (math.pi - 0.1)) < 1e-12


def test_the_prior_halves_the_jitter():
    rng = np.random.default_rng(17)
    m = 48
    ups, lats, track, _ = _track(m, rng, jitter_deg=1.0, noisy=False, period=400.0)
    smooth = oseq.fit_sequences(ups, lats, None, [0] * m, 0.1, False, None, 300)
    alone = [oc.fit(u, l, None, False, None, 300) for u, l in zip(ups, lats)]

    def rms(out):
        th = np.array([o["theta"][:2] for o in out])
        return math.sqrt(np.mean((th - track) ** 2))

    assert all(o["status"] == 0 for o in smooth)
    assert rms(smooth) <= 0.5 * rms(alone), (rms(smooth), rms(alone))


def test_the_banded_solve_is_the_dense_one():
    rng = np.random.default_rng(19)
    n, K = 40, 3
    B = rng.standard_normal((n + K, n + K))
    M = B @ B.T + (n + K) * np.eye(n + K)
    for i in range(n):   # zero outside the locals' band and the shared border
        for j in range(n):
            if abs(i - j) > 3:
                M[i, j] = 0.0
    b = rng.standard_normal(n + K)
    assert np.max(np.abs(oseq._solve_banded(M, b, K) - oseq._solve_dense(M, b))) < 1e-10
