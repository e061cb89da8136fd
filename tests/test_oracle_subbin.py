"""CPU: the sub-bin decode oracle (tests/oracle_subbin.py) against the reference's bin decode where it must not refine, and against
the properties DESIGN.md section 1 "Sub-bin decode" states: exact on quadratic peaks, continuous across adjacent argmax switches
(the pole bins of the latitude head excepted), |delta| <= 1/2, and delta = 0 on non-finite logits."""
import numpy as np
import pytest
import torch

import oracle_subbin as osb
from oracle import model as om

G, L = 73, 180   # classes of the up and latitude heads
F32 = np.float32


def _quadratic(mu, nc, sigma, circular):
    """Logits -d^2 / (2 sigma^2) in the (circular) bin distance d to mu; for the up head bin 72 lies far below."""
    k = np.arange(nc - 1 if circular else nc)
    d = k[None, :] - np.asarray(mu, np.float64)[:, None]
    if circular:
        d = (d + (nc - 1) / 2) % (nc - 1) - (nc - 1) / 2
    l = -d * d / (2 * sigma * sigma)
    if circular:
        l = np.concatenate([l, np.full((len(l), 1), -1e4)], 1)
    return l.astype(F32)


def _argmax_gravity(l):
    return om.decode_bin(torch.from_numpy(l.argmax(-1)), G).numpy().T


def _argmax_latitude(l):
    return om.decode_bin_latitude(torch.from_numpy(l.argmax(-1)), L).numpy()


def test_unrefined_cases_equal_the_reference_decode():
    rng = np.random.default_rng(0)
    g = rng.normal(size=(6 + G, G)).astype(F32)
    g[0, 10], g[0, 9], g[0, 11] = 5, 3, 3                  # symmetric neighbours
    g[1, 0], g[1, 71], g[1, 1] = 5, 2, 2                   # symmetric across the wrap
    g[2, 72] = 9                                           # the no-direction bin
    g[3, :] = 1                                            # all tied: bin 0, flat
    g[4, 5] = g[4, 9] = 7                                  # two-way tie, first wins; bin 5's neighbours are random
    g[4, 4] = g[4, 6] = 0
    g[5, 40], g[5, 39], g[5, 41] = 4, -np.inf, 3            # a non-finite neighbour
    for c in range(G):                                     # every bin with symmetric neighbours
        g[6 + c] = -10
        g[6 + c, c] = 1
    want = _argmax_gravity(g)
    got = osb.decode_gravity(g)
    assert got.dtype == np.float32 and np.array_equal(got, want.astype(F32))

    l = rng.normal(size=(4 + L, L)).astype(F32)
    l[0, 0], l[0, 1] = 9, 8                                # pole bins: not refined whatever the neighbour
    l[1, L - 1], l[1, L - 2] = 9, 1
    l[2, 100], l[2, 99], l[2, 101] = 3, 1, 1
    l[3, :] = 0
    for c in range(L):
        l[4 + c] = -10
        l[4 + c, c] = 1
    got = osb.decode_latitude(l)
    assert got.dtype == np.float32 and np.array_equal(got, _argmax_latitude(l).astype(F32))
    c, d = osb.position(l, False)
    assert d[0] == 0 and d[1] == 0


@pytest.mark.parametrize("sigma", [0.5, 1.0, 2.0])
def test_quadratic_peaks_are_recovered(sigma):
    rng = np.random.default_rng(int(sigma * 10))
    mu = np.concatenate([rng.uniform(0, 72, 4000), [0.0, 0.3, 71.5, 71.7, 71.99, 35.5]])
    c, d = osb.position(_quadratic(mu, G, sigma, True), True)
    err = np.abs((c + d.astype(np.float64) - mu + 36) % 72 - 36)
    assert err.max() <= 1e-4, err.max()
    up = osb.decode_gravity(_quadratic(mu, G, sigma, True))
    ang = np.deg2rad(mu * 5 - 180)
    assert np.abs(up - np.stack([np.cos(ang), np.sin(ang)], -1)).max() < 1e-5

    mu = np.concatenate([rng.uniform(0.5, L - 1.5, 4000), [1.0, 1.49, 100.5, L - 1.51]])
    c, d = osb.position(_quadratic(mu, L, sigma, False), False)
    assert np.abs(c + d.astype(np.float64) - mu).max() <= 1e-4
    lat = osb.decode_latitude(_quadratic(mu, L, sigma, False))
    assert np.abs(lat - (mu - 89.5)).max() < 1e-4 * 1.0 + 1e-5


def test_fine_sweep_is_continuous():
    step = 0.02
    mu = np.arange(0, 72 + step / 2, step)
    c, d = osb.position(_quadratic(mu, G, 1.0, True), True)
    pos = c + d.astype(np.float64)
    jump = np.abs((np.diff(pos) + 36) % 72 - 36)
    assert jump.max() <= step + 1e-4, jump.max()         # including 71 -> 0 across the wrap
    up = osb.decode_gravity(_quadratic(mu, G, 1.0, True))
    assert np.linalg.norm(np.diff(up, axis=0), axis=1).max() <= np.deg2rad(5 * step) + 1e-4

    mu = np.arange(-1, L + step / 2, step)
    c, d = osb.position(_quadratic(mu, L, 1.0, False), False)
    pos = c + d.astype(np.float64)
    jump = np.abs(np.diff(pos))
    interior = (c[1:] > 0) & (c[1:] < L - 1) & (c[:-1] > 0) & (c[:-1] < L - 1)
    assert jump[interior].max() <= step + 1e-4
    assert jump.max() <= 0.5 + step + 1e-4                # the documented exception: entering or leaving a pole bin
    assert jump[~interior].max() > 0.4


def test_switch_between_adjacent_bins_meets_in_the_middle():
    rng = np.random.default_rng(3)
    for c0 in list(range(G - 1)):
        l = rng.normal(size=G).astype(F32) - 10
        c1 = (c0 + 1) % (G - 1)
        l[c0] = l[c1] = 0.0
        l[(c0 - 1) % (G - 1)] = -1.0
        l[(c1 + 1) % (G - 1)] = -1.0
        a = l.copy()
        b = l.copy()
        a[c0] += F32(1e-6)
        b[c1] += F32(1e-6)
        pa = osb.position(a, True)
        pb = osb.position(b, True)
        wa = (pa[0] + float(pa[1]) - (c0 + 0.5) + 36) % 72 - 36
        wb = (pb[0] + float(pb[1]) - (c0 + 0.5) + 36) % 72 - 36
        assert abs(wa) < 1e-5 and abs(wb) < 1e-5, c0


def test_delta_is_bounded_and_zero_on_non_finite_logits():
    rng = np.random.default_rng(5)
    for nc, grav in ((G, True), (L, False)):
        l = (rng.normal(size=(20000, nc)) * rng.choice([0.01, 1, 100], size=(20000, 1))).astype(F32)
        _, d = osb.position(l, grav)
        assert np.abs(d).max() <= 0.5
    inf, nan = F32(np.inf), F32(np.nan)
    assert osb.delta_of(1, -inf, 0) == 0 and osb.delta_of(1, 0, -inf) == 0
    assert osb.delta_of(inf, 0, 1) == 0 and osb.delta_of(1, nan, 0) == 0 and osb.delta_of(1, 0, nan) == 0
    assert osb.delta_of(1, 1, 1) == 0
    assert osb.delta_of(1, 0, 0) == 0 and osb.delta_of(1, 0, 1) == 0.5 and osb.delta_of(1, 1, 0) == -0.5
    big = F32(3e38)
    assert osb.delta_of(big, -big, 0) == 0      # a overflows to inf
    g = np.zeros((1, G), F32)
    g[0, 10], g[0, 9], g[0, 11] = 1, -np.inf, 0
    assert np.array_equal(osb.decode_gravity(g), _argmax_gravity(g).astype(F32))


def test_chw_layout_and_post_process():
    rng = np.random.default_rng(7)
    lg = rng.normal(size=(2, G, 5, 6)).astype(F32)
    ll = rng.normal(size=(2, L, 5, 6)).astype(F32)
    up = osb.decode_gravity(lg, axis=1)
    lat = osb.decode_latitude(ll, axis=1)
    assert up.shape == (2, 2, 5, 6) and lat.shape == (2, 5, 6)
    assert np.array_equal(up, np.moveaxis(osb.decode_gravity(np.moveaxis(lg, 1, -1)), -1, 1))
    assert np.array_equal(lat, osb.decode_latitude(np.moveaxis(ll, 1, -1)))
    # with unrefined logits the post-process is oracle.model's
    lg = np.full((G, 320, 320), -5, F32)
    ll = np.full((L, 320, 320), -5, F32)
    ci = rng.integers(0, G, size=(320, 320))
    li = rng.integers(0, L, size=(320, 320))
    np.put_along_axis(lg, ci[None], 1, 0)
    np.put_along_axis(ll, li[None], 1, 0)
    cfg = {"gravity": "classification", "latitude": "classification", "gravity_classes": G, "latitude_classes": L}
    tg, tl = torch.from_numpy(lg), torch.from_numpy(ll)
    assert torch.allclose(osb.postprocess_gravity(lg, 120, 170), om.postprocess_gravity(cfg, tg, 120, 170), atol=1e-6)
    assert torch.allclose(osb.postprocess_latitude(ll, 120, 170), om.postprocess_latitude(cfg, tl, 120, 170), atol=1e-5)
    # at another working size, the crop and scale follow net_hw
    sub = np.ascontiguousarray(ll[:, :256, :288])
    assert osb.postprocess_latitude(sub, 64, 80, (256, 288)).shape == (64, 80)
