"""CPU: the grouped camera fit's rule (tests/oracle_calib_shared.py) against scipy.optimize.least_squares on the joint problem,
exact fields, the per-image fit (tests/oracle_calib.py) and its degenerate cases."""
import math

import numpy as np
import pytest
import scipy.optimize

import oracle_calib as oc
import oracle_calib_shared as ocs

SIZES = [(30, 40), (36, 48), (24, 32), (33, 44)]   # scaled copies of one 4:3 camera
# per group: the shared (ln f_rel, cx_rel, cy_rel), then each member's (roll, pitch)
GROUPS = [((math.log(0.9), 0.05, -0.03), [(0.2, -0.3), (-0.4, 0.5), (0.1, 0.1), (0.6, -0.8)]),
          ((math.log(1.3), -0.07, 0.04), [(-0.1, 0.2), (0.3, -0.1), (-0.7, 0.9)]),
          ((math.log(0.6), 0.0, 0.08), [(2.8, -0.2), (-2.9, 0.3), (0.05, -0.6)])]


def _case(seed, principal_point, noisy=True):
    rng = np.random.default_rng(seed)
    ups, lats, masks, groups, truth = [], [], [], [], []
    for gid, (shared, members) in enumerate(GROUPS):
        for j, (r, e) in enumerate(members):
            h, w = SIZES[(gid + j) % len(SIZES)]
            cam = (r, e, shared[0]) + (shared[1:] if principal_point else (0.0, 0.0))
            if noisy:
                u, l = oc.noisy_fields(rng, cam, h, w)
                masks.append(rng.random((h, w)) > 0.1)
            else:
                u, l = oc.model(cam, h, w)
                l = np.degrees(l)
                masks.append(None)
            ups.append(u)
            lats.append(l)
            groups.append(gid)
            truth.append(cam)
    return ups, lats, masks, groups, truth


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(3.0)])
def test_grouped_fit_agrees_with_scipy(principal_point, huber):
    P = 5 if principal_point else 3
    K = P - 2
    ups, lats, masks, groups, _ = _case(5, principal_point)
    out = ocs.fit_groups(ups, lats, masks, groups, principal_point, huber, max_iterations=300)
    fields = list(zip(ups, lats, masks))
    kw = dict(loss="linear") if huber is None else dict(loss="huber", f_scale=huber)
    for gid in range(len(GROUPS)):
        mem = [i for i, g in enumerate(groups) if g == gid]
        assert all(out[i]["status"] == 0 and out[i]["iterations"] < 300 for i in mem)
        starts, shared = ocs.group_start(fields, mem, principal_point)
        x0 = np.array([v for i in mem for v in starts[i][:2]] + shared[:K])
        sp = scipy.optimize.least_squares(lambda x: ocs.joint_residuals(x, mem, fields, P)[0], x0,
                                          jac=lambda x: ocs.joint_residuals(x, mem, fields, P)[1], method="trf", x_scale="jac",
                                          ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=1000, **kw)
        cost = sum(out[i]["cost"] for i in mem)
        assert cost <= sp.cost * (1 + 1e-9), (gid, cost, sp.cost)
        for j, i in enumerate(mem):
            t = oc.normalise(list(sp.x[2 * j:2 * j + 2]) + list(sp.x[2 * len(mem):]) + [0.0] * (3 - K))
            assert np.max(np.abs(np.asarray(out[i]["theta"]) - t)) < 1e-6, (i, out[i]["theta"], t)
        # one shared value per group
        assert all(out[i]["theta"][2:] == out[mem[0]]["theta"][2:] for i in mem)


@pytest.mark.parametrize("principal_point", [False, True])
def test_exact_fields_recover_the_cameras(principal_point):
    ups, lats, masks, groups, truth = _case(0, principal_point, noisy=False)
    out = ocs.fit_groups(ups, lats, masks, groups, principal_point)
    for o, cam in zip(out, truth):
        assert o["status"] == 0
        assert np.max(np.abs(np.asarray(o["theta"]) - np.asarray(oc.normalise(list(cam))))) < 1e-9


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(3.0)])
def test_a_group_of_one_is_the_per_image_fit(principal_point, huber):
    ups, lats, masks, _, _ = _case(9, principal_point)
    for i in (0, 5, 8):
        want = oc.fit(ups[i], lats[i], masks[i], principal_point, huber)
        got = ocs.fit_groups([ups[i]], [lats[i]], [masks[i]], [0], principal_point, huber)[0]
        assert got["status"] == want["status"] == 0
        assert np.max(np.abs(np.asarray(got["theta"]) - want["theta"])) < 1e-9
        assert abs(got["cost"] - want["cost"]) <= 1e-9 * want["cost"]
        one = ocs.fit_groups([ups[i]], [lats[i]], [masks[i]], [0], principal_point, huber, max_iterations=1)[0]
        want1 = oc.fit(ups[i], lats[i], masks[i], principal_point, huber, max_iterations=1)
        assert one["status"] == want1["status"] == 1 and one["params"] == want1["params"] and one["cost"] == want1["cost"]


def test_grouping_steadies_the_focal_length():
    rng = np.random.default_rng(21)
    f = 0.85
    ups, lats = [], []
    for _ in range(16):
        cam = (rng.uniform(-0.5, 0.5), rng.uniform(-0.6, 0.6), math.log(f), 0.0, 0.0)
        u, l = oc.noisy_fields(rng, cam, 30, 40, up_noise_deg=4.0, lat_noise_deg=3.0)
        ups.append(u)
        lats.append(l)
    single = [abs(oc.fit(u, l, None, huber=math.radians(4.0))["params"][2] - f) for u, l in zip(ups, lats)]
    grouped = ocs.fit_groups(ups, lats, None, [0] * 16, huber=math.radians(4.0))
    assert len({o["params"][2] for o in grouped}) == 1
    assert abs(grouped[0]["params"][2] - f) < np.median(single), (grouped[0]["params"][2], single)


def test_dropped_members_and_degenerate_groups():
    ups, lats, masks, groups, _ = _case(3, True, noisy=False)
    dead_up, dead_lat = np.full_like(ups[1], np.nan), np.full_like(lats[1], np.nan)
    ups[1], lats[1] = dead_up, dead_lat
    out = ocs.fit_groups(ups, lats, masks, groups, True)
    g0 = [i for i, g in enumerate(groups) if g == 0]
    assert out[1]["status"] == 2 and all(math.isnan(v) for v in out[1]["params"]) and math.isnan(out[1]["cost"])
    assert out[1]["iterations"] == out[0]["iterations"] > 1
    assert all(out[i]["status"] == 0 for i in g0 if i != 1)
    # the rest of the group as the fit without the dropped member (exact fields: one optimum)
    rest = [i for i in g0 if i != 1]
    alone = ocs.fit_groups([ups[i] for i in rest], [lats[i] for i in rest], [masks[i] for i in rest], [0] * len(rest), True)
    for i, o in zip(rest, alone):
        assert np.max(np.abs(np.asarray(out[i]["theta"]) - o["theta"])) < 1e-9
    # every member dead: the whole group has status 2 after one evaluation
    dead = ocs.fit_groups([dead_up] * 2, [dead_lat] * 2, None, [0, 0])
    assert all(o["status"] == 2 and o["iterations"] == 1 and math.isnan(o["cost"]) for o in dead)
    # two members with 2 residuals each: 4 residuals < 2 * 2 + 3 parameters
    m = np.zeros(lats[0].shape, bool)
    m[5, 7] = True
    few = ocs.fit_groups([ups[0], ups[2]], [lats[0], lats[2]], [m, m[: lats[2].shape[0], : lats[2].shape[1]]], [0, 0], True)
    assert all(o["status"] == 2 and all(math.isnan(v) for v in o["params"]) for o in few)
    # a member whose one residual is too few is dropped; the others go on
    m1 = np.zeros(lats[2].shape, bool)
    m1[4, 4] = True
    lat_only = lats[2].copy()
    up_none = np.full_like(ups[2], np.nan)
    mixed = ocs.fit_groups([ups[0], up_none], [lats[0], lat_only], [None, m1], [0, 0], False)
    assert mixed[1]["status"] == 2 and mixed[0]["status"] == 0
