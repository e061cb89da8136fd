"""GPU: the weighted camera fit (calibrate.fit_camera(weights=...), pf_fit_camera_weighted / pf_fit_camera_groups_weighted) against
the weighted float64 oracle (tests/oracle_confidence.py), the unweighted and masked fits, and real confidence maps."""
import math

import numpy as np
import pytest
import torch

import oracle_calib as oc
import oracle_confidence as ocf
import pf_test_util as U
from oracle import weights_gen as wg
from perspectivefields_b200 import _native, calibrate, panocam

pytestmark = pytest.mark.gpu

CAMS = [(0.3, -0.4, math.log(0.9), 0.05, -0.03), (-0.5, 0.9, math.log(0.6), -0.06, 0.02), (0.02, 0.1, math.log(1.5), 0.0, 0.0)]
SIZES = [(60, 80), (48, 96), (61, 45)]
PKEYS = ("pred_roll", "pred_pitch", "pred_rel_focal", "pred_rel_cx", "pred_rel_cy")


def _same(a, b):
    """Two fit_camera outputs, bit for bit on every key."""
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert list(x) == list(y)
        for k in x:
            assert torch.equal(x[k], y[k]) or (torch.isnan(x[k]) and torch.isnan(y[k])), (k, float(x[k]), float(y[k]))


def _as_results(ups, lats):
    return [{"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l} for u, l in zip(ups, lats)]


def _case(seed=9):
    rng = np.random.default_rng(seed)
    ups, lats, wts = [], [], []
    for k, (cam, (h, w)) in enumerate(zip(CAMS, SIZES)):
        u, l = oc.noisy_fields(rng, cam, h, w)
        wu = rng.uniform(0.1, 2.0, (h, w)).astype(np.float32)
        wl = rng.uniform(0.1, 2.0, (h, w)).astype(np.float32)
        wu[rng.random((h, w)) < 0.05] = 0.0
        wl[rng.random((h, w)) < 0.03] = np.nan
        ups.append(u)
        lats.append(l)
        wts.append((wu, None if k == 2 else wl))
    return ups, lats, wts


def _cuda(ups, lats, wts):
    res = _as_results([torch.from_numpy(u).cuda() for u in ups], [torch.from_numpy(l).cuda() for l in lats])
    return res, [tuple(None if x is None else torch.from_numpy(x).cuda() for x in p) for p in wts]


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_against_the_weighted_oracle(principal_point, huber):
    ups, lats, wts = _case()
    res, w = _cuda(ups, lats, wts)
    first = calibrate.fit_camera(res, principal_point=principal_point, huber=huber, max_iterations=1, weights=w)
    out = calibrate.fit_camera(res, principal_point=principal_point, huber=huber, weights=w)
    scale = np.array([180 / math.pi, 180 / math.pi, 1.0, 1.0, 1.0])
    for i in range(len(ups)):
        want0 = ocf.fit(ups[i], lats[i], None, principal_point, huber, max_iterations=1, wu=wts[i][0], wl=wts[i][1])
        got0 = [float(first[i][k]) for k in PKEYS]
        assert np.max(np.abs(np.asarray(got0) - want0["params"])) < 1e-9, (i, got0, want0["params"])
        want = ocf.fit(ups[i], lats[i], None, principal_point, huber, wu=wts[i][0], wl=wts[i][1])
        got = [float(out[i][k]) for k in PKEYS]
        assert int(out[i]["fit_status"]) == want["status"] == 0
        assert np.all(np.abs(np.asarray(got) - want["params"]) <= 1e-7 * scale * np.maximum(1.0, np.abs(want["theta"]))), (i, got, want["params"])
        assert abs(float(out[i]["fit_cost"]) - want["cost"]) <= 1e-9 * want["cost"]


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_groups_against_the_weighted_grouped_oracle(principal_point, huber):
    ups, lats, wts = _case(seed=4)
    res, w = _cuda(ups, lats, wts)
    groups = [0, 0, 1]
    first = calibrate.fit_camera(res, principal_point=principal_point, huber=huber, groups=groups, weights=w, max_iterations=1)
    want0 = ocf.fit_groups(ups, lats, None, wts, groups, principal_point, huber, max_iterations=1)
    for o, x in zip(first, want0):
        assert int(o["fit_status"]) == 1 and int(o["fit_iterations"]) == 1
        assert np.max(np.abs(np.asarray([float(o[k]) for k in PKEYS]) - x["params"])) < 1e-9, ([float(o[k]) for k in PKEYS], x["params"])
        assert abs(float(o["fit_cost"]) - x["cost"]) <= 1e-9 * x["cost"]
    out = calibrate.fit_camera(res, principal_point=principal_point, huber=huber, groups=groups, weights=w, max_iterations=300)
    want = ocf.fit_groups(ups, lats, None, wts, groups, principal_point, huber, max_iterations=300)
    scale = np.array([180 / math.pi, 180 / math.pi, 1.0, 1.0, 1.0])
    for i, (o, x) in enumerate(zip(out, want)):
        assert int(o["fit_status"]) == x["status"] == 0, i
        got = np.asarray([float(o[k]) for k in PKEYS])
        assert np.all(np.abs(got - x["params"]) <= 1e-7 * scale * np.maximum(1.0, np.abs(x["theta"]))), (i, got, x["params"])
        assert abs(float(o["fit_cost"]) - x["cost"]) <= 1e-9 * x["cost"]
    for k in ("pred_rel_focal", "pred_rel_cx", "pred_rel_cy"):
        assert torch.equal(out[0][k], out[1][k])


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, 0.05])
@pytest.mark.parametrize("groups", [None, [0, 0, 1]])
def test_unit_weights_and_zero_weights_are_bit_identical(principal_point, huber, groups):
    ups, lats, _ = _case(seed=2)
    res, _ = _cuda(ups, lats, [(None, None)] * 3)
    kw = dict(principal_point=principal_point, huber=huber, groups=groups)
    base = calibrate.fit_camera(res, **kw)
    ones = [(torch.ones_like(r["pred_latitude_original"]), torch.ones_like(r["pred_latitude_original"])) for r in res]
    _same(base, calibrate.fit_camera(res, weights=ones, **kw))
    _same(base, calibrate.fit_camera(res, weights=[(ones[0][0], None), None, (None, ones[2][1])], **kw))
    masks, zw = [], []
    for r in res:
        h, w = r["pred_latitude_original"].shape
        keep = torch.ones((h, w), dtype=torch.bool, device="cuda")
        keep[h // 4:h // 2, w // 3:] = False
        masks.append(keep)
        wz = keep.float()
        zw.append((wz, wz.clone()))
    a = calibrate.fit_camera(res, mask=masks, **kw)
    b = calibrate.fit_camera(res, weights=zw, **kw)
    _same(a, b)
    _same(b, calibrate.fit_camera(res, weights=zw, **kw))     # a weighted call repeats bit for bit


@pytest.mark.parametrize("logits", [True, False])
def test_confidence_weights_on_real_results(logits):
    m = U.make_model("PersNet-360Cities", seed=0, device="cuda", model_kwargs={"logits": logits, "confidence": True})[0]
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(2, 120, 160, seed=6)]
    res = m.inference_batch(imgs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = calibrate.fit_camera(res, weights="confidence", huber=0.05)
        b = calibrate.fit_camera(res, weights=[(r["pred_gravity_confidence_original"], r["pred_latitude_confidence_original"]) for r in res],
                                 huber=0.05)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for x, y in zip(a, b):
        assert int(x["fit_status"]) in (0, 1)
        for k in x:
            assert torch.equal(x[k], y[k]), k


def test_weights_improve_the_fit_with_outliers():
    rng = np.random.default_rng(21)
    n, h, w = 12, 96, 128
    roll = rng.uniform(-30, 30, n)
    pitch = rng.uniform(-30, 30, n)
    focal = rng.uniform(0.6, 1.4, n)
    ups, lats = panocam.camera_fields(list(focal), [h] * n, [w] * n, list(np.radians(pitch)), list(np.radians(roll)), [0.0] * n, [0.0] * n)
    res, wts = [], []
    for i in range(n):
        u = ups[i].clone()
        l = lats[i].clone()
        sig_u = torch.from_numpy(np.where(rng.random((h, w)) < 0.3, 40.0, 1.0)).cuda().float()    # degrees: 30 % gross outliers
        sig_l = torch.from_numpy(np.where(rng.random((h, w)) < 0.3, 25.0, 0.5)).cuda().float()
        gen = torch.Generator(device="cuda").manual_seed(i)
        ang = torch.atan2(u[..., 1], u[..., 0]) + torch.deg2rad(sig_u * torch.randn((h, w), device="cuda", generator=gen))
        u = torch.stack([torch.cos(ang), torch.sin(ang)], dim=2)
        l = l + sig_l * torch.randn((h, w), device="cuda", generator=gen)
        res.append({"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l})
        wts.append((1.0 / sig_u ** 2, 1.0 / sig_l ** 2))            # the known inlier precision
    plain = calibrate.fit_camera(res)
    weighted = calibrate.fit_camera(res, weights=wts)
    err = lambda out, key, truth: np.median([abs(float(o[key]) - t) for o, t in zip(out, truth)])
    assert err(weighted, "pred_rel_focal", focal) < err(plain, "pred_rel_focal", focal)
    assert err(weighted, "pred_roll", roll) < err(plain, "pred_roll", roll)


def test_rejected_weights_raise_before_any_launch():
    L = _native.lib()
    ups, lats = panocam.camera_fields([0.9, 0.8], [40, 40], [50, 50], [0.2, 0.1], [0.1, 0.0], [0.0, 0.0], [0.0, 0.0])
    res = _as_results(ups, lats)
    good = torch.ones((40, 50), device="cuda")
    torch.cuda.synchronize()
    before = L.pf_kernel_launch_count()
    bad = ["bogus", "confidence", torch.ones(2, 40, 50, device="cuda"), [None], [None, None, None], [None, good], [(good,), None],
           [(good, good, good), None], [(good.double(), None), None], [(None, good[:, :49]), None], [(good.cpu(), None), None],
           [(good.half(), None), None], [(np.ones((40, 50), np.float32), None), None], 3]
    for wt in bad:
        with pytest.raises(ValueError):
            calibrate.fit_camera(res, weights=wt)
        with pytest.raises(ValueError):
            calibrate.fit_camera(res, weights=wt, groups=[0, 0])
    assert L.pf_kernel_launch_count() == before
