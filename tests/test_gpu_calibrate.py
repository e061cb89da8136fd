"""GPU: the camera fit (csrc/calib.cuh) through calibrate.fit_camera and pf_fit_camera, against exact camera fields, the CPU
oracle (tests/oracle_calib.py) and inference_batch results read in place."""
import ctypes
import itertools
import math

import numpy as np
import pytest
import torch

import oracle_calib as oc
import pf_test_util as U
from perspectivefields_b200 import _native, calibrate, metrics, panocam

pytestmark = pytest.mark.gpu

PARAM_KEYS = ("pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy", "pred_rel_focal")


def _as_results(ups, lats):
    return [{"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l} for u, l in zip(ups, lats)]


def _f(t):
    return float(t)


@pytest.mark.parametrize("principal_point", [False, True])
def test_round_trip_on_camera_fields(principal_point):
    sizes = [(480, 640), (375, 500), (1080, 1920), (67, 93)]
    pps = [(0.0, 0.0)] + ([(0.08, -0.05)] if principal_point else [])
    cams = list(itertools.product((-40.0, 0.0, 25.0), (-60.0, -10.0, 0.0, 15.0, 70.0), (35.0, 60.0, 100.0), pps))
    hw = [sizes[i % len(sizes)] for i in range(len(cams))]
    focal = [1.0 / (2.0 * math.tan(math.radians(v) / 2.0)) for _, _, v, _ in cams]
    ups, lats = panocam.camera_fields(focal, [h for h, _ in hw], [w for _, w in hw], [math.radians(c[1]) for c in cams],
                                      [math.radians(c[0]) for c in cams], [c[3][0] for c in cams], [c[3][1] for c in cams])
    out = calibrate.fit_camera(_as_results(ups, lats), principal_point=principal_point)
    for (roll, pitch, _, (cx, cy)), f, o in zip(cams, focal, out):
        assert int(o["fit_status"]) == 0, (roll, pitch, f, cx, cy, {k: float(v) for k, v in o.items()})
        assert abs(_f(o["pred_roll"]) - roll) < 1e-4 and abs(_f(o["pred_pitch"]) - pitch) < 1e-4, (roll, pitch, f)
        assert abs(_f(o["pred_rel_focal"]) - f) < 1e-5
        assert abs(_f(o["pred_rel_cx"]) - cx) < 1e-5 and abs(_f(o["pred_rel_cy"]) - cy) < 1e-5
        assert all(o[k].dtype == torch.float64 and o[k].is_cuda and o[k].dim() == 0 for k in PARAM_KEYS)
        if not principal_point:
            assert abs(_f(o["pred_vfov"]) - math.degrees(2 * math.atan(0.5 / f))) < 1e-4
            assert list(o)[:7] == ["pred_roll", "pred_pitch", "pred_vfov", "pred_rel_focal", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy"]
        else:
            assert list(o)[:6] == list(PARAM_KEYS)


ORACLE_CAMS = [(0.3, -0.4, math.log(0.9), 0.05, -0.03), (-0.5, 0.9, math.log(0.6), -0.06, 0.02), (0.02, 0.1, math.log(1.5), 0.0, 0.0),
               (2.9, -0.2, math.log(1.1), 0.1, 0.1)]
ORACLE_SIZES = [(60, 80), (48, 96), (61, 45), (72, 72)]


def _oracle_case(seed=7):
    rng = np.random.default_rng(seed)
    ups, lats, masks = [], [], []
    for cam, (h, w) in zip(ORACLE_CAMS, ORACLE_SIZES):
        u, l = oc.noisy_fields(rng, cam, h, w)
        ups.append(u)
        lats.append(l)
        masks.append(rng.random((h, w)) > 0.15)
    masks[2] = None
    return ups, lats, masks


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_against_the_oracle(principal_point, huber):
    ups, lats, masks = _oracle_case()
    res = _as_results([torch.from_numpy(u).cuda() for u in ups], [torch.from_numpy(l).cuda() for l in lats])
    mk = [None if m is None else torch.from_numpy(m).cuda() for m in masks]
    first = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber, max_iterations=1)
    out = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber)
    for i in range(len(ups)):
        want0 = oc.fit(ups[i], lats[i], masks[i], principal_point, huber, max_iterations=1)
        assert int(first[i]["fit_status"]) == 1 and int(first[i]["fit_iterations"]) == 1
        got0 = [_f(first[i][k]) for k in ("pred_roll", "pred_pitch", "pred_rel_focal", "pred_rel_cx", "pred_rel_cy")]
        assert np.max(np.abs(np.asarray(got0) - want0["params"])) < 1e-9, (i, got0, want0["params"])
        want = oc.fit(ups[i], lats[i], masks[i], principal_point, huber)
        got = [_f(out[i][k]) for k in ("pred_roll", "pred_pitch", "pred_rel_focal", "pred_rel_cx", "pred_rel_cy")]
        assert int(out[i]["fit_status"]) == want["status"] == 0
        # degrees for the angles: 1e-7 relative to the radian parameters is 5.7e-6 degrees
        scale = np.array([180 / math.pi, 180 / math.pi, 1.0, 1.0, 1.0])
        assert np.all(np.abs(np.asarray(got) - want["params"]) <= 1e-7 * scale * np.maximum(1.0, np.abs(want["theta"]))), (i, got, want["params"])
        assert abs(_f(out[i]["fit_cost"]) - want["cost"]) <= 1e-9 * want["cost"], (i, _f(out[i]["fit_cost"]), want["cost"])


def _fit_raw(res, n_pad, principal_point=0, huber=0.0, max_iterations=50, init=None, ws_bytes=None, mutate=None):
    """pf_fit_camera on [2, H, W] / [H, W] CUDA fields with outputs inside NaN-prefilled buffers n_pad entries longer."""
    L = _native.lib()
    n = len(res)
    pu = [r["pred_gravity_original"] for r in res]
    pl = [r["pred_latitude_original"] for r in res]
    bu, bl = min(t.data_ptr() for t in pu), min(t.data_ptr() for t in pl)
    descs = (_native.pf_fit_image * max(n, 1))()
    for i in range(n):
        d = descs[i]
        d.height, d.width = pu[i].shape[1], pu[i].shape[2]
        d.up_offset = (pu[i].data_ptr() - bu) // 4
        d.up_stride[0], d.up_stride[1], d.up_stride[2] = pu[i].stride(1), pu[i].stride(2), pu[i].stride(0)
        d.lat_offset = (pl[i].data_ptr() - bl) // 4
        d.mask_offset = -1
        for k in range(5):
            d.init[k] = math.nan if init is None else init[k]
    params = torch.full((n + n_pad, 5), math.nan, dtype=torch.float64, device="cuda")
    cost = torch.full((n + n_pad,), math.nan, dtype=torch.float64, device="cuda")
    its = torch.full((n + n_pad,), -7, dtype=torch.int32, device="cuda")
    st = torch.full((n + n_pad,), -7, dtype=torch.int32, device="cuda")
    need = L.pf_fit_camera_workspace(descs, max(n, 1))
    ws = torch.empty(max(need, 256), dtype=torch.uint8, device="cuda")
    args = [0, descs, n, bu, bl, None, principal_point, huber, max_iterations, params.data_ptr(), cost.data_ptr(), its.data_ptr(), st.data_ptr(),
            ws.data_ptr(), need if ws_bytes is None else ws_bytes, torch.cuda.current_stream().cuda_stream]
    if mutate:
        mutate(args)
    rc = L.pf_fit_camera(*args)
    return rc, params, cost, its, st


def test_outputs_are_written_for_the_images_only():
    ups, lats, _ = _oracle_case(3)
    res = _as_results([torch.from_numpy(u).cuda() for u in ups], [torch.from_numpy(l).cuda() for l in lats])
    rc, params, cost, its, st = _fit_raw(res, 3)
    assert rc == 0
    n = len(res)
    assert torch.isnan(params[n:]).all() and torch.isnan(cost[n:]).all() and (its[n:] == -7).all() and (st[n:] == -7).all()
    assert not torch.isnan(params[:n]).any() and (st[:n] == 0).all()
    api = calibrate.fit_camera(res)
    for i in range(n):
        assert _f(api[i]["pred_roll"]) == float(params[i, 0]) and _f(api[i]["fit_cost"]) == float(cost[i])


@pytest.mark.parametrize("version,kw", [("PersNet-360Cities", {}), ("PersNet-360Cities", {"logits": False}),
                                        ("Paramnet-360Cities-edina-uncentered", {"resize": (384, 512)})])
def test_in_place_and_deterministic(version, kw):
    from oracle import weights_gen as wg
    m = U.make_model(version, seed=0, device="cuda", model_kwargs=kw)[0]
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(2, 240, 320, seed=4)] + \
        [torch.from_numpy(x).cuda() for x in wg.smooth_images(1, 200, 300, seed=5)]
    res = m.inference_batch(imgs)
    for pp, huber in ((False, None), (True, 0.05)):
        a = calibrate.fit_camera(res, principal_point=pp, huber=huber)
        b = calibrate.fit_camera(res, principal_point=pp, huber=huber)
        clones = [{"pred_gravity_original": r["pred_gravity_original"].clone(), "pred_latitude_original": r["pred_latitude_original"].clone()}
                  for r in res]
        c = calibrate.fit_camera(clones, principal_point=pp, huber=huber)
        for x, y, z in zip(a, b, c):
            for k in x:
                assert torch.equal(x[k], y[k]) or (torch.isnan(x[k]) and torch.isnan(y[k])), k
                assert torch.equal(x[k], z[k]) or (torch.isnan(x[k]) and torch.isnan(z[k])), k


@pytest.mark.parametrize("version,pp", [("Paramnet-360Cities-edina-centered", False), ("Paramnet-360Cities-edina-uncentered", True)])
def test_init_from_results(version, pp):
    from oracle import weights_gen as wg
    m = U.make_model(version, seed=0, device="cuda")[0]
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(2, 120, 160, seed=6)]
    res = m.inference_batch(imgs)
    out = calibrate.fit_camera(res, principal_point=pp, init="results", max_iterations=200)
    for r, o in zip(res, out):
        up = r["pred_gravity_original"].permute(1, 2, 0).cpu().numpy()
        lat = r["pred_latitude_original"].cpu().numpy()
        f = panocam.general_vfov_to_focal(float(r["pred_rel_cx"]), float(r["pred_rel_cy"]), 1, float(r["pred_general_vfov"]), True)
        th = oc.params_to_theta(float(r["pred_roll"]), float(r["pred_pitch"]), float(f), float(r["pred_rel_cx"]), float(r["pred_rel_cy"]))
        c0 = oc.cost_at(th, up, lat, None, pp)
        assert int(o["fit_status"]) in (0, 1)
        assert _f(o["fit_cost"]) <= c0 * (1 + 1e-9)
    keys = ("roll", "pitch", "vfov") if not pp else ("roll", "pitch", "general_vfov", "rel_cx", "rel_cy")
    pe = metrics.param_errors(out, {k: [0.0, 0.0] for k in keys})
    assert set(pe) == set(keys)
    # the fit of a real camera's fields draws those fields again
    ups, lats = panocam.camera_fields([0.8], [120], [160], [0.3], [-0.2], [0.05 if pp else 0.0], [-0.04 if pp else 0.0])
    fit = calibrate.fit_camera(_as_results(ups, lats), principal_point=pp)
    u2, l2 = panocam.fields_from_predictions(fit, [(120, 160)])
    assert (l2[0] - lats[0]).abs().max().item() < 1e-3 and (u2[0] - ups[0]).abs().max().item() < 1e-4


def test_edge_cases():
    assert calibrate.fit_camera([]) == []
    ups, lats = panocam.camera_fields([0.9, 0.9], [40, 40], [50, 50], [0.2, 0.2], [0.1, 0.1], [0.0, 0.0], [0.0, 0.0])
    dead_up = torch.zeros_like(ups[1])
    dead_lat = torch.full_like(lats[1], float("nan"))
    out = calibrate.fit_camera(_as_results([ups[0], dead_up], [lats[0], dead_lat]))
    assert int(out[0]["fit_status"]) == 0 and int(out[1]["fit_status"]) == 2
    assert all(math.isnan(_f(out[1][k])) for k in PARAM_KEYS) and math.isnan(_f(out[1]["fit_cost"]))
    one = calibrate.fit_camera(_as_results(ups, lats), max_iterations=1)
    assert all(int(o["fit_status"]) == 1 and int(o["fit_iterations"]) == 1 for o in one)
    mask = [torch.zeros((40, 50), dtype=torch.bool, device="cuda"), None]
    out = calibrate.fit_camera(_as_results(ups, lats), mask=mask)
    assert int(out[0]["fit_status"]) == 2 and int(out[1]["fit_status"]) == 0


def test_invalid_arguments_are_rejected_before_any_launch():
    L = _native.lib()
    ups, lats = panocam.camera_fields([0.9], [40], [50], [0.2], [0.1], [0.0], [0.0])
    res = _as_results(ups, lats)
    torch.cuda.synchronize()
    before = L.pf_kernel_launch_count()
    bad = [
        lambda a: a.__setitem__(2, 0),                              # n < 1
        lambda a: a.__setitem__(1, None),                           # no descriptors
        lambda a: a.__setitem__(3, None),                           # no up field
        lambda a: a.__setitem__(4, None),                           # no latitude field
        lambda a: a.__setitem__(6, 2),                              # principal_point not 0 / 1
        lambda a: a.__setitem__(7, -1.0),                           # huber < 0
        lambda a: a.__setitem__(7, math.inf),
        lambda a: a.__setitem__(7, math.nan),
        lambda a: a.__setitem__(8, 0),                              # max_iterations < 1
        lambda a: a.__setitem__(8, 1001),
        lambda a: a.__setitem__(9, None),                           # no params output
        lambda a: a.__setitem__(12, None),                          # no status output
        lambda a: a.__setitem__(13, a[13] + 8),                     # misaligned workspace
        lambda a: setattr(a[1][0], "height", 2),                    # smaller than 3 x 3
        lambda a: setattr(a[1][0], "width", 0),
        lambda a: setattr(a[1][0], "up_offset", -1),
        lambda a: setattr(a[1][0], "mask_offset", 0),               # a mask offset without a mask
        lambda a: setattr(a[1][0], "mask_offset", -2),
        lambda a: (a[1][0].init.__setitem__(0, 0.1), a[1][0].init.__setitem__(2, 0.0)),     # f_rel <= 0
        lambda a: (a[1][0].init.__setitem__(0, 0.1), a[1][0].init.__setitem__(2, 1.0), a[1][0].init.__setitem__(3, math.inf)),
    ]
    for k, mutate in enumerate(bad):
        rc, params, cost, its, st = _fit_raw(res, 1, mutate=mutate)
        assert rc == -1, (k, rc)
        assert torch.isnan(params).all() and torch.isnan(cost).all() and (its == -7).all() and (st == -7).all()
    rc, params, *_ = _fit_raw(res, 1, ws_bytes=64)
    assert rc == -4 and torch.isnan(params).all()
    assert L.pf_fit_camera_workspace(None, 1) < 0
    assert L.pf_kernel_launch_count() == before
    for call in (lambda: calibrate.fit_camera(res, init="bogus"), lambda: calibrate.fit_camera(res, huber=0.0),
                 lambda: calibrate.fit_camera(res, huber=math.nan), lambda: calibrate.fit_camera(res, max_iterations=0),
                 lambda: calibrate.fit_camera(res, principal_point=1), lambda: calibrate.fit_camera(res, init="results"),
                 lambda: calibrate.fit_camera(res, mask=[torch.ones((40, 49), dtype=torch.bool, device="cuda")]),
                 lambda: calibrate.fit_camera([{"pred_gravity_original": res[0]["pred_gravity_original"][:, :2],
                                                "pred_latitude_original": res[0]["pred_latitude_original"][:2]}])):
        with pytest.raises(ValueError):
            call()
    with pytest.raises(ValueError):
        calibrate.fit_camera([{"pred_gravity_original": res[0]["pred_gravity_original"].cpu(), "pred_latitude_original": lats[0].cpu()}])
    assert L.pf_kernel_launch_count() == before
