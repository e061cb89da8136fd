"""GPU: the camera fit with shared intrinsics (csrc/calib.cuh, fit_group_step_kernel) through calibrate.fit_camera(groups=...)
and pf_fit_camera_groups, against the grouped CPU oracle (tests/oracle_calib_shared.py), exact camera fields, the per-image fit
and inference_batch results read in place."""
import ctypes
import math

import numpy as np
import pytest
import torch

import oracle_calib as oc
import oracle_calib_shared as ocs
import pf_test_util as U
from perspectivefields_b200 import _native, calibrate, panocam

pytestmark = pytest.mark.gpu

KEYS = ("pred_roll", "pred_pitch", "pred_rel_focal", "pred_rel_cx", "pred_rel_cy")
SIZES = [(60, 80), (48, 64), (72, 96), (45, 60)]
# per group: the shared (ln f_rel, cx_rel, cy_rel), then each member's (roll, pitch)
GROUPS = [((math.log(0.9), 0.05, -0.03), [(0.3, -0.4), (-0.5, 0.9), (0.02, 0.1)]),
          ((math.log(1.3), -0.06, 0.02), [(2.9, -0.2), (0.4, 0.3), (-0.3, -0.7), (0.1, 0.5)])]


def _as_results(ups, lats):
    return [{"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l} for u, l in zip(ups, lats)]


def _params(o):
    return np.array([float(o[k]) for k in KEYS])


def _case(seed=7, principal_point=True):
    rng = np.random.default_rng(seed)
    ups, lats, masks, groups = [], [], [], []
    for gid, (shared, members) in enumerate(GROUPS):
        for j, (r, e) in enumerate(members):
            h, w = SIZES[(gid + j) % len(SIZES)]
            cam = (r, e, shared[0]) + (shared[1:] if principal_point else (0.0, 0.0))
            u, l = oc.noisy_fields(rng, cam, h, w)
            ups.append(u)
            lats.append(l)
            masks.append(rng.random((h, w)) > 0.15)
            groups.append(gid)
    masks[2] = None
    # interleave the groups: images 0, 2, 4 ... of the list above go first
    order = [0, 3, 1, 4, 2, 5, 6]
    return [ups[i] for i in order], [lats[i] for i in order], [masks[i] for i in order], [groups[i] for i in order]


def _cuda(ups, lats, masks):
    res = _as_results([torch.from_numpy(u).cuda() for u in ups], [torch.from_numpy(l).cuda() for l in lats])
    return res, [None if m is None else torch.from_numpy(m).cuda() for m in masks]


def _same(a, b):
    for x, y in zip(a, b):
        for k in x:
            assert torch.equal(x[k], y[k]) or (torch.isnan(x[k]) and torch.isnan(y[k])), k


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_against_the_grouped_oracle(principal_point, huber):
    ups, lats, masks, groups = _case(7, principal_point)
    res, mk = _cuda(ups, lats, masks)
    first = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber, max_iterations=1, groups=groups)
    want0 = ocs.fit_groups(ups, lats, masks, groups, principal_point, huber, max_iterations=1)
    for o, w in zip(first, want0):
        assert int(o["fit_status"]) == 1 and int(o["fit_iterations"]) == 1
        assert np.max(np.abs(_params(o) - w["params"])) < 1e-9, (_params(o), w["params"])
        assert abs(float(o["fit_cost"]) - w["cost"]) <= 1e-9 * w["cost"]
    out = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber, max_iterations=300, groups=groups)
    want = ocs.fit_groups(ups, lats, masks, groups, principal_point, huber, max_iterations=300)
    scale = np.array([180 / math.pi, 180 / math.pi, 1.0, 1.0, 1.0])
    for i, (o, w) in enumerate(zip(out, want)):
        assert int(o["fit_status"]) == w["status"] == 0, i
        got = _params(o)
        assert np.all(np.abs(got - w["params"]) <= 1e-7 * scale * np.maximum(1.0, np.abs(w["theta"]))), (i, got, w["params"])
        assert abs(float(o["fit_cost"]) - w["cost"]) <= 1e-9 * w["cost"], (i, float(o["fit_cost"]), w["cost"])
    for gid in set(groups):   # the shared values are bit-identical across each group
        mem = [i for i, g in enumerate(groups) if g == gid]
        for k in ("pred_rel_focal", "pred_rel_cx", "pred_rel_cy", "pred_general_vfov"):
            assert all(torch.equal(out[i][k], out[mem[0]][k]) for i in mem)
        assert len({int(out[i]["fit_iterations"]) for i in mem}) == 1


@pytest.mark.parametrize("principal_point", [False, True])
def test_round_trip_on_camera_fields(principal_point):
    rolls, pitches = [-40.0, 0.0, 25.0, 10.0, -5.0, 30.0], [-60.0, -10.0, 15.0, 70.0, 0.0, -30.0]
    cams = [(0.8, 0.08, -0.05), (1.6, -0.04, 0.06)] if principal_point else [(0.8, 0.0, 0.0), (1.6, 0.0, 0.0)]
    sizes = [(480, 640), (240, 320), (96, 128)]
    groups = [i % 2 for i in range(6)]
    hw = [sizes[i % 3] for i in range(6)]
    c = [cams[g] for g in groups]
    ups, lats = panocam.camera_fields([x[0] for x in c], [h for h, _ in hw], [w for _, w in hw], [math.radians(p) for p in pitches],
                                      [math.radians(r) for r in rolls], [x[1] for x in c], [x[2] for x in c])
    out = calibrate.fit_camera(_as_results(ups, lats), principal_point=principal_point, groups=groups)
    for o, r, p, (f, cx, cy) in zip(out, rolls, pitches, c):
        assert int(o["fit_status"]) == 0
        assert abs(float(o["pred_roll"]) - r) < 1e-4 and abs(float(o["pred_pitch"]) - p) < 1e-4
        assert abs(float(o["pred_rel_focal"]) - f) < 1e-5
        assert abs(float(o["pred_rel_cx"]) - cx) < 1e-5 and abs(float(o["pred_rel_cy"]) - cy) < 1e-5
        assert all(o[k].dtype == torch.float64 and o[k].is_cuda and o[k].dim() == 0 for k in KEYS)
        assert o["fit_iterations"].dtype == torch.int32 and o["fit_status"].dtype == torch.int32
    single = calibrate.fit_camera(_as_results(ups, lats), principal_point=principal_point)
    assert [list(o) for o in out] == [list(o) for o in single]


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
def test_one_member_groups_are_the_per_image_fit(principal_point, huber):
    ups, lats, masks, _ = _case(11, principal_point)
    res, mk = _cuda(ups, lats, masks)
    n = len(res)
    a = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber, max_iterations=1)
    b = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber, max_iterations=1, groups=list(range(n)))
    _same(a, b)
    a = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber, max_iterations=300)
    b = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, huber=huber, max_iterations=300, groups=np.arange(n))
    scale = np.array([180 / math.pi, 180 / math.pi, 1.0, 1.0, 1.0])
    for i, (x, y) in enumerate(zip(a, b)):
        w = oc.fit(ups[i], lats[i], masks[i], principal_point, huber, max_iterations=300)
        assert int(x["fit_status"]) == int(y["fit_status"]) == w["status"] == 0
        for got in (_params(x), _params(y)):
            assert np.all(np.abs(got - w["params"]) <= 1e-7 * scale * np.maximum(1.0, np.abs(w["theta"]))), (i, got, w["params"])
        assert abs(float(y["fit_cost"]) - w["cost"]) <= 1e-9 * w["cost"]


def test_layouts_labels_and_repeats_are_bit_identical():
    ups, lats, masks, groups = _case(13)
    res, mk = _cuda(ups, lats, masks)
    kw = dict(principal_point=True, huber=math.radians(2.5), mask=mk)
    a = calibrate.fit_camera(res, groups=groups, **kw)
    _same(a, calibrate.fit_camera(res, groups=groups, **kw))
    _same(a, calibrate.fit_camera(res, groups=[7 if g == 0 else -3 for g in groups], **kw))   # relabelled
    _same(a, calibrate.fit_camera(res, groups=[np.int64(g + 100) for g in groups], **kw))
    order = sorted(range(len(res)), key=lambda i: groups[i])   # contiguous, the same order inside each group
    c = calibrate.fit_camera([res[i] for i in order], groups=[groups[i] for i in order], principal_point=True, huber=math.radians(2.5),
                             mask=[mk[i] for i in order])
    _same([a[i] for i in order], c)


def test_a_dropped_member():
    rolls, pitches = [10.0, -20.0, 5.0, 30.0], [5.0, -15.0, 20.0, 0.0]
    ups, lats = panocam.camera_fields([0.9] * 4, [60, 90, 60, 45], [80, 120, 80, 60], [math.radians(p) for p in pitches],
                                      [math.radians(r) for r in rolls], [0.04] * 4, [-0.03] * 4)
    ups[2] = torch.zeros_like(ups[2])
    lats[2] = torch.full_like(lats[2], float("nan"))
    out = calibrate.fit_camera(_as_results(ups, lats), principal_point=True, groups=[0, 0, 0, 0])
    assert int(out[2]["fit_status"]) == 2 and all(math.isnan(float(out[2][k])) for k in KEYS) and math.isnan(float(out[2]["fit_cost"]))
    assert int(out[2]["fit_iterations"]) == int(out[0]["fit_iterations"])
    keep = [0, 1, 3]
    alone = calibrate.fit_camera(_as_results([ups[i] for i in keep], [lats[i] for i in keep]), principal_point=True, groups=[0, 0, 0])
    for i, o in zip(keep, alone):
        assert int(out[i]["fit_status"]) == int(o["fit_status"]) == 0
        assert np.max(np.abs(_params(out[i]) - _params(o))) < 1e-9
    # every member dead, or too few residuals: status 2 for the whole group after one evaluation
    dead = calibrate.fit_camera(_as_results([ups[2], ups[2]], [lats[2], lats[2]]), groups=[0, 0])
    assert all(int(o["fit_status"]) == 2 and int(o["fit_iterations"]) == 1 for o in dead)
    m = torch.zeros((60, 80), dtype=torch.bool, device="cuda")
    m[30, 40] = True
    few = calibrate.fit_camera(_as_results([ups[0], ups[0]], [lats[0], lats[0]]), principal_point=True, mask=[m, m], groups=[0, 0])
    assert all(int(o["fit_status"]) == 2 for o in few)


@pytest.mark.parametrize("version,kw,init,pp", [("PersNet-360Cities", {}, "fields", False), ("PersNet-360Cities", {}, "fields", True),
                                                ("Paramnet-360Cities-edina-uncentered", {}, "results", True)])
def test_inference_results_in_place(version, kw, init, pp):
    from oracle import weights_gen as wg
    m = U.make_model(version, seed=0, device="cuda", model_kwargs=kw)[0]
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(3, 120, 160, seed=4)]
    res = m.inference_batch(imgs)
    out = calibrate.fit_camera(res, principal_point=pp, init=init, groups=[0, 0, 0], max_iterations=100)
    again = calibrate.fit_camera(res, principal_point=pp, init=init, groups=[0, 0, 0], max_iterations=100)
    _same(out, again)
    ups = [r["pred_gravity_original"].permute(1, 2, 0).cpu().numpy() for r in res]
    lats = [r["pred_latitude_original"].cpu().numpy() for r in res]
    inits = calibrate._init_from_results(res) if init == "results" else None
    want = ocs.fit_groups(ups, lats, None, [0, 0, 0], pp, None, 100, inits)
    assert len({float(o["pred_rel_focal"]) for o in out if int(o["fit_status"]) != 2}) <= 1
    for o, w in zip(out, want):
        assert (int(o["fit_status"]) == 2) == (w["status"] == 2)
        if w["status"] == 0 and int(o["fit_status"]) == 0:
            assert abs(float(o["fit_cost"]) - w["cost"]) <= 1e-6 * max(w["cost"], 1e-12)


def test_a_group_of_4096_small_images():
    n = 4096
    g = torch.Generator().manual_seed(3)
    roll = (torch.rand(n, generator=g, dtype=torch.float64) * 60 - 30).tolist()
    pitch = (torch.rand(n, generator=g, dtype=torch.float64) * 60 - 30).tolist()
    ups, lats = panocam.camera_fields([0.7] * n, [64] * n, [64] * n, [math.radians(p) for p in pitch], [math.radians(r) for r in roll],
                                      [0.0] * n, [0.0] * n)
    out = calibrate.fit_camera(_as_results(ups, lats), groups=[0] * n, max_iterations=100)
    st = torch.stack([o["fit_status"] for o in out])
    f = torch.stack([o["pred_rel_focal"] for o in out])
    assert (st == 0).all() and (f == f[0]).all() and abs(float(f[0]) - 0.7) < 1e-6
    r = torch.stack([o["pred_roll"] for o in out]).cpu()
    assert (r - torch.tensor(roll, dtype=torch.float64)).abs().max().item() < 1e-4


def _raw(res, group_of, ngroups, n_pad=1, mutate=None, ws_bytes=None):
    """pf_fit_camera_groups on [2, H, W] / [H, W] CUDA fields, outputs inside NaN / -7 prefilled buffers n_pad entries longer."""
    L = _native.lib()
    n = len(res)
    pu = [r["pred_gravity_original"] for r in res]
    pl = [r["pred_latitude_original"] for r in res]
    bu, bl = min(t.data_ptr() for t in pu), min(t.data_ptr() for t in pl)
    descs = (_native.pf_fit_image * n)()
    for i in range(n):
        d = descs[i]
        d.height, d.width = pu[i].shape[1], pu[i].shape[2]
        d.up_offset = (pu[i].data_ptr() - bu) // 4
        d.up_stride[0], d.up_stride[1], d.up_stride[2] = pu[i].stride(1), pu[i].stride(2), pu[i].stride(0)
        d.lat_offset = (pl[i].data_ptr() - bl) // 4
        d.mask_offset = -1
        for k in range(5):
            d.init[k] = math.nan
    gof = (ctypes.c_int32 * n)(*group_of)
    params = torch.full((n + n_pad, 5), math.nan, dtype=torch.float64, device="cuda")
    cost = torch.full((n + n_pad,), math.nan, dtype=torch.float64, device="cuda")
    its = torch.full((n + n_pad,), -7, dtype=torch.int32, device="cuda")
    st = torch.full((n + n_pad,), -7, dtype=torch.int32, device="cuda")
    need = L.pf_fit_camera_groups_workspace(descs, n, gof, ngroups)
    ws = torch.empty(max(need, 256), dtype=torch.uint8, device="cuda")
    args = [0, descs, n, gof, ngroups, bu, bl, None, 1, 0.0, 50, params.data_ptr(), cost.data_ptr(), its.data_ptr(), st.data_ptr(),
            ws.data_ptr(), need if ws_bytes is None else ws_bytes, torch.cuda.current_stream().cuda_stream]
    if mutate:
        mutate(args)
    rc = L.pf_fit_camera_groups(*args)
    torch.cuda.synchronize()
    return rc, need, params, cost, its, st


def test_invalid_arguments_are_rejected_before_any_launch():
    L = _native.lib()
    ups, lats = panocam.camera_fields([0.9, 0.9], [40, 40], [50, 50], [0.2, -0.1], [0.1, 0.3], [0.0, 0.0], [0.0, 0.0])
    res = _as_results(ups, lats)
    rc, need, params, cost, its, st = _raw(res, [0, 0], 1)
    assert rc == 0 and need > 0 and (st[:2] == 0).all() and torch.isnan(params[2:]).all() and (st[2:] == -7).all()
    assert torch.equal(params[0, 2], params[1, 2])
    torch.cuda.synchronize()
    before = L.pf_kernel_launch_count()
    bad = [
        lambda a: a.__setitem__(3, None),                           # no group_of
        lambda a: a.__setitem__(4, 0),                              # ngroups < 1
        lambda a: a.__setitem__(4, 3),                              # group 2 (and 1) empty
        lambda a: a[3].__setitem__(1, 1),                           # group 1 of 1 group: out of range
        lambda a: a[3].__setitem__(0, -1),
        lambda a: a.__setitem__(2, 0),                              # n < 1
        lambda a: a.__setitem__(1, None),                           # no descriptors
        lambda a: a.__setitem__(5, None),                           # no up field
        lambda a: a.__setitem__(6, None),                           # no latitude field
        lambda a: a.__setitem__(8, 2),                              # principal_point not 0 / 1
        lambda a: a.__setitem__(9, -1.0),                           # huber < 0
        lambda a: a.__setitem__(9, math.nan),
        lambda a: a.__setitem__(10, 0),                             # max_iterations outside 1 .. 1000
        lambda a: a.__setitem__(10, 1001),
        lambda a: a.__setitem__(11, None),                          # no params output
        lambda a: a.__setitem__(14, None),                          # no status output
        lambda a: a.__setitem__(15, a[15] + 8),                     # misaligned workspace
        lambda a: setattr(a[1][0], "height", 2),                    # smaller than 3 x 3
        lambda a: setattr(a[1][1], "up_offset", -1),
        lambda a: setattr(a[1][0], "mask_offset", 0),               # a mask offset without a mask
        lambda a: (a[1][0].init.__setitem__(0, 0.1), a[1][0].init.__setitem__(2, 0.0)),     # f_rel <= 0
    ]
    for k, mutate in enumerate(bad):
        rc, _, params, cost, its, st = _raw(res, [0, 0], 1, mutate=mutate)
        assert rc == -1, (k, rc)
        assert torch.isnan(params).all() and torch.isnan(cost).all() and (its == -7).all() and (st == -7).all()
    rc, _, params, *_ = _raw(res, [0, 0], 1, ws_bytes=64)
    assert rc == -4 and torch.isnan(params).all()
    descs = (_native.pf_fit_image * 2)()
    for d in descs:
        d.height, d.width = 40, 50
    for gof, ng in (((0, 2), 2), ((0, 1), 3), ((0, 0), 0)):
        assert L.pf_fit_camera_groups_workspace(descs, 2, (ctypes.c_int32 * 2)(*gof), ng) < 0
    assert L.pf_fit_camera_groups_workspace(descs, 2, None, 1) < 0
    assert L.pf_kernel_launch_count() == before
    for groups in ([0], [0, 1, 2], [True, False], [0, 1.0], [0, "a"], 5, [np.bool_(True), 0], [0, None], torch.tensor([0, 1])):
        with pytest.raises(ValueError):
            calibrate.fit_camera(res, groups=groups)
    with pytest.raises(ValueError):
        calibrate.fit_camera(res, groups=[0, 0], max_iterations=0)
    assert L.pf_kernel_launch_count() == before
