"""GPU: the camera-track fit (csrc/calib.cuh, fit_seq_step_kernel) through calibrate.fit_camera(groups=..., smoothness=...) and
pf_fit_camera_sequences, against the sequence CPU oracle (tests/oracle_calib_sequence.py), the per-image fit, a banded oracle
on a long sequence and inference_batch results read in place."""
import ctypes
import math

import numpy as np
import pytest
import torch

import oracle_calib as oc
import oracle_calib_sequence as oseq
import pf_test_util as U
from perspectivefields_b200 import _native, calibrate, panocam

pytestmark = pytest.mark.gpu

KEYS = ("pred_roll", "pred_pitch", "pred_rel_focal", "pred_rel_cx", "pred_rel_cy")
SCALE = np.array([180 / math.pi, 180 / math.pi, 1.0, 1.0, 1.0])


def _as_results(ups, lats):
    return [{"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l} for u, l in zip(ups, lats)]


def _params(o):
    return np.array([float(o[k]) for k in KEYS])


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert list(x) == list(y)
        for k in x:
            assert torch.equal(x[k], y[k]) or (torch.isnan(x[k]) and torch.isnan(y[k])), k


def _case(seed=7, principal_point=True, weighted=False):
    """Two interleaved sequences (4 and 3 frames) of jittered slow tracks, noisy fields, masks and optional weight maps."""
    rng = np.random.default_rng(seed)
    seqs = [((math.log(0.9), 0.05, -0.03), (48, 64), (0.3, -0.2)), ((math.log(1.3), -0.06, 0.02), (45, 60), (-0.4, 0.3))]
    lens = [4, 3]
    ups, lats, masks, wts, groups = [], [], [], [], []
    for gid, ((s, cx, cy), (h, w), (r0, e0)) in enumerate(seqs):
        for t in range(lens[gid]):
            cam = (r0 + 0.02 * t + math.radians(1.0) * rng.standard_normal(), e0 - 0.015 * t + math.radians(1.0) * rng.standard_normal(), s)
            cam = cam + ((cx, cy) if principal_point else (0.0, 0.0))
            u, l = oc.noisy_fields(rng, cam, h, w)
            ups.append(u)
            lats.append(l)
            masks.append(rng.random((h, w)) > 0.15)
            wu = rng.uniform(0.1, 2.0, (h, w)).astype(np.float32)
            wl = rng.uniform(0.1, 2.0, (h, w)).astype(np.float32)
            wu[rng.random((h, w)) < 0.05] = 0.0
            wts.append((wu, wl))
            groups.append(gid)
    masks[1] = None
    order = [0, 4, 1, 5, 2, 6, 3]   # interleaved, each sequence in frame order
    pick = lambda v: [v[i] for i in order]
    return pick(ups), pick(lats), pick(masks), (pick(wts) if weighted else None), pick(groups)


def _cuda(ups, lats, masks, wts):
    res = _as_results([torch.from_numpy(u).cuda() for u in ups], [torch.from_numpy(l).cuda() for l in lats])
    mk = [None if m is None else torch.from_numpy(m).cuda() for m in masks]
    w = None if wts is None else [tuple(torch.from_numpy(x).cuda() for x in p) for p in wts]
    return res, mk, w


@pytest.mark.parametrize("principal_point", [False, True])
@pytest.mark.parametrize("huber", [None, math.radians(2.5)])
@pytest.mark.parametrize("weighted", [False, True])
def test_against_the_sequence_oracle(principal_point, huber, weighted):
    ups, lats, masks, wts, groups = _case(7, principal_point, weighted)
    res, mk, w = _cuda(ups, lats, masks, wts)
    sigma = (0.7, 0.4)
    kw = dict(principal_point=principal_point, mask=mk, huber=huber, groups=groups, weights=w, smoothness=sigma)
    # the start (one evaluation), then one and two steps of the joint solve against the oracle's direct one
    for its in (1, 2, 3):
        early = calibrate.fit_camera(res, max_iterations=its, **kw)
        want0 = oseq.fit_sequences(ups, lats, masks, groups, sigma, principal_point, huber, its, weights=wts)
        for i, (o, x) in enumerate(zip(early, want0)):
            assert int(o["fit_status"]) == x["status"] == 1 and int(o["fit_iterations"]) == x["iterations"] == its, (its, i)
            assert np.max(np.abs(_params(o) - x["params"])) < 1e-9, (its, i, _params(o), x["params"])
            assert abs(float(o["fit_cost"]) - x["cost"]) <= 1e-9 * x["cost"], (its, i)
    out = calibrate.fit_camera(res, max_iterations=300, **kw)
    want = oseq.fit_sequences(ups, lats, masks, groups, sigma, principal_point, huber, 300, weights=wts)
    for i, (o, x) in enumerate(zip(out, want)):
        assert int(o["fit_status"]) == x["status"] == 0, i
        got = _params(o)
        assert np.all(np.abs(got - x["params"]) <= 1e-7 * SCALE * np.maximum(1.0, np.abs(x["theta"]))), (i, got, x["params"])
        assert abs(float(o["fit_cost"]) - x["cost"]) <= 1e-9 * x["cost"], (i, float(o["fit_cost"]), x["cost"])
    for gid in set(groups):
        mem = [i for i, g in enumerate(groups) if g == gid]
        for k in ("pred_rel_focal", "pred_rel_cx", "pred_rel_cy"):
            assert all(torch.equal(out[i][k], out[mem[0]][k]) for i in mem)
        assert len({int(out[i]["fit_iterations"]) for i in mem}) == 1


def test_labels_layouts_and_repeats_are_bit_identical():
    ups, lats, masks, _, groups = _case(13)
    res, mk, _ = _cuda(ups, lats, masks, None)
    kw = dict(principal_point=True, huber=math.radians(2.5), smoothness=0.5)
    a = calibrate.fit_camera(res, groups=groups, mask=mk, **kw)
    _same(a, calibrate.fit_camera(res, groups=groups, mask=mk, **kw))
    _same(a, calibrate.fit_camera(res, groups=[7 if g == 0 else -3 for g in groups], mask=mk, **kw))
    _same(a, calibrate.fit_camera(res, groups=[np.int64(g + 100) for g in groups], mask=mk, **kw))
    order = sorted(range(len(res)), key=lambda i: groups[i])
    c = calibrate.fit_camera([res[i] for i in order], groups=[groups[i] for i in order], mask=[mk[i] for i in order], **kw)
    _same([a[i] for i in order], c)


@pytest.mark.parametrize("principal_point", [False, True])
def test_one_frame_sequences_are_the_per_image_fit(principal_point):
    ups, lats, masks, _, _ = _case(11, principal_point)
    res, mk, _ = _cuda(ups, lats, masks, None)
    n = len(res)
    a = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, max_iterations=300)
    b = calibrate.fit_camera(res, principal_point=principal_point, mask=mk, max_iterations=300, groups=range(n), smoothness=1.0)
    for i, (x, y) in enumerate(zip(a, b)):
        assert int(x["fit_status"]) == int(y["fit_status"]) == 0
        assert np.all(np.abs(_params(x) - _params(y)) <= 1e-7 * SCALE * np.maximum(1.0, np.abs(_params(x)))), i
        assert abs(float(x["fit_cost"]) - float(y["fit_cost"])) <= 1e-9 * float(x["fit_cost"])


def test_a_frame_without_data_is_interpolated():
    m = 5
    rolls, pitches = [4.0, 5.0, 6.0, 7.0, 8.0], [-3.0, -2.5, -2.0, -1.5, -1.0]
    ups, lats = panocam.camera_fields([0.9] * m, [48] * m, [64] * m, [math.radians(p) for p in pitches], [math.radians(r) for r in rolls],
                                      [0.0] * m, [0.0] * m)
    mk = [None] * m
    mk[2] = torch.zeros((48, 64), dtype=torch.bool, device="cuda")
    out = calibrate.fit_camera(_as_results(ups, lats), mask=mk, groups=[0] * m, smoothness=0.5, max_iterations=300)
    assert all(int(o["fit_status"]) == 0 for o in out)
    assert float(out[2]["fit_cost"]) == 0.0
    for k in ("pred_roll", "pred_pitch"):
        assert abs(float(out[2][k]) - 0.5 * (float(out[1][k]) + float(out[3][k]))) < 1e-7
    dead = calibrate.fit_camera(_as_results(ups[:2], lats[:2]), mask=[mk[2], mk[2]], groups=[0, 0], smoothness=0.5)
    assert all(int(o["fit_status"]) == 2 and int(o["fit_iterations"]) == 1 and math.isnan(float(o["pred_roll"])) for o in dead)


def test_a_sequence_of_4096_small_frames_matches_the_banded_oracle():
    n = 4096
    t = np.arange(n)
    roll = 10.0 * np.sin(2 * np.pi * t / 900.0) + np.random.default_rng(3).normal(0.0, 1.0, n)
    pitch = 6.0 * np.cos(2 * np.pi * t / 1300.0) + np.random.default_rng(4).normal(0.0, 1.0, n)
    ups, lats = panocam.camera_fields([0.7] * n, [32] * n, [32] * n, np.radians(pitch).tolist(), np.radians(roll).tolist(), [0.0] * n, [0.0] * n)
    out = calibrate.fit_camera(_as_results(ups, lats), groups=[0] * n, smoothness=0.3, max_iterations=100)
    got = np.array([[float(o["pred_roll"]), float(o["pred_pitch"]), float(o["pred_rel_focal"])] for o in out])
    st = {int(o["fit_status"]) for o in out}
    want = oseq.fit_sequences([u.cpu().numpy() for u in ups], [l.cpu().numpy() for l in lats], None, [0] * n, 0.3, False, None, 100)
    assert st == {want[0]["status"]} == {0}
    ref = np.array([w["params"][:3] for w in want])
    assert np.max(np.abs(got[:, :2] - ref[:, :2])) < 1e-6 and np.max(np.abs(got[:, 2] - ref[:, 2])) < 1e-8


@pytest.mark.parametrize("pp", [False, True])
def test_inference_results_in_place(pp):
    from oracle import weights_gen as wg
    m = U.make_model("PersNet-360Cities", seed=0, device="cuda")[0]
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(3, 120, 160, seed=4)]
    res = m.inference_batch(imgs)
    kw = dict(principal_point=pp, groups=[0, 0, 0], smoothness=0.5, max_iterations=100)
    out = calibrate.fit_camera(res, **kw)
    _same(out, calibrate.fit_camera(res, **kw))
    ups = [r["pred_gravity_original"].permute(1, 2, 0).cpu().numpy() for r in res]
    lats = [r["pred_latitude_original"].cpu().numpy() for r in res]
    want = oseq.fit_sequences(ups, lats, None, [0, 0, 0], 0.5, pp, None, 100)
    for i, (o, w) in enumerate(zip(out, want)):
        assert int(o["fit_status"]) == w["status"] == 0, (i, int(o["fit_status"]), w["status"])
        got = _params(o)
        assert np.all(np.abs(got - w["params"]) <= 1e-7 * SCALE * np.maximum(1.0, np.abs(w["theta"]))), (i, got, w["params"])
        assert abs(float(o["fit_cost"]) - w["cost"]) <= 1e-9 * max(w["cost"], 1e-12), (i, float(o["fit_cost"]), w["cost"])


def _raw(res, group_of, nseq, mutate=None, ws_bytes=None):
    """pf_fit_camera_sequences on [2, H, W] / [H, W] CUDA fields, outputs in NaN / -7 prefilled buffers one entry longer."""
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
    params = torch.full((n + 1, 5), math.nan, dtype=torch.float64, device="cuda")
    cost = torch.full((n + 1,), math.nan, dtype=torch.float64, device="cuda")
    its = torch.full((n + 1,), -7, dtype=torch.int32, device="cuda")
    st = torch.full((n + 1,), -7, dtype=torch.int32, device="cuda")
    need = L.pf_fit_camera_sequences_workspace(descs, n, gof, nseq)
    ws = torch.empty(max(need, 256), dtype=torch.uint8, device="cuda")
    args = [0, descs, n, gof, nseq, bu, bl, None, None, None, None, 1, 0.0, 50, 0.5, 0.5, params.data_ptr(), cost.data_ptr(),
            its.data_ptr(), st.data_ptr(), ws.data_ptr(), need if ws_bytes is None else ws_bytes, torch.cuda.current_stream().cuda_stream]
    if mutate:
        mutate(args)
    rc = L.pf_fit_camera_sequences(*args)
    torch.cuda.synchronize()
    return rc, need, params, cost, its, st


def test_invalid_arguments_are_rejected_before_any_launch():
    L = _native.lib()
    ups, lats = panocam.camera_fields([0.9, 0.9], [40, 40], [50, 50], [0.2, -0.1], [0.1, 0.3], [0.0, 0.0], [0.0, 0.0])
    res = _as_results(ups, lats)
    rc, need, params, cost, its, st = _raw(res, [0, 0], 1)
    assert rc == 0 and need > 0 and (st[:2] == 0).all() and torch.isnan(params[2:]).all() and (st[2:] == -7).all()
    torch.cuda.synchronize()
    before = L.pf_kernel_launch_count()
    bad = [
        lambda a: a.__setitem__(3, None),                           # no group_of
        lambda a: a.__setitem__(4, 0),                              # nseq < 1
        lambda a: a.__setitem__(4, 3),                              # sequences 1 and 2 empty
        lambda a: a[3].__setitem__(0, -1),
        lambda a: a.__setitem__(2, 0),                              # n < 1
        lambda a: a.__setitem__(5, None),                           # no up field
        lambda a: a.__setitem__(11, 2),                             # principal_point not 0 / 1
        lambda a: a.__setitem__(12, -1.0),                          # huber < 0
        lambda a: a.__setitem__(13, 0),                             # max_iterations outside 1 .. 1000
        lambda a: a.__setitem__(14, 0.0),                           # sigma_roll <= 0
        lambda a: a.__setitem__(15, -1.0),
        lambda a: a.__setitem__(14, math.nan),
        lambda a: a.__setitem__(15, math.inf),
        lambda a: a.__setitem__(16, None),                          # no params output
        lambda a: a.__setitem__(20, a[20] + 8),                     # misaligned workspace
        lambda a: setattr(a[1][0], "height", 2),                    # smaller than 3 x 3
    ]
    for k, mutate in enumerate(bad):
        rc, _, params, cost, its, st = _raw(res, [0, 0], 1, mutate=mutate)
        assert rc == -1, (k, rc)
        assert torch.isnan(params).all() and torch.isnan(cost).all() and (its == -7).all() and (st == -7).all()
    rc, _, params, *_ = _raw(res, [0, 0], 1, ws_bytes=64)
    assert rc == -4 and torch.isnan(params).all()
    assert L.pf_kernel_launch_count() == before
    for sm in (0.0, -1.0, math.nan, math.inf, True, (1.0,), (1.0, 2.0, 3.0), (1.0, 0.0), "a", (1.0, None)):
        with pytest.raises(ValueError):
            calibrate.fit_camera(res, groups=[0, 0], smoothness=sm)
    with pytest.raises(ValueError):
        calibrate.fit_camera(res, smoothness=1.0)                   # no groups
    assert L.pf_kernel_launch_count() == before
