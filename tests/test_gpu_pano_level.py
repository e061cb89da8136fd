"""GPU: panorama levelling (csrc/calib.cuh fit_pano_*_kernel, csrc/equi.cuh rotate_panoramas_kernel) through
calibrate.fit_panorama, rectify.rotate_panoramas and rectify.level_panoramas, against tests/oracle_pano_level.py, exact fields of
the views' effective cameras, the crop rule and the product's own calls."""
import math

import numpy as np
import pytest
import torch

import oracle_calib as oc
import oracle_pano_level as opl
import pf_test_util as U
from perspectivefields_b200 import _native, calibrate, panocam, rectify

pytestmark = pytest.mark.gpu

# (vfov, im_w, im_h, azimuth, elevation, roll, ar): mixed sizes and aspect ratios, elevations of +-30 degrees
VIEWS = [(70.0, 64, 48, 0.0, 0.0, 0.0, 64 / 48), (60.0, 40, 60, 90.0, 30.0, 5.0, 0.8), (80.0, 56, 56, 200.0, -30.0, -10.0, 1.0),
         (65.0, 72, 48, 300.0, 10.0, 0.0, 1.2)]
TILTS = [(0.0, 0.0), (5.0, -3.0), (-12.0, 20.0), (25.0, 8.0)]


def _rot(axis, deg):
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    a = math.radians(deg)
    return np.eye(3) + math.sin(a) * K + (1.0 - math.cos(a)) * K @ K


def _rotations():
    rng = np.random.default_rng(5)
    out = [np.eye(3), _rot((1, 0, 0), 90), _rot((0, 1, 0), 90), _rot((0, 0, 1), 90)]
    for _ in range(2):
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        out.append(q * np.sign(np.linalg.det(q)))
    return out


def smooth_pano(h, w, channels=3, dtype=np.uint8, seed=0):
    """A panorama that is a smooth function of the direction (no seam at the wrap or the poles)."""
    rng = np.random.default_rng(seed)
    j, i = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    th, ph = 2 * np.pi * j / w - np.pi, np.pi / 2 - np.pi * i / h
    d = np.stack([np.cos(ph) * np.sin(th), -np.sin(ph), np.cos(ph) * np.cos(th)])
    planes = []
    for _ in range(channels):
        a = rng.standard_normal((3, 3))
        planes.append(127.5 + 60 * np.sin(np.einsum("k,khw->hw", a[0] * 2, d) + a[1, 0]) + 50 * np.cos(np.einsum("k,khw->hw", a[2] * 3, d)))
    p = np.stack(planes, axis=2)
    p = np.clip(np.rint(p), 0, 255) if dtype == np.uint8 else p
    p = p.astype(dtype)
    return p[:, :, 0] if channels == 1 else p


def _effective_fields(views, T):
    """Exact fields of each view's effective camera T A_k, as fit results: oracle_calib's float64 model (the ground truth
    get_up_general / get_lat_general draw) rounded to float32."""
    res = []
    for vfov, w, h, az, el, roll, ar in views:
        A = opl.crop_rotation(az, el, roll)
        _, e2, r2 = opl.decompose(T @ A)
        u, l = oc.model((math.radians(r2), math.radians(e2), math.log(opl.crop_focal(vfov, w, ar) / h)), h, w)
        up = torch.from_numpy((u / np.linalg.norm(u, axis=2, keepdims=True)).astype(np.float32)).cuda()
        res.append({"pred_gravity_original": up.permute(2, 0, 1), "pred_latitude_original": torch.from_numpy(np.degrees(l).astype(np.float32)).cuda()})
    return res


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
def test_warp_against_the_oracle(dtype, channels, mode):
    rots = _rotations()
    for (h, w), seed in (((97, 194), 1), ((50, 100), 2)):
        rng = np.random.default_rng(seed)
        pano = rng.integers(0, 256, (h, w, channels)).astype(dtype) if dtype == np.uint8 else rng.uniform(0, 255, (h, w, channels)).astype(dtype)
        pano = pano[:, :, 0] if channels == 1 else pano
        out = rectify.rotate_panoramas([torch.from_numpy(pano).cuda()] * len(rots), rots, mode=mode, outputs=("map",))
        for R, got, gmap in zip(rots, out["im"], out["map"]):
            want, _, u, v = opl.rotate(pano, R, mode)
            got, gmap = got.cpu().numpy(), gmap.cpu().numpy().astype(np.float64)
            diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
            if mode == "nearest":
                near = lambda t: np.abs((t + 0.5) - np.rint(t + 0.5)) < 1e-6
                tie = near(u) | near(v)
                bad = diff.reshape(h, w, -1).max(axis=2) > 0
                assert not np.any(bad & ~tie), (h, w, R, np.argwhere(bad & ~tie)[:5])
            elif dtype == np.uint8:
                # rounding ties: quarter turns about y on an even width land on half pixels, where the last bits of the weights
                # decide which way a sample of x.5 rounds
                s = opl.rotate(pano, R, mode)[1].reshape(diff.shape)
                tie = np.abs(s - np.floor(s) - 0.5) < 1e-6
                assert diff.max() <= 1 and np.mean((diff > 0) & ~tie) < 0.01, (h, w, R, diff.max(), np.mean((diff > 0) & ~tie))
            else:
                assert diff.max() <= 1.0 and np.mean(diff > 1e-3) < 0.01, (h, w, R, diff.max())
            if np.array_equal(R, np.eye(3)):   # the identity keeps every row below the pole
                assert np.array_equal(got[1:], pano[1:])
            du = np.abs(np.mod(gmap[..., 0] - u + w / 2, w) - w / 2)
            assert du.max() <= 1e-4 and np.abs(gmap[..., 1] - v).max() <= 1e-4, (h, w, R, np.argwhere(du > 1e-4)[:8])


def test_crop_composition():
    pano = smooth_pano(256, 512)
    R = _rotations()[4]
    rot = rectify.rotate_panoramas([torch.from_numpy(pano).cuda()], [R])["im"][0]
    for view in [(60.0, 96, 64, 30.0, 0.0, 0.0, 1.5), (50.0, 64, 64, 250.0, 10.0, 5.0, 1.0)]:
        vfov, w, h, az, el, roll, ar = view
        a2, e2, r2 = opl.decompose(R @ opl.crop_rotation(az, el, roll))
        if abs(e2) > 40:
            continue
        a = panocam.crop_equi_views(rot, [view], outputs=())["im"][0].cpu().numpy().astype(int)
        b = panocam.crop_equi_views(pano, [(vfov, w, h, a2, e2, r2, ar)], outputs=())["im"][0].cpu().numpy().astype(int)
        assert np.abs(a - b).max() <= 2, (view, np.abs(a - b).max())


def test_recovery_from_exact_fields():
    results, views, pano_of = [], [], []
    for P, (psi, phi) in enumerate(TILTS):
        results += _effective_fields(VIEWS, opl.tilt(math.radians(psi), math.radians(phi)))
        views += VIEWS
        pano_of += [P] * len(VIEWS)
    fits = calibrate.fit_panorama(results, views, pano_of, max_iterations=100)
    for (psi, phi), f in zip(TILTS, fits):
        assert int(f["fit_status"]) == 0
        assert abs(float(f["pano_roll"]) - psi) < 1e-7 and abs(float(f["pano_pitch"]) - phi) < 1e-7, (psi, phi, float(f["pano_roll"]), float(f["pano_pitch"]))
        g = f["pano_up"].cpu().numpy()
        R = f["rotation"].cpu().numpy()
        assert np.allclose(R @ opl.N, g, atol=1e-14) and np.allclose(R @ R.T, np.eye(3), atol=1e-14)


def _noisy_case(rng, tilt):
    T = opl.tilt(math.radians(tilt[0]), math.radians(tilt[1]))
    ups, lats, masks, wts, oviews = [], [], [], [], []
    for vfov, w, h, az, el, roll, ar in VIEWS:
        A = opl.crop_rotation(az, el, roll)
        F = opl.crop_focal(vfov, w, ar)
        _, e2, r2 = opl.decompose(T @ A)
        up, lat = oc.noisy_fields(rng, (math.radians(r2), math.radians(e2), math.log(F / h)), h, w)
        m = rng.random((h, w)) > 0.1
        wt = (rng.uniform(0.0, 1.0, (h, w)).astype(np.float32), rng.uniform(0.1, 1.0, (h, w)).astype(np.float32))
        ups.append(up); lats.append(lat); masks.append(m); wts.append(wt)
        oviews.append({"A": A, "F": F, "up": up, "lat": lat, "mask": m, "weights": wt})
    return ups, lats, masks, wts, oviews


@pytest.mark.parametrize("huber", [None, math.radians(2.0)])
@pytest.mark.parametrize("max_iterations", [1, 3, 100])
def test_fit_against_the_oracle(huber, max_iterations):
    rng = np.random.default_rng(11)
    results, views, pano_of, masks, weights, wants = [], [], [], [], [], []
    for P, tilt in enumerate([(-12.0, 20.0), (25.0, 8.0)]):
        ups, lats, ms, wts, oviews = _noisy_case(rng, tilt)
        results += [{"pred_gravity_original": torch.from_numpy(u).cuda().permute(2, 0, 1), "pred_latitude_original": torch.from_numpy(l).cuda()}
                    for u, l in zip(ups, lats)]
        masks += [torch.from_numpy(m).cuda() for m in ms]
        weights += [tuple(torch.from_numpy(t).cuda() for t in wt) for wt in wts]
        views += VIEWS
        pano_of += [P] * len(VIEWS)
        wants.append(opl.fit(oviews, huber=huber, max_iterations=max_iterations))
    fits = calibrate.fit_panorama(results, views, pano_of, mask=masks, weights=weights, huber=huber, max_iterations=max_iterations)
    for f, w in zip(fits, wants):
        # a converged fit's last accept / reject decisions compare costs that agree to the last bits only, so the number of
        # evaluations is compared where the cap stops both
        assert int(f["fit_status"]) == w["status"]
        assert w["status"] == 0 or int(f["fit_iterations"]) == w["iterations"]
        got = np.array([float(f["pano_roll"]), float(f["pano_pitch"])])
        assert np.all(np.abs(got - w["angles"]) <= 1e-9 * np.maximum(1.0, np.abs(w["angles"]))), (got, w["angles"])
        assert abs(float(f["fit_cost"]) - w["cost"]) <= 1e-9 * w["cost"]
        assert np.allclose(f["rotation"].cpu().numpy(), w["rotation"], atol=1e-9)


def test_round_trip():
    pano = smooth_pano(256, 512, seed=3)
    Q = _rot((math.cos(0.5), 0.0, math.sin(0.5)), 14.0)      # a tilt about a horizontal axis: levelling it needs no yaw
    tilted = rectify.rotate_panoramas([torch.from_numpy(pano).cuda()], [Q])["im"][0]
    views = list(rectify.DEFAULT_LEVEL_VIEWS)
    fits = calibrate.fit_panorama(_effective_fields(views, Q), views, [0] * len(views))
    assert int(fits[0]["fit_status"]) == 0
    R = fits[0]["rotation"].cpu().numpy()
    assert np.allclose(R, Q.T, atol=1e-9)
    level = rectify.rotate_panoramas([tilted], [fits[0]["rotation"]])["im"][0].cpu().numpy().astype(int)
    diff = np.abs(level - pano.astype(int))[32:-32]
    assert diff.max() <= 4 and diff.mean() < 0.5, (diff.max(), diff.mean())


def test_status_2_leaves_the_other_panoramas_alone():
    good = _effective_fields(VIEWS, opl.tilt(math.radians(5.0), math.radians(-3.0)))
    bad = [{k: torch.full_like(v, math.nan) for k, v in r.items()} for r in good]
    both = calibrate.fit_panorama(bad + good, VIEWS * 2, [0] * 4 + [1] * 4)
    alone = calibrate.fit_panorama(good, VIEWS, [0] * 4)
    assert int(both[0]["fit_status"]) == 2
    for k in ("pano_roll", "pano_pitch", "pano_up", "rotation", "fit_cost"):
        assert torch.isnan(both[0][k]).all()
    for k in both[1]:
        assert torch.equal(both[1][k], alone[0][k]), k


def test_deterministic_and_no_synchronisation():
    rng = np.random.default_rng(4)
    ups, lats, ms, wts, _ = _noisy_case(rng, (-12.0, 20.0))
    results = [{"pred_gravity_original": torch.from_numpy(u).cuda().permute(2, 0, 1), "pred_latitude_original": torch.from_numpy(l).cuda()}
               for u, l in zip(ups, lats)]
    masks = [torch.from_numpy(m).cuda() for m in ms]
    pano = torch.from_numpy(smooth_pano(97, 194)).cuda()
    calibrate.fit_panorama(results, VIEWS, [0] * 4, mask=masks)       # load the library and warm up outside the sync check
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        runs = []
        for _ in range(2):
            f = calibrate.fit_panorama(results, VIEWS, [0] * 4, mask=masks, huber=0.03)
            r = rectify.rotate_panoramas([pano, pano], torch.stack([f[0]["rotation"], f[0]["rotation"].t().contiguous()]), outputs=("map",))
            runs.append((f, r))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    (f1, r1), (f2, r2) = runs
    for k in f1[0]:
        assert torch.equal(f1[0][k], f2[0][k]), k
    for a, b in zip(r1["im"] + r1["map"], r2["im"] + r2["map"]):
        assert torch.equal(a, b)


def test_pipeline_is_the_four_calls():
    model, _ = U.make_model("Paramnet-360Cities-edina-uncentered", seed=0, device="cuda:0")
    panos = [torch.from_numpy(smooth_pano(128, 256, seed=s)).cuda() for s in (6, 7)]
    views = [(70.0, 320, 320, float(az), 0.0, 0.0, 1.0) for az in range(0, 360, 90)]
    got = rectify.level_panoramas(model, panos, views=views)
    crops = [c for p in panos for c in panocam.crop_equi_views(p, views, outputs=())["im"]]
    fits = calibrate.fit_panorama(model.inference_batch(crops), views * 2, [0] * 4 + [1] * 4)
    want = rectify.rotate_panoramas(panos, [f["rotation"] for f in fits])
    for a, b in zip(got["fits"], fits):
        for k in a:
            assert torch.equal(a[k], b[k]) or (torch.isnan(a[k]).all() and torch.isnan(b[k]).all()), k
    for a, b in zip(got["im"], want["im"]):
        assert torch.equal(a, b)


def test_invalid_arguments_raise_before_any_launch():
    L = _native.lib()
    good = _effective_fields(VIEWS[:1], np.eye(3))
    pano = torch.zeros((50, 100, 3), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = L.pf_kernel_launch_count()
    cases = [
        lambda: calibrate.fit_panorama(good, VIEWS[:1], [1]),                       # panorama 0 has no view
        lambda: calibrate.fit_panorama(good, VIEWS[1:2], [0]),                      # view size differs from the fields
        lambda: calibrate.fit_panorama(good, VIEWS[:1], [0], huber=-1.0),
        lambda: calibrate.fit_panorama(good, VIEWS[:1], [0], max_iterations=0),
        lambda: calibrate.fit_panorama(good, VIEWS[:1], [0], init=[(0.0,)]),
        lambda: calibrate.fit_panorama(good, [(190.0,) + VIEWS[0][1:]], [0]),       # vfov outside (0, 180)
        lambda: rectify.rotate_panoramas([pano], [np.diag([1.0, 1.0, 2.0])]),        # not a rotation
        lambda: rectify.rotate_panoramas([pano], [np.eye(3)], mode="cubic"),
        lambda: rectify.rotate_panoramas([pano], [np.eye(3)] * 2),
        lambda: rectify.rotate_panoramas([pano[:1]], [np.eye(3)]),                 # 1 row
        lambda: rectify.rotate_panoramas([pano, pano.float()], [np.eye(3)] * 2),
        lambda: rectify.rotate_panoramas([pano], torch.eye(3, device="cuda")[None].float()),
    ]
    for c in cases:
        with pytest.raises((ValueError, TypeError)):
            c()
    assert L.pf_kernel_launch_count() == before
