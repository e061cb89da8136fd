"""GPU: the scoring kernels (csrc/metrics.cuh) through metrics.encode_bin / encode_bin_latitude / field_errors / param_errors and
PerspectiveFields.targets_from_fields / losses, against the unmodified reference's outputs (tests/golden/losses.npz) and the
CPU oracle (tests/oracle_metrics.py)."""
import math
import os

import numpy as np
import pytest
import torch

import oracle_metrics as om
import pf_test_util as U
from perspectivefields_b200 import _native, metrics

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "losses.npz"))
REGRESSION = ["Paramnet-360Cities-edina-centered", "Paramnet-360Cities-edina-uncentered", "PersNet_Paramnet-GSV-centered",
              "PersNet_Paramnet-GSV-uncentered"]
CLASSIFICATION = "PersNet-360Cities"
CASE = {(t, n, h, w): name for name, t, n, h, w, _ in om.LOSS_CASES}


def near_bin_boundary(v):
    """Pixels whose float64 angle lies within 1e-4 degrees of a rounding boundary (k + 0.5 bins of 5 degrees)."""
    a = (np.degrees(np.arctan2(v[1].double().cpu().numpy(), v[0].double().cpu().numpy())) + 180.0) % 360.0
    return np.abs((a / 5.0) % 1.0 - 0.5) * 5.0 < 1e-4


def labels_close(got, want, allow):
    got, want = got.cpu().numpy(), want.cpu().numpy()
    d = (got - want) % (om.NUM_BIN - 1)
    off = (got != want) & ~(allow & ((d == 1) | (d == om.NUM_BIN - 2)))
    return int(off.sum())


def test_encoders_match_reference_and_oracle():
    v, _ = om.special_vectors()
    got = metrics.encode_bin(v.cuda(), om.NUM_BIN)
    assert got.dtype == torch.int64 and got.is_cuda and tuple(got.shape) == tuple(v.shape[1:])
    assert labels_close(got, torch.from_numpy(G["enc_special"].astype(np.int64)), near_bin_boundary(v)) == 0
    g = torch.Generator().manual_seed(9)
    up = om.random_up(g, 3, 61, 77).permute(0, 3, 1, 2).contiguous()
    gb = metrics.encode_bin(up.cuda(), om.NUM_BIN)
    want = torch.stack([om.encode_bin(u, om.NUM_BIN) for u in up])
    assert labels_close(gb, want, np.stack([near_bin_boundary(u) for u in up])) == 0
    assert int((gb.cpu() != want).sum()) <= 3
    lat = torch.from_numpy(np.concatenate([om.latitude_boundaries(om.NUM_LAT), np.array([-90.0, 90.0, 0.0, -0.0, -100.0], np.float32)]))
    assert torch.equal(metrics.encode_bin_latitude(lat.view(1, -1).cuda(), om.NUM_LAT).cpu()[0], om.encode_bin_latitude(lat.numpy(), om.NUM_LAT))
    la = om.random_lat_deg(g, 2, 45, 50)
    assert torch.equal(metrics.encode_bin_latitude(la.cuda(), om.NUM_LAT).cpu(), torch.stack([om.encode_bin_latitude(x.numpy(), om.NUM_LAT) for x in la]))


def _model(version, **kw):
    return U.make_model(version, seed=0, device="cuda", model_kwargs=kw)[0]


def _results(pg, pl, rows=True):
    """inference_batch-like results: rows of one buffer (read in place) or separate tensors (stacked once)."""
    if rows:
        g, l = pg.cuda(), pl.cuda()
        return [{"pred_gravity": a, "pred_latitude": b} for a, b in zip(g.unbind(0), l.unbind(0))]
    return [{"pred_gravity": a.cuda().clone(), "pred_latitude": b.cuda().clone()} for a, b in zip(pg, pl)]


LOSS_RUNS = [(v, None, "fp32") for v in REGRESSION + [CLASSIFICATION]] + [(v, (384, 512), "fp32") for v in (REGRESSION[1], CLASSIFICATION)] + \
    [(v, None, "bf16") for v in (REGRESSION[0], CLASSIFICATION)]


@pytest.mark.parametrize("version,resize,precision", LOSS_RUNS)
def test_losses_match_reference_and_oracle(version, resize, precision):
    m = _model(version, resize=resize, precision=precision)
    t = "classification" if version == CLASSIFICATION else "regression"
    h, w = m.net_size()
    n = 3 if (t, 3, h, w) in CASE else 1
    name = CASE[(t, n, h, w)]
    pg, pl, up, lat = om.loss_inputs(t, n, h, w, dict((c[0], c[5]) for c in om.LOSS_CASES)[name])
    tg = m.targets_from_fields([u.cuda() for u in up], [x.cuda() for x in lat])
    og, ol = om.targets(up, lat, t)
    if t == "classification":
        assert torch.equal(tg["gt_latitude"].cpu(), ol)
        assert labels_close(tg["gt_gravity"], og, np.stack([near_bin_boundary(u.permute(2, 0, 1)) for u in up])) == 0
        tg["gt_gravity"] = og.cuda()     # the same targets as the reference's
    else:
        assert torch.equal(tg["gt_gravity"].cpu(), og)
        assert float((tg["gt_latitude"].cpu() - ol).abs().max()) <= 6e-8
    got = m.losses(_results(pg, pl), tg)
    again = m.losses(_results(pg, pl, rows=False), tg)
    want = om.losses(pg, pl, og if t == "regression" else og, ol, t)
    assert list(got) == list(want)
    for k, v in got.items():
        assert v.dim() == 0 and v.dtype == torch.float32 and v.is_cuda
        assert float(v) == pytest.approx(float(G[f"{name}/{k}"]), rel=1e-5), k
        assert float(v) == pytest.approx(want[k], rel=1e-5), k
        assert torch.equal(v, again[k]), k           # bit-identical, whichever way the predictions arrive


def test_losses_edge_cases():
    m = _model(CLASSIFICATION)
    pg, pl, up, lat = om.loss_inputs("classification", 1, 320, 320, 5)
    tg = m.targets_from_fields([up[0].cuda()], [lat[0].cuda()])
    bad = tg["gt_latitude"].clone()
    bad[0, 7, 9] = 180
    out = m.losses(_results(pg, pl), {"gt_gravity": tg["gt_gravity"], "gt_latitude": bad})
    assert math.isnan(float(out["loss_latitude"])) and not math.isnan(float(out["loss_gravity"]))
    bad = tg["gt_gravity"].clone()
    bad[0, 0, 0] = -5
    assert math.isnan(float(m.losses(_results(pg, pl), {"gt_gravity": bad, "gt_latitude": tg["gt_latitude"]})["loss_gravity"]))
    ign = torch.full_like(tg["gt_gravity"], om.IGNORE_GRAVITY)
    assert math.isnan(float(m.losses(_results(pg, pl), {"gt_gravity": ign, "gt_latitude": tg["gt_latitude"]})["loss_gravity"]))
    r = _model(REGRESSION[0])
    pg, pl, up, lat = om.loss_inputs("regression", 1, 320, 320, 5)
    tg = r.targets_from_fields([torch.zeros_like(up[0]).cuda()], [lat[0].cuda()])
    out = r.losses(_results(pg, pl), tg)
    assert math.isnan(float(out["gravity-l2-loss"])) and float(out["gravity-msg-normal-loss"]) == 0.0
    a, b = r.losses(_results(pg, pl), tg), r.losses(_results(pg, pl), tg)
    assert all(torch.equal(a[k].view(1).view(torch.int32), b[k].view(1).view(torch.int32)) for k in a)


@pytest.mark.parametrize("version", [CLASSIFICATION, REGRESSION[1]])
def test_end_to_end_crops_inference_losses(version):
    from oracle import weights_gen as wg
    from perspectivefields_b200 import panocam

    m = _model(version)
    h, w = m.net_size()
    pano = torch.from_numpy(wg.smooth_images(1, 256, 512, seed=4)[0]).cuda()
    views = [(260.0, 0.0, h, w, 10.0 + 40 * i, -15.0 + 12 * i, 8.0 - 5 * i) for i in range(3)]
    crops = panocam.crop_distortion_views(pano, views)
    res = m.inference_batch(crops["im"])
    tg = m.targets_from_fields(crops["up"], crops["lat"], lat_mode="rad")
    got = m.losses(res, tg)
    t = "classification" if version == CLASSIFICATION else "regression"
    pg = torch.stack([r["pred_gravity"] for r in res]).cpu()
    pl = torch.stack([r["pred_latitude"] for r in res]).cpu()
    up = torch.stack([u.cpu() for u in crops["up"]])
    lat = torch.stack([x.cpu() for x in crops["lat"]])
    og, ol = om.targets(up, lat, t, lat_mode="rad")
    if t == "classification":
        assert labels_close(tg["gt_gravity"], og, np.stack([near_bin_boundary(u.permute(2, 0, 1)) for u in up])) == 0
        assert torch.equal(tg["gt_latitude"].cpu(), ol)
        og = tg["gt_gravity"].cpu()
    want = om.losses(pg, pl, og, ol, t)
    for k, v in got.items():
        assert float(v) == pytest.approx(want[k], rel=1e-5), k


def _field_case(seed, sizes):
    g = torch.Generator().manual_seed(seed)
    results, ups, lats = [], [], []
    blob_g = torch.empty(sum(2 * h * w for h, w in sizes)).cuda()
    blob_l = torch.empty(sum(h * w for h, w in sizes)).cuda()
    og = ol = 0
    for h, w in sizes:
        u = om.random_up(g, 1, h, w)[0]
        pu = (u + 0.1 * torch.randn((h, w, 2), generator=g)).permute(2, 0, 1).contiguous()
        pu[:, : h // 7, : w // 5] = 0           # the decoder's "no direction" bin
        la = om.random_lat_deg(g, 1, h, w)[0]
        la[-2:, :3] = float("nan")
        pl = la + torch.randn((h, w), generator=g) * 3
        blob_g[og:og + 2 * h * w] = pu.reshape(-1).cuda()
        blob_l[ol:ol + h * w] = pl.reshape(-1).cuda()
        results.append({"pred_gravity_original": blob_g[og:og + 2 * h * w].view(2, h, w), "pred_latitude_original": blob_l[ol:ol + h * w].view(h, w)})
        og, ol = og + 2 * h * w, ol + h * w
        ups.append(u.cuda())
        lats.append(la.cuda())
    return results, ups, lats


def _check_errors(out, results, ups, lats, thr, lat_mode="deg", masks=None):
    for i, r in enumerate(results):
        mk = None if masks is None or masks[i] is None else masks[i].cpu().numpy()
        ou, ol = om.error_maps(r["pred_gravity_original"].cpu().numpy(), r["pred_latitude_original"].cpu().numpy(), ups[i].cpu().numpy(),
                               lats[i].cpu().numpy(), lat_mode, mk)
        for key, o in (("up", ou), ("latitude", ol)):
            mp = out[key]["map"][i].cpu().numpy()
            assert np.array_equal(np.isnan(mp), np.isnan(o)), (key, i)
            fin = ~np.isnan(o)
            assert np.all(np.abs(mp[fin].astype(np.float64) - o[fin]) <= 1e-4), (key, i)
            c, mean, med, fr = om.stats(mp.astype(np.float64), thr)
            assert int(out[key]["count"][i]) == c
            if c == 0:
                assert math.isnan(float(out[key]["mean"][i])) and math.isnan(float(out[key]["median"][i]))
                continue
            assert float(out[key]["median"][i]) == med, (key, i)
            assert out[key]["fraction"][i].cpu().tolist() == fr, (key, i)
            assert float(out[key]["mean"][i]) == pytest.approx(mean, rel=1e-12), (key, i)


def test_field_errors_mixed_sizes_masks_and_determinism():
    sizes = [(240, 320), (97, 131), (480, 640), (5, 3), (320, 320)]
    results, ups, lats = _field_case(1, sizes)
    ups[3] = torch.zeros_like(ups[3])                   # no valid up pixel
    lats[3] = torch.full_like(lats[3], float("nan"))    # no valid latitude pixel
    thr = (0.5, 1.0, 5.0, 10.0, 30.0, 90.0, 180.0, 1e9)
    out = metrics.field_errors(results, ups, lats, thresholds=thr, return_maps=True)
    _check_errors(out, results, ups, lats, thr)
    again = metrics.field_errors(results, ups, lats, thresholds=thr, return_maps=True)
    for key in ("up", "latitude"):
        for s in ("count", "mean", "median", "fraction"):
            assert torch.equal(out[key][s], again[key][s]) or torch.equal(out[key][s].isnan(), again[key][s].isnan())
        plain = metrics.field_errors(results, ups, lats, thresholds=thr)[key]
        assert torch.equal(plain["count"], out[key]["count"]) and torch.equal(plain["median"].nan_to_num(), out[key]["median"].nan_to_num())
    g = torch.Generator().manual_seed(2)
    masks = [torch.rand(s, generator=g).lt(0.5).cuda() for s in sizes]
    masks[1] = None
    masks[2][:] = False
    out = metrics.field_errors(results, ups, lats, mask=masks, thresholds=(2.0,), return_maps=True)
    _check_errors(out, results, ups, lats, (2.0,), masks=masks)
    rad = [x * (math.pi / 180) for x in lats]
    out = metrics.field_errors(results, ups, rad, lat_mode="rad", return_maps=True)
    _check_errors(out, results, ups, rad, (1.0, 5.0, 10.0), lat_mode="rad")
    empty = metrics.field_errors([], [], [], return_maps=True)
    assert empty["up"]["count"].numel() == 0 and tuple(empty["latitude"]["fraction"].shape) == (0, 3) and empty["up"]["map"] == []


def test_field_errors_on_predictions():
    m = _model(REGRESSION[1])
    from oracle import weights_gen as wg
    from perspectivefields_b200 import panocam
    imgs = [torch.from_numpy(x).cuda() for x in wg.smooth_images(2, 240, 320, seed=1)]
    res = m.inference_batch(imgs)
    ups, lats = panocam.camera_fields([1.1, 0.9], [240, 240], [320, 320], [0.1, -0.2], [0.05, 0.3], [0.0, 0.0], [0.0, 0.0])
    out = metrics.field_errors(res, ups, lats, return_maps=True)
    _check_errors(out, res, ups, lats, (1.0, 5.0, 10.0))
    pe = metrics.param_errors(res, {"roll": [1.0, 2.0], "rel_cx": torch.tensor([0.0, 0.1])})
    assert torch.allclose(pe["roll"].cpu(), (torch.stack([r["pred_roll"] for r in res]).double().cpu() - torch.tensor([1.0, 2.0], dtype=torch.float64)).abs())
    with pytest.raises(ValueError):
        metrics.param_errors(res, {"vfov": [1.0, 2.0]})
    with pytest.raises(ValueError):
        metrics.param_errors([{"pred_gravity": None}], {"roll": [1.0]})


def test_invalid_arguments_raise_before_any_launch():
    L = _native.lib()
    m = _model(CLASSIFICATION)
    pg, pl, up, lat = om.loss_inputs("classification", 1, 320, 320, 5)
    tg = m.targets_from_fields([up[0].cuda()], [lat[0].cuda()])
    torch.cuda.synchronize()
    before = L.pf_kernel_launch_count()
    res = _results(pg, pl)
    torch.cuda.synchronize()
    before = L.pf_kernel_launch_count()
    with pytest.raises(ValueError):
        m.targets_from_fields([up[0][:64].cuda()], [lat[0][:64].cuda()])      # not the working size
    with pytest.raises(TypeError):
        m.targets_from_fields([up[0].double().cuda()], [lat[0].cuda()])
    with pytest.raises(ValueError):
        m.targets_from_fields([up[0]], [lat[0]])                             # on the CPU
    with pytest.raises(ValueError):
        m.losses(res, {"gt_gravity": tg["gt_gravity"].float(), "gt_latitude": tg["gt_latitude"]})
    with pytest.raises(ValueError):
        m.losses([{"pred_gravity": r["pred_gravity"][:, :64], "pred_latitude": r["pred_latitude"]} for r in res], tg)
    with pytest.raises(ValueError):
        _model(CLASSIFICATION, logits=False).losses(res, tg)
    with pytest.raises(ValueError):
        metrics.field_errors([{"pred_gravity_original": up[0].permute(2, 0, 1).cuda(), "pred_latitude_original": lat[0].cuda()}],
                             [up[0].cuda()], [lat[0].cuda()], thresholds=tuple(range(9)))
    with pytest.raises(ValueError):
        metrics.field_errors([{"pred_gravity_original": up[0].permute(2, 0, 1).cuda(), "pred_latitude_original": lat[0].cuda()}],
                             [up[0][:5].cuda()], [lat[0].cuda()])
    with pytest.raises(ValueError):
        metrics.encode_bin(up[0].cuda(), 73)                                 # [H, W, 2] is not [2, H, W]
    with pytest.raises(ValueError):
        metrics.encode_bin_latitude(lat[0], 180)                             # on the CPU
    with pytest.raises(TypeError):
        metrics.encode_bin_latitude(lat[0].double().cuda(), 180)
    assert L.pf_kernel_launch_count() == before
    assert L.pf_head_losses_workspace(1, 320, 320, 73, 1) < 0               # mixed head types
    assert L.pf_field_errors_workspace(None, 1, 0) < 0
