"""GPU: pf_equi_views (PanoCam.crop_equi / get_image, batched) against the oracle restatement (tests/oracle_equi.py) for every
panorama dtype, channel count, sampling mode, output kind and channel order, on batches of mixed sizes spanning two launches with
NaN / 0xA5-prefilled, padded blobs; the Python API against the reference's goldens (tests/golden/equi.npz); the ground-truth
fields; PerspectiveFields.inference_batch on device-resident crops; and argument rejection before any launch."""
import itertools
import os
import warnings

import numpy as np
import pytest
import torch

import oracle_equi as oe
import oracle_pano as op
from perspectivefields_b200 import _native
from perspectivefields_b200 import panocam as pc

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "equi.npz"))
GOLD_PANO = op.make_panorama(*[int(x) for x in GOLD["pano"]])


def _views():
    """30 views (two launches of up to 24) of mixed sizes, with the seam, both poles, roll 180 and ar != W / H."""
    rs = np.random.RandomState(3)
    views = []
    for _ in range(30):
        w, h = int(rs.randint(1, 90)), int(rs.randint(1, 70))
        views.append((float(rs.uniform(20, 120)), w, h, float(rs.uniform(-180, 180)), float(rs.uniform(-60, 60)),
                      float(rs.uniform(-40, 40)), float(rs.choice([w / h, 4 / 3, 0.8]))))
    views[2] = (60.0, 64, 48, 180.0, 0.0, 0.0, 4 / 3)        # across the seam
    views[5] = (50.0, 48, 40, 20.0, 86.0, 5.0, 1.2)          # north pole: rows clamp at 0
    views[9] = (50.0, 48, 40, -70.0, -87.0, -3.0, 1.2)       # south pole: rows clamp at Hp - 1
    views[13] = (70.0, 40, 30, 45.0, 20.0, 180.0, 4 / 3)     # upside down
    views[17] = (90.0, 100, 33, -10.0, 10.0, 0.0, 2.5)       # ar != W / H
    views[25] = (40.0, 128, 96, 100.0, -5.0, 7.0, 4 / 3)     # a larger view: several blocks
    return views


VIEWS = _views()
RAW = op.make_panorama(11, 512, 1024)
PANOS = {("u8", 3): RAW, ("u8", 1): np.ascontiguousarray(RAW[:, :, 2]),
         ("f32", 3): RAW.astype(np.float32) * np.float32(1.0 / 64) - np.float32(1.5)}
PANOS[("f32", 1)] = np.ascontiguousarray(PANOS[("f32", 3)][:, :, 0])


def run_abi(pano, views, mode, unit, swap, pad=True):
    """pf_equi_views through the C ABI into a 0xA5 (uint8) or NaN (float32) prefilled blob with gaps between views.  Returns
    (per-view numpy crops, raw blob as the output dtype, descriptors)."""
    L = _native.lib()
    dev = torch.device("cuda", torch.cuda.current_device())
    f32 = pano.dtype == np.float32
    es, ch = (4 if f32 else 1), (3 if pano.ndim == 3 else 1)
    n = len(views)
    descs = (_native.pf_equi_view * n)()
    off = 0
    for i, (vfov, w, h, az, el, roll, ar) in enumerate(views):
        descs[i] = _native.pf_equi_view(h, w, vfov, az, el, roll, ar, off)
        off += ((ch * h * w * es + 15) // 16 * 16 + 16) if pad else ch * h * w * es + es
    src = torch.from_numpy(pano).to(dev)
    blob = torch.full((off // es,), float("nan"), dtype=torch.float32, device=dev) if f32 else torch.full((off,), 0xA5, dtype=torch.uint8, device=dev)
    _native.check(L.pf_equi_views(dev.index, src.data_ptr(), pano.shape[0], pano.shape[1], ch, _native.PF_EQUI_F32 if f32 else _native.PF_EQUI_U8,
                                  descs, n, {"bilinear": 0, "nearest": 1}[mode], int(unit), int(swap), blob.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream))
    raw = blob.cpu().numpy()
    outs = [raw[d.offset // es:d.offset // es + ch * d.height * d.width].reshape((d.height, d.width, ch) if ch == 3 else (d.height, d.width))
            for d in descs]
    return outs, raw, descs


def compare(g, o, mode, unit, dtype, tag):
    s = o["sample"] if o["im"].ndim == 3 else o["sample"][:, :, 0]
    if mode == "nearest":       # exact away from the half-pixel boundaries, where either neighbour is right
        fu, fv = np.abs((o["u"] % 1) - 0.5), np.abs((o["v"] % 1) - 0.5)
        ok = (fu > 1e-6) & (fv > 1e-6)
        ok = ok[:, :, None] if g.ndim == 3 else ok
        ok = np.broadcast_to(ok, g.shape)
        assert np.array_equal(g[ok], o["im"][ok]), tag
        return
    if dtype == np.float32:
        assert (np.abs(g.astype(np.float64) - s) <= np.spacing(np.abs(s).astype(np.float32)).astype(np.float64)).all(), tag
        return
    pre = s.astype(np.float32).astype(np.float64) * 255 if unit else s
    strict = np.abs(pre - np.round(pre)) >= 1e-3
    d = np.abs(g.astype(np.int32) - o["im"].astype(np.int32))
    assert (d[strict] == 0).all() and d.max() <= 1, tag


COMBOS = [(dt, ch, mode, unit, swap) for dt, ch, mode, unit, swap in itertools.product(("u8", "f32"), (1, 3), ("bilinear", "nearest"), (False, True), (False, True))
          if not (unit and dt == "f32") and not (swap and ch == 1)]


@pytest.mark.parametrize("dt,ch,mode,unit,swap", COMBOS)
def test_abi_matches_oracle(dt, ch, mode, unit, swap):
    pano = PANOS[(dt, ch)]
    outs, raw, descs = run_abi(pano, VIEWS, mode, unit, swap)
    for i, (g, view) in enumerate(zip(outs, VIEWS)):
        o = oe.crop_equi_full(pano, *view, mode=mode, unit=unit, swap_rb=swap)
        assert g.shape == o["im"].shape
        compare(g, o, mode, unit, pano.dtype, (i, view))
    es = 4 if dt == "f32" else 1
    written = np.zeros(raw.size, bool)
    for d in descs:
        written[d.offset // es:d.offset // es + ch * d.height * d.width] = True
    assert (np.isnan(raw[~written]) if dt == "f32" else raw[~written] == 0xA5).all()      # the padding is never written


def test_unaligned_offsets_take_the_same_values():
    for dt in ("u8", "f32"):
        pano = PANOS[(dt, 3)]
        a, _, _ = run_abi(pano, VIEWS, "bilinear", False, False, pad=True)
        b, raw, descs = run_abi(pano, VIEWS, "bilinear", False, False, pad=False)
        assert any(d.offset % 16 for d in descs)
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), dt


def test_crop_equi_and_get_image_match_reference_goldens(tmp_path):
    gray = np.ascontiguousarray(GOLD_PANO[:, :, 1])
    f32 = GOLD_PANO.astype(np.float32) * np.float32(1.0 / 64) - np.float32(1.5)
    for i, c in enumerate(GOLD["crop_cases"]):
        view = (c[0], int(c[1]), int(c[2]), c[3], c[4], c[5], c[6])
        for key, img, mode in (("u8", GOLD_PANO, "bilinear"), ("gray", gray, "bilinear"), ("f32", f32, "bilinear"), ("near", GOLD_PANO, "nearest")):
            got = pc.PanoCam.crop_equi(img, *view, mode)
            assert got.is_cuda and got.dtype == (torch.float32 if img.dtype == np.float32 else torch.uint8)
            assert tuple(got.shape) == ((view[2], view[1], 3) if img.ndim == 3 else (view[2], view[1]))
            o = oe.crop_equi_full(img, *view, mode=mode)
            compare(got.cpu().numpy(), o, mode, False, img.dtype, (key, i))
            compare(GOLD[f"{key}{i}"].reshape(got.shape), o, mode, False, img.dtype, ("golden", key, i))
    from PIL import Image
    path = tmp_path / "pano.png"
    Image.fromarray(GOLD_PANO).save(path)
    cam = pc.PanoCam(str(path))
    for k, c in enumerate(GOLD["image_cases"]):
        view = (c[0], int(c[1]), int(c[2]), c[3], c[4], c[5], c[6])
        for fmt in ("RGB", "BGR"):
            crop, horizon, vvp = cam.get_image(*view, img_format=fmt)
            assert crop.is_cuda and crop.dtype == torch.uint8 and tuple(crop.shape) == (view[2], view[1], 3)
            o = oe.crop_equi_full(GOLD_PANO, *view, unit=True, swap_rb=fmt == "BGR")
            compare(crop.cpu().numpy(), o, "bilinear", True, np.uint8, (fmt, k))
            compare(GOLD[f"image_{fmt}{k}"], o, "bilinear", True, np.uint8, ("golden", fmt, k))
            assert list(horizon) == GOLD[f"image_horizon{k}"].tolist() and list(vvp) == GOLD[f"image_vvp{k}"].tolist()
    # the defaults of get_image
    crop, horizon, vvp = cam.get_image()
    assert tuple(crop.shape) == (480, 640, 3) and len(vvp) == 3


def test_batched_api_fields_horizon_and_blob():
    views = [(70.0, 64, 48, 30.0, 20.0, 0.0, 4 / 3), {"vfov": 60.0, "im_w": 33, "im_h": 17, "azimuth": -50.0, "elevation": 0.0, "roll": 10.0, "ar": 2.0},
             (80.0, 48, 64, 100.0, -35.0, 180.0, 0.75)]
    r = pc.crop_equi_views(torch.from_numpy(GOLD_PANO).cuda(), views, outputs=("up", "lat"), img_format="BGR")
    assert set(r) == {"im", "up", "lat", "horizon", "vvp"}
    rad = lambda x: x / 180 * np.pi
    for (vfov, w, h, az, el, roll, ar), im, up, lat in zip([pc._check_equi_view(v, 0) for v in views], r["im"], r["up"], r["lat"]):
        assert torch.equal(up, pc.PanoCam.get_up(rad(vfov), w, h, rad(el), rad(roll)))
        assert torch.equal(lat, pc.PanoCam.get_lat(rad(vfov), w, h, rad(el), rad(roll)))
        assert torch.equal(im, pc.PanoCam.crop_equi(GOLD_PANO, vfov, w, h, az, el, roll, ar, "bilinear").flip(2))
        assert im.data_ptr() % 16 == 0
    base = r["im"][0].untyped_storage().data_ptr()
    assert all(im.untyped_storage().data_ptr() == base for im in r["im"])         # one blob
    assert r["horizon"].shape == (3, 2) and r["vvp"].shape == (3, 3)
    assert np.isinf(r["vvp"][1, :2]).all() and np.isnan(r["vvp"][1, 2])           # elevation 0: the reference's (inf, inf)
    h, v = pc.horizon_vvp(80.0, 48, 64, -35.0, 180.0)
    assert r["horizon"][2].tolist() == list(h) and r["vvp"][2].tolist() == list(v)


@pytest.mark.parametrize("version", ["Paramnet-360Cities-edina-centered", "PersNet-360Cities"])
def test_inference_on_device_crops_equals_host(version):
    import pf_test_util as U
    model, _ = U.make_model(version, seed=1, device="cuda")
    r = pc.crop_equi_views(GOLD_PANO, [(60.0, 320, 240, 20.0, 5.0, 3.0, 4 / 3), (75.0, 300, 200, -70.0, -12.0, 0.0, 1.5)],
                           outputs=(), img_format="BGR")
    dev_out = model.inference_batch(r["im"])
    host_out = model.inference_batch([c.cpu().numpy() for c in r["im"]])
    for d, h in zip(dev_out, host_out):
        assert list(d) == list(h)
        for k in d:
            assert torch.equal(d[k], h[k]) if isinstance(d[k], torch.Tensor) else d[k] == h[k], k


def test_invalid_inputs_raise_before_launch():
    L = _native.lib()
    pano = torch.zeros((8, 16, 3), dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 12, dtype=torch.uint8, device="cuda")
    before = L.pf_kernel_launch_count()
    good = _native.pf_equi_view(4, 4, 60.0, 0.0, 0.0, 0.0, 1.0, 0)

    def call(view=good, h=8, w=16, ch=3, dt=0, mode=0, kind=0, swap=0, p=pano.data_ptr(), o=out.data_ptr(), n=1):
        arr = (_native.pf_equi_view * 1)(view)
        return L.pf_equi_views(0, p, h, w, ch, dt, arr, n, mode, kind, swap, o, None)

    bad = [dict(view=_native.pf_equi_view(0, 4, 60.0, 0, 0, 0, 1.0, 0)), dict(view=_native.pf_equi_view(4, 4, 0.0, 0, 0, 0, 1.0, 0)),
           dict(view=_native.pf_equi_view(4, 4, 180.0, 0, 0, 0, 1.0, 0)), dict(view=_native.pf_equi_view(4, 4, 60.0, float("nan"), 0, 0, 1.0, 0)),
           dict(view=_native.pf_equi_view(4, 4, 60.0, 0, 0, float("inf"), 1.0, 0)), dict(view=_native.pf_equi_view(4, 4, 60.0, 0, 0, 0, 0.0, 0)),
           dict(view=_native.pf_equi_view(4, 4, 170.0, 0, 0, 0, 1e20, 0)), dict(view=_native.pf_equi_view(4, 4, 60.0, 0, 0, 0, 1.0, -16)),
           dict(view=_native.pf_equi_view(4, 4, 60.0, 0, 0, 0, 1.0, 2), dt=1), dict(h=0), dict(ch=2), dict(dt=2), dict(mode=2), dict(kind=2),
           dict(kind=1, dt=1), dict(swap=1, ch=1), dict(swap=2), dict(p=None), dict(o=None), dict(n=0)]
    for kw in bad:
        assert call(**kw) == -1, kw
    np_pano = np.zeros((8, 16, 3), np.uint8)
    for args, exc in (((np_pano.astype(np.float64), [(60.0, 4, 4, 0, 0, 0, 1.0)]), TypeError), ((np_pano, [(60.0, 4, 4, 0, float("nan"), 0, 1.0)]), ValueError),
                      ((np_pano, []), ValueError), ((pano, [(60.0, 4, 4, 0, 0, 0, 1.0)], ("up",), "bilinear", "RGB", "cuda:1"), ValueError)):
        with pytest.raises(exc):
            pc.crop_equi_views(*args)
    with pytest.raises(ValueError):
        pc.PanoCam.crop_equi(np_pano, 60.0, 4, 4, 0, 0, 0, 1.0, "bicubic")
    assert L.pf_kernel_launch_count() == before
    assert call() == 0
