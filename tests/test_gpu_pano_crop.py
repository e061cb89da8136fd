"""GPU: pf_pano_views (PanoCam.crop_distortion, batched) against the oracle restatement (tests/oracle_pano.py) on the golden cases
and on a batch of random views of mixed sizes spanning several launches; NaN-prefilled outputs; skipped outputs; the Python
API; and PerspectiveFields.inference_batch on device-resident crops."""
import os
import warnings

import numpy as np
import pytest
import torch

import oracle_pano as op
from perspectivefields_b200 import _native
from perspectivefields_b200 import panocam as pc

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "pano.npz"))
GOLD_PANO = op.make_panorama(*[int(x) for x in GOLD["pano"]])
GOLD_CASES = [tuple(c) for c in GOLD["cases"]]
FIELDS = ("ntheta", "nphi", "up", "lat", "xy_map")


def oracle(pano, view):
    f, xi, h, w, az, el, roll = view
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return op.crop_distortion_full(pano, f, xi, int(h), int(w), az, el, roll)


def run_abi(pano, views, skip=(), pad=True):
    """pf_pano_views through the C ABI with NaN-prefilled field blobs and a 0xA5-prefilled crop blob.  Returns (per-view dicts of
    numpy arrays, the raw blobs, descriptors)."""
    L = _native.lib()
    dev = torch.device("cuda", torch.cuda.current_device())
    n = len(views)
    descs = (_native.pf_pano_view * n)()
    im_off = fld_off = 0
    for i, (f, xi, h, w, az, el, roll) in enumerate(views):
        h, w = int(h), int(w)
        descs[i] = _native.pf_pano_view(h, w, f, xi, az, el, roll, im_off, fld_off)
        im_off += ((3 * h * w + 15) // 16 * 16 + 16) if pad else 3 * h * w      # padded: aligned, with a gap after every view
        fld_off += ((h * w + 3) // 4 * 4 + 4) if pad else h * w
    src = torch.from_numpy(np.ascontiguousarray(pano)).to(dev)
    im = torch.full((im_off,), 0xA5, dtype=torch.uint8, device=dev)
    blobs = {k: torch.full(((2 if k in ("up", "xy_map") else 1) * fld_off,), float("nan"), dtype=torch.float32, device=dev) for k in FIELDS}
    offset = torch.full((n,), -7.0, dtype=torch.float64, device=dev)
    status = torch.full((n,), -7, dtype=torch.int32, device=dev)
    ptr = lambda k: None if k in skip else blobs[k].data_ptr()
    _native.check(L.pf_pano_views(dev.index, src.data_ptr(), pano.shape[0], pano.shape[1], descs, n, None if "im" in skip else im.data_ptr(),
                                  ptr("ntheta"), ptr("nphi"), ptr("up"), ptr("lat"), ptr("xy_map"), offset.data_ptr(), status.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    raw = {"im": im.cpu().numpy(), "offset": offset.cpu().numpy(), "status": status.cpu().numpy()}
    raw.update({k: v.cpu().numpy() for k, v in blobs.items()})
    outs = []
    for i, d in enumerate(descs):
        h, w = d.height, d.width
        o = {"im": raw["im"][d.im_offset:d.im_offset + 3 * h * w].reshape(h, w, 3), "offset": raw["offset"][i], "status": raw["status"][i]}
        for k in FIELDS:
            c = 2 if k in ("up", "xy_map") else 1
            o[k] = raw[k][c * d.field_offset:c * (d.field_offset + h * w)].reshape((h, w, 2) if c == 2 else (h, w))
        outs.append(o)
    return outs, raw, descs


def compare(g, o, tag, fields=FIELDS, stats=None):
    for k in ("ntheta", "nphi", "lat"):
        if k in fields:
            assert np.abs(g[k] - o[k]).max() <= 1e-6, (tag, k)
    if "xy_map" in fields:
        ulp = np.spacing(np.abs(o["xy_map"]).astype(np.float32)).astype(np.float64)
        assert (np.abs(g["xy_map"] - o["xy_map"]) <= ulp + 1e-9).all(), tag
    if "up" in fields:
        big, zero = o["up_len"] >= 1e-6, o["up_len"] == 0
        assert np.abs(g["up"] - o["up"])[big].max(initial=0.0) <= 2e-6, tag
        assert (g["up"][zero] == 0).all(), tag
        if stats is not None:
            stats.append((o["up_len"] < 1e-6).sum() / o["up_len"].size)
    s = o["sample"]
    strict = np.abs(s - np.round(s)) >= 1e-3
    if o["mask"] is not None:
        strict |= ~o["mask"][:, :, None]
    d = np.abs(g["im"].astype(np.int32) - o["im"].astype(np.int32))
    assert (d[strict] == 0).all() and d.max() <= 1, tag
    assert int(g["status"]) == o["status"], tag
    if np.isnan(o["offset"]):
        assert np.isnan(g["offset"]), tag
    else:
        assert abs(g["offset"] - o["offset"]) <= 1e-6, tag


def test_golden_cases_match_oracle():
    outs, _, _ = run_abi(GOLD_PANO, GOLD_CASES)
    stats = []
    for i, (g, view) in enumerate(zip(outs, GOLD_CASES)):
        o = oracle(GOLD_PANO, view)
        compare(g, o, i, stats=stats)
        if GOLD["raises"][i]:
            assert int(g["status"]) == op.STATUS_ASSERT
    print("fraction of pixels whose unnormalised up vector is below 1e-6 px, per golden case:", [round(float(x), 4) for x in stats])


def test_random_views_mixed_sizes_several_launches():
    rs = np.random.RandomState(5)
    pano = op.make_panorama(11, 512, 1024)
    views = []
    for i in range(55):                                     # 5 launches of up to 12 views
        h, w = int(rs.randint(1, 70)), int(rs.randint(1, 90))
        xi = float(rs.choice([0.0, 0.5, 0.9, 1.2, 1.4]))
        views.append((float(rs.uniform(8, 60)), xi, h, w, float(rs.uniform(-180, 180)), float(rs.uniform(-89, 89)), float(rs.uniform(-40, 40))))
    views[3] = (300.0, 0.0, 240, 320, 0.0, 0.0, 0.0)        # level camera, even H
    views[7] = (250.0, 0.9, 241, 321, 170.0, -5.0, 2.0)     # odd size, across the seam
    views[20] = (30.0, 0.0, 24, 32, 15.0, 10.0, 180.0)      # upside down
    for pad in (True, False):
        outs, _, _ = run_abi(pano, views, pad=pad)
        for i, (g, view) in enumerate(zip(outs, views)):
            compare(g, oracle(pano, view), (pad, i))
    assert int(outs[20]["status"]) == op.STATUS_ASSERT and int(outs[3]["status"]) == op.STATUS_MULTI


def test_skipped_outputs_are_never_written():
    views = GOLD_CASES[:5] + [(60.0, 0.2, 50, 70, 33.0, -20.0, 4.0)]
    full, _, _ = run_abi(GOLD_PANO, views)
    part, raw, descs = run_abi(GOLD_PANO, views, skip=("ntheta", "nphi", "xy_map"))
    for k in ("ntheta", "nphi", "xy_map"):
        assert np.isnan(raw[k]).all(), k                      # prefilled NaN untouched
    for g, f in zip(part, full):
        assert np.array_equal(g["im"], f["im"]) and np.array_equal(g["up"], f["up"], equal_nan=True) and np.array_equal(g["lat"], f["lat"])
    # the padding between views is never written either
    written = np.zeros(raw["im"].size, bool)
    fw = np.zeros(raw["lat"].size, bool)
    for d in descs:
        written[d.im_offset:d.im_offset + 3 * d.height * d.width] = True
        fw[d.field_offset:d.field_offset + d.height * d.width] = True
    assert (raw["im"][~written] == 0xA5).all() and np.isnan(raw["lat"][~fw]).all() and not np.isnan(raw["lat"][fw]).any()
    fw2 = np.repeat(fw, 2)
    assert np.isnan(raw["up"][~fw2]).all() and not np.isnan(raw["up"][fw2]).any()
    # only the crop
    only_im, raw2, _ = run_abi(GOLD_PANO, views, skip=FIELDS)
    assert all(np.isnan(raw2[k]).all() for k in FIELDS)
    assert all(np.array_equal(g["im"], f["im"]) for g, f in zip(only_im, full))


def test_abi_rejects_bad_arguments_before_launch():
    L = _native.lib()
    pano = torch.zeros((8, 16, 3), dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 12, dtype=torch.float32, device="cuda")
    before = L.pf_kernel_launch_count()

    def call(view, h=8, w=16, p=pano.data_ptr(), o=out.data_ptr()):
        arr = (_native.pf_pano_view * 1)(view)
        return L.pf_pano_views(0, p, h, w, arr, 1, None, None, None, None, o, None, None, None, None)

    assert call(_native.pf_pano_view(0, 4, 10.0, 0.0, 0, 0, 0, 0, 0)) == -1
    assert call(_native.pf_pano_view(4, 4, 0.0, 0.0, 0, 0, 0, 0, 0)) == -1
    assert call(_native.pf_pano_view(4, 4, 10.0, float("nan"), 0, 0, 0, 0, 0)) == -1
    assert call(_native.pf_pano_view(4, 4, 10.0, 0.0, 0, 0, 0, 0, -4)) == -1
    assert call(_native.pf_pano_view(4, 4, 10.0, 0.0, 0, 0, 0, 0, 0), h=1) == -1
    assert call(_native.pf_pano_view(4, 4, 10.0, 0.0, 0, 0, 0, 0, 0), p=None) == -1
    assert call(_native.pf_pano_view(4, 4, 10.0, 0.0, 0, 0, 0, 0, 0), o=None) == -1
    assert L.pf_kernel_launch_count() == before
    assert call(_native.pf_pano_view(4, 4, 10.0, 0.0, 0, 0, 0, 0, 0)) == 0


def test_python_api(capsys, tmp_path):
    view = (40.0, 0.5, 48, 64, 30.0, 10.0, 5.0)
    o = oracle(GOLD_PANO, view)
    im, ntheta, nphi, offset, up, lat, xy = pc.PanoCam.crop_distortion(GOLD_PANO, *view)
    assert im.is_cuda and im.dtype == torch.uint8 and tuple(im.shape) == (48, 64, 3) and isinstance(offset, float)
    assert up.dtype == torch.float32 and tuple(up.shape) == (48, 64, 2) and tuple(xy.shape) == (48, 64, 2)
    g = {"im": im.cpu().numpy(), "ntheta": ntheta.cpu().numpy(), "nphi": nphi.cpu().numpy(), "lat": lat.cpu().numpy(), "up": up.cpu().numpy(),
         "xy_map": xy.cpu().numpy(), "offset": offset, "status": o["status"]}
    compare(g, o, "single")
    # a CUDA panorama and a path give the same crop
    dev_pano = torch.from_numpy(GOLD_PANO).cuda()
    assert torch.equal(pc.PanoCam.crop_distortion(dev_pano, *view)[0], im)
    from PIL import Image
    Image.fromarray(GOLD_PANO).save(tmp_path / "pano.png")
    assert torch.equal(pc.PanoCam.crop_distortion(str(tmp_path / "pano.png"), *view)[0], im)
    # the reference's warning and assertion
    pc.PanoCam.crop_distortion(GOLD_PANO, 30.0, 0.0, 32, 48, 0.0, 0.0, 0.0)
    assert "WARNING | Number of zero crossings: 2" in capsys.readouterr().out
    with pytest.raises(AssertionError):
        pc.PanoCam.crop_distortion(GOLD_PANO, 30.0, 0.0, 24, 32, 0.0, 0.0, 180.0)
    # batched form: selected outputs only, device offset / status
    r = pc.crop_distortion_views(dev_pano, [view, (30.0, 0.0, 24, 32, 0.0, 0.0, 180.0)], outputs=("up", "lat"))
    assert set(r) == {"im", "up", "lat", "offset", "status"}
    assert r["offset"].is_cuda and r["status"].tolist() == [o["status"], op.STATUS_ASSERT]
    assert torch.equal(r["im"][0], im) and torch.equal(r["up"][0], up) and torch.equal(r["lat"][0], lat)


@pytest.mark.parametrize("version,kw", [("Paramnet-360Cities-edina-centered", {}), ("PersNet-360Cities", {}),
                                        ("Paramnet-360Cities-edina-uncentered", {"resize": (320, 448)})])
def test_inference_on_device_crops_equals_host(version, kw):
    import pf_test_util as U
    model, _ = U.make_model(version, seed=1, device="cuda", model_kwargs=kw)
    r = pc.crop_distortion_views(GOLD_PANO, [(200.0, 0.0, 240, 320, 20.0, 5.0, 3.0), (150.0, 0.9, 200, 300, -70.0, -12.0, 0.0),
                                            (250.0, 0.3, 256, 256, 170.0, 30.0, -10.0)], outputs=())
    crops = r["im"]
    dev_out = model.inference_batch(crops)
    host_out = model.inference_batch([c.cpu().numpy() for c in crops])
    for d, h in zip(dev_out, host_out):
        assert list(d) == list(h)
        for k in d:
            if isinstance(d[k], torch.Tensor):
                assert torch.equal(d[k], h[k]), k
            else:
                assert d[k] == h[k], k
    single = model.inference(crops[0])
    assert all(torch.equal(single[k], dev_out[0][k]) for k in single if isinstance(single[k], torch.Tensor))
    # RGB input format flips the channels as the host path does
    model.input_format = "RGB"
    try:
        d, h = model.inference(crops[1]), model.inference(crops[1].cpu().numpy())
        assert all(torch.equal(d[k], h[k]) for k in d if isinstance(d[k], torch.Tensor))
    finally:
        model.input_format = "BGR"
    with pytest.raises(TypeError):
        model.inference_batch([crops[0], crops[1].cpu().numpy()])
    with pytest.raises(TypeError):
        model.inference_batch([crops[0].float()])
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            model.inference_batch([crops[0].to("cuda:1")])
