"""GPU: the whole inference path through the product API (which calls libpf_b200.so through its C ABI) against the CPU
oracle on the same synthetic checkpoint and images, and against the golden fixtures made by the unmodified reference.

Tolerance (BASELINE.json north_star): 1e-3 relative fp32, metric = max|a - b| / max|b| per returned tensor.  The synthetic
gravity head emits vectors with |v| well away from 0 (oracle/weights_gen.py), so the normalised field is compared
directly.  argmax-decoded fields of the classification variant are compared only where the top-2 logit margin exceeds
the logit error bound (argmax is discontinuous)."""
import numpy as np
import pytest
import torch

import pf_test_util as U
from golden_util import compare_with_golden, golden_images
from oracle import model as om
from oracle import weights_gen as wg

pytestmark = pytest.mark.gpu
TOL = 1e-3

_models = {}


def model(version):
    if version not in _models:
        _models[version] = U.make_model(version)
    return _models[version]


def _check(out, ora, version, skip=()):
    worst = {}
    assert len(out) == len(ora)
    for o, r in zip(out, ora):
        assert list(o.keys()) == list(r.keys())
        for k, v in r.items():
            if isinstance(v, str):
                assert o[k] == v
                continue
            assert tuple(o[k].shape) == tuple(v.shape) and o[k].dtype == torch.float32, k
            if k in skip:
                continue
            if k == "pred_latitude_original" and v.abs().max() > 75:
                # degrees = asin(sin_lat): asin is not Lipschitz at +-1 (d/dx = 1/sqrt(1-x^2)), where the regression head
                # clamps; compare in the sine domain everywhere and in degrees away from the poles.
                a, b = o[k].detach().cpu().double(), v.double()
                e = U.rel_err(torch.sin(torch.deg2rad(a)), torch.sin(torch.deg2rad(b)))
                far = b.abs() < 75
                if far.any():
                    e = max(e, ((a - b).abs()[far].max() / b.abs().max()).item())
            else:
                e = U.rel_err(o[k], v)
            worst[k] = max(worst.get(k, 0.0), e)
            assert e < TOL, (version, k, e)
    return worst


@pytest.mark.parametrize("version", ["Paramnet-360Cities-edina-centered", "Paramnet-360Cities-edina-uncentered",
                                     "PersNet_Paramnet-GSV-uncentered", "PersNet_Paramnet-GSV-centered"])
def test_regression_variants_match_oracle_and_golden(version):
    m, sd = model(version)
    imgs = golden_images()
    out = m.inference_batch(imgs)
    assert all(o["pred_gravity"].is_cuda for o in out)
    print(version, _check(out, om.inference_batch(sd, version, imgs), version))
    print(version, "golden", compare_with_golden(version, out, tol=TOL, check_stats=True))


def _check_decoded_fields(out, ora, tag):
    """pred_gravity_original / pred_latitude_original of the classification variant: argmax is discontinuous in the logits, so
    the decoded fields are compared on the pixels whose four bilinear source taps all have an unambiguous argmax in the oracle
    (top-2 margin > 4 x the measured logit error; tests/pf_test_util.py:stable_mask) -- there at the usual 1e-3."""
    for i, (o, r) in enumerate(zip(out, ora)):
        h, w = r["pred_latitude_original"].shape
        for key, okey, scale in (("pred_gravity", "pred_gravity_original", 1.0), ("pred_latitude", "pred_latitude_original", 90.0)):
            err = (o[key].cpu() - r[key]).abs().max().item()
            stable320 = U.stable_mask(r[key], err)
            assert stable320.float().mean() > 0.9
            assert torch.equal(o[key].cpu().argmax(0)[stable320], r[key].argmax(0)[stable320])
            stable = U.stable_mask(r[key], err, h, w)
            frac = stable.float().mean().item()
            assert frac > 0.8, (tag, okey, frac)
            a, b = o[okey].cpu(), r[okey]
            d = (a - b).abs()
            d = d.amax(0) if d.ndim == 3 else d
            e = d[stable].max().item() / scale
            assert e < TOL, (tag, i, okey, e, frac)


def test_classification_variant():
    version = "PersNet-360Cities"
    m, sd = model(version)
    imgs = golden_images()
    out = m.inference_batch(imgs)
    ora = om.inference_batch(sd, version, imgs)
    print(_check(out, ora, version, skip=("pred_gravity_original", "pred_latitude_original")))
    compare_with_golden(version, out, tol=TOL, skip_keys=("pred_gravity_original", "pred_latitude_original"))
    _check_decoded_fields(out, ora, "default")
    for o in out:
        assert o["pred_latitude_original_mode"] == "deg"


def test_classification_decode_only_mode():
    """SURVEY 8f-3 / option "decode_only" (PerspectiveFields(version, logits=False)): logits are never written; the decoded 320x320
    fields equal the decode of the default path's logits bit for bit, and the *_original outputs are identical."""
    version = "PersNet-360Cities"
    m, sd = model(version)
    imgs = golden_images()
    base = m.inference_batch(imgs)
    m2, _ = U.make_model(version, model_kwargs={"logits": False})
    out = m2.inference_batch(imgs)
    for o, r in zip(out, base):
        assert list(o.keys()) == list(r.keys())
        assert tuple(o["pred_gravity"].shape) == (2, 320, 320) and tuple(o["pred_latitude"].shape) == (1, 320, 320)
        idx_g, idx_l = r["pred_gravity"].argmax(0).cpu(), r["pred_latitude"].argmax(0).cpu()
        assert (o["pred_gravity"].cpu() - om.decode_bin(idx_g, 73)).abs().max() < 2e-6
        assert torch.equal(o["pred_latitude"].cpu()[0], om.decode_bin_latitude(idx_l, 180))
        assert torch.equal(o["pred_gravity_original"], r["pred_gravity_original"])
        assert torch.equal(o["pred_latitude_original"], r["pred_latitude_original"])
    with pytest.raises(ValueError):
        from perspectivefields_b200 import PerspectiveFields
        PerspectiveFields("Paramnet-360Cities-edina-centered", logits=False)


def test_every_layer_tap_matches_oracle():
    version = "Paramnet-360Cities-edina-centered"
    m, sd = model(version)
    imgs = golden_images()
    m.debug_taps(True)
    try:
        m.inference_batch(imgs)
        taps = m.read_taps()
    finally:
        m.debug_taps(False)
    otaps = {}
    om.inference_batch(sd, version, imgs, otaps)
    checked = 0
    for name, t in taps.items():
        if name.startswith("mit."):
            ref = otaps[name]
        elif name == "ll" or name.startswith("cnx.s"):
            ref = otaps[name].permute(0, 2, 3, 1)
        elif name in ("head.raw_g", "head.raw_l"):
            ref = otaps["g.raw" if name.endswith("_g") else "l.raw"]          # NCHW, pre-normalise / pre-clamp 1x1 conv output
        elif name.startswith("head."):
            k = name[5:]
            ref = torch.cat([otaps["g." + k], otaps["l." + k]], 1).permute(0, 2, 3, 1)
        else:
            continue
        e = U.rel_err(t, ref.contiguous().reshape(-1))
        assert e < TOL, (name, e)
        checked += 1
    assert checked > 72 and "head.raw_g" in taps and "head.raw_l" in taps


def test_mixed_sizes_identity_upscale_and_batch_invariance():
    version = "Paramnet-360Cities-edina-uncentered"
    m, sd = model(version)
    imgs = [wg.synth_images(1, 320, 320, 5)[0], wg.smooth_images(1, 33, 47, 6)[0], wg.smooth_images(1, 768, 1024, 7)[0],
            wg.synth_images(1, 240, 320, 8)[0]]
    keep = [im.copy() for im in imgs]
    out = m.inference_batch(imgs)
    assert all(np.array_equal(a, b) for a, b in zip(imgs, keep))  # inputs are not modified
    _check(out, om.inference_batch(sd, version, imgs), version)
    for i, im in enumerate(imgs):
        assert out[i]["pred_gravity_original"].shape == (2,) + im.shape[:2]
        assert out[i]["pred_latitude_original"].shape == im.shape[:2]
        single = m.inference(im)   # inference == inference_batch([x])[0]; sharding/batching never changes an image's result
        for k, v in single.items():
            if not isinstance(v, str):
                assert torch.equal(v, out[i][k]), (i, k)
    # a 320x320 input passes through the resize unchanged and the post-process resample is the identity
    assert torch.allclose(out[0]["pred_latitude_original"], torch.rad2deg(torch.asin(out[0]["pred_latitude"][0])), rtol=1e-6, atol=1e-5)
    assert torch.allclose(out[0]["pred_gravity_original"], out[0]["pred_gravity"], rtol=1e-6, atol=1e-6)


def test_forward_entry_with_preresized_float_images():
    version = "Paramnet-360Cities-edina-centered"
    m, sd = model(version)
    imgs = golden_images()
    inputs = [{"image": om.preprocess(im), "height": im.shape[0], "width": im.shape[1]} for im in imgs]
    a = m.forward(inputs)
    b = m.inference_batch(imgs)
    for x, y in zip(a, b):
        for k, v in x.items():
            if not isinstance(v, str):
                assert torch.equal(v, y[k]), k


def test_full_size_batch_properties():
    """BASELINE config C2 shape (batch 32, 640x480): size-independent properties + spot parity."""
    version = "Paramnet-360Cities-edina-centered"
    m, sd = model(version)
    imgs = wg.synth_images(32, 480, 640, 11)
    out = m.inference_batch(imgs)
    g = torch.stack([o["pred_gravity"] for o in out])
    go = torch.stack([o["pred_gravity_original"] for o in out])
    lat = torch.stack([o["pred_latitude"] for o in out])
    lo = torch.stack([o["pred_latitude_original"] for o in out])
    assert torch.isfinite(g).all() and torch.isfinite(go).all() and torch.isfinite(lo).all()
    assert (g.norm(dim=1) - 1).abs().max() < 1e-5 and (go.norm(dim=1) - 1).abs().max() < 1e-5
    assert lat.abs().max() <= 1 and lo.abs().max() <= 90.0001
    for i in (0, 17, 31):  # batch position never changes an image's result (what multi-GPU sharding relies on)
        single = m.inference(imgs[i])
        for k, v in single.items():
            if not isinstance(v, str):
                assert torch.equal(v, out[i][k]), (i, k)
    _check([out[5]], om.inference_batch(sd, version, [imgs[5]]), version)


def test_kernel_launches_are_counted():
    from perspectivefields_b200 import _native

    m, _ = model("Paramnet-360Cities-edina-uncentered")
    before = _native.lib().pf_kernel_launch_count()
    m.inference(wg.synth_images(1, 64, 64, 1)[0])
    assert _native.lib().pf_kernel_launch_count() - before > 300


OPTION_DEFAULTS = {"pdl": 1, "decode_only": 0, "bf16": 0}    # include/pf_b200.h


@pytest.mark.parametrize("opts", [{"pdl": 0}])
def test_engine_options_end_to_end(opts):
    """The same forward without programmatic dependent launch.  "pdl" only changes how the same kernels are scheduled: the
    outputs equal the default run's exactly.  Each option is restored to the value it had, so that later tests see the model
    as it was."""
    version = "Paramnet-360Cities-edina-centered"
    m, _ = model(version)
    imgs = golden_images()
    base = m.inference_batch(imgs)
    prev = {k: m._options.get(k, OPTION_DEFAULTS[k]) for k in opts}
    for k, v in opts.items():
        m.set_option(k, v)
    try:
        out = m.inference_batch(imgs)
    finally:
        for k, v in prev.items():
            m.set_option(k, v)
    for a, b in zip(out, base):
        for k, v in a.items():
            assert torch.equal(v, b[k]) if isinstance(v, torch.Tensor) else v == b[k], k


def test_unknown_engine_options_are_rejected():
    """pf_set_option knows "pdl", "decode_only" and "bf16"; any other name is an error and leaves the model as it was."""
    from perspectivefields_b200 import _native

    m, _ = model("Paramnet-360Cities-edina-centered")
    before = dict(m._options)
    for name in ("fork", "dw_ln", "attn_mma", "attn_split", "stem_tc", "phase_conv1"):
        for value in (0, 1):
            with pytest.raises(_native.PfError, match="unknown option"):
                m.set_option(name, value)
    assert m._options == before


def test_resolution_sweep_large_image_properties_and_parity():
    """BASELINE config C5 shape class: 2048x1536 and 1024x768 inputs (only the pre/post-processing bytes change)."""
    version = "PersNet_Paramnet-GSV-uncentered"
    m, sd = model(version)
    imgs = [wg.smooth_images(1, 1536, 2048, 21)[0], wg.synth_images(1, 768, 1024, 22)[0]]
    out = m.inference_batch(imgs)
    _check(out, om.inference_batch(sd, version, imgs), version)
    assert out[0]["pred_gravity_original"].shape == (2, 1536, 2048) and out[1]["pred_latitude_original"].shape == (768, 1024)
    assert (out[0]["pred_gravity_original"].norm(dim=0) - 1).abs().max() < 1e-5


def test_c3_shape_512x512_batch():
    """BASELINE config C3 shape: 512x512 inputs, uncentered ParamNet (64x64 nearest sub-sample), batch 8 here."""
    version = "Paramnet-360Cities-edina-uncentered"
    m, sd = model(version)
    imgs = wg.synth_images(8, 512, 512, 31)
    out = m.inference_batch(imgs)
    _check([out[3]], om.inference_batch(sd, version, [imgs[3]]), version)
    for o in out:
        assert torch.isfinite(o["pred_rel_focal"]) and o["pred_rel_focal"] > 0


def test_weight_driven_gravity_field_second_seed():
    """SURVEY.md 7.4-1: the default synthetic gravity head has a dominant bias (a near-constant normalised field).  Here the bias is
    zero and the 1x1 conv's gain is 10x larger: the up-vector turns through all directions, so the comparison exercises the
    weight-driven part; pixels where |v_raw| is small (F.normalize amplifies any error by 1/|v|) are masked."""
    version = "Paramnet-360Cities-edina-centered"
    m, sd = U.make_model(version, seed=1, gravity_bias=(0.0, 0.0), gravity_gain=0.8)
    imgs = [wg.smooth_images(1, 360, 500, 41)[0], wg.synth_images(1, 480, 640, 42)[0]]
    m.debug_taps(True)
    try:
        out = m.inference_batch(imgs)
        taps = m.read_taps()
    finally:
        m.debug_taps(False)
    otaps = {}
    ora = om.inference_batch(sd, version, imgs, otaps)
    raw = otaps["g.raw"]                                   # [n, 2, 320, 320] before F.normalize
    e_raw = U.rel_err(taps["head.raw_g"], raw.reshape(-1))
    assert e_raw < TOL, e_raw
    assert U.rel_err(taps["head.raw_l"], otaps["l.raw"].reshape(-1)) < TOL
    nrm = raw.norm(dim=1)
    ang = torch.atan2(raw[:, 1], raw[:, 0])
    assert (ang.max() - ang.min()) > 3.0                    # the field really turns
    ok = nrm > 0.05 * nrm.max()
    assert ok.float().mean() > 0.9
    for i, (o, r) in enumerate(zip(out, ora)):
        d = (o["pred_gravity"].cpu() - r["pred_gravity"]).abs().amax(0)
        assert d[ok[i]].max() < TOL, (i, d[ok[i]].max())
        for k in ("pred_latitude", "pred_latitude_original", "pred_roll", "pred_pitch", "pred_vfov", "pred_rel_focal"):
            if k == "pred_latitude_original":
                e = U.rel_err(torch.sin(torch.deg2rad(o[k].cpu().double())), torch.sin(torch.deg2rad(r[k].double())))
            else:
                e = U.rel_err(o[k], r[k])
            assert e < TOL, (k, e)


def test_c4_shape_gsv_uncentered_64_images_one_call():
    """BASELINE config C4 (PersNet_Paramnet-GSV-uncentered, 640x480, here 64 images in ONE inference_batch call = two GPUs' worth
    of its 32-per-GPU shards): size-independent properties on all 64, oracle parity on two of them, batch-position invariance."""
    version = "PersNet_Paramnet-GSV-uncentered"
    m, sd = model(version)
    imgs = wg.synth_images(60, 480, 640, 51) + wg.smooth_images(4, 480, 640, 52)
    out = m.inference_batch(imgs)
    assert len(out) == 64
    g = torch.stack([o["pred_gravity_original"] for o in out])
    lo = torch.stack([o["pred_latitude_original"] for o in out])
    assert torch.isfinite(g).all() and torch.isfinite(lo).all()
    assert (g.norm(dim=1) - 1).abs().max() < 1e-5 and lo.abs().max() <= 90.0001
    for o in out:
        assert list(o.keys())[5:] == ["pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy", "pred_rel_focal"]
    _check([out[7], out[62]], om.inference_batch(sd, version, [imgs[7], imgs[62]]), version)
    single = m.inference(imgs[62])
    for k, v in single.items():
        if not isinstance(v, str):
            assert torch.equal(v, out[62][k]), k


def test_c5_point_320x240_batch8():
    """BASELINE config C5, smallest resolution: 8 x (240, 320) -- the post-process DOWN-samples in y (320 -> 240 rows)."""
    version = "Paramnet-360Cities-edina-centered"
    m, sd = model(version)
    imgs = wg.smooth_images(8, 240, 320, 61)
    out = m.inference_batch(imgs)
    _check(out[2:4], om.inference_batch(sd, version, imgs[2:4]), version)
    assert all(o["pred_gravity_original"].shape == (2, 240, 320) for o in out)


def test_float_input_branch_and_apply_image():
    """perspectivefields.py:47-66: non-uint8 images bypass PIL and take the non-antialiased F.interpolate branch;
    ``model.aug.apply_image`` is the same transform stand-alone (uint8: Pillow-exact)."""
    from PIL import Image

    version = "Paramnet-360Cities-edina-centered"
    m, sd = model(version)
    img = wg.smooth_images(1, 360, 500, 71)[0]
    f = img.astype(np.float32) + 0.25
    out = m.inference(f)
    ora = om.inference_float(sd, version, f)
    _check([out], [ora], version)
    got = m.aug.apply_image(img)
    assert got.dtype == np.uint8 and np.array_equal(got, np.asarray(Image.fromarray(img).resize((320, 320), Image.BILINEAR)))
    gf = m.aug.apply_image(f)
    assert gf.dtype == np.float32 and np.abs(gf - om.resize_float(f, 320, 320)).max() < 1e-3
    with pytest.raises(NotImplementedError):
        m.aug.apply_image(img, interp=Image.BICUBIC)


def test_state_dict_kwargs_and_stream_switch():
    version = "Paramnet-360Cities-edina-uncentered"
    m, sd = model(version)
    d = m.state_dict(prefix="x.")
    assert all(k.startswith("x.") for k in d) and len(d) == len(sd)
    img = wg.smooth_images(1, 120, 160, 81)[0]
    base = m.inference(img)
    s2 = torch.cuda.Stream()
    with torch.cuda.stream(s2):          # a caller that switches streams between calls (ADVICE: workspace hand-over)
        o2 = m.inference(img)
    s2.synchronize()
    o3 = m.inference(wg.smooth_images(1, 480, 640, 82)[0])   # larger workspace on the first stream again
    torch.cuda.synchronize()
    for k, v in base.items():
        if not isinstance(v, str):
            assert torch.equal(v, o2[k]), k
    assert torch.isfinite(o3["pred_latitude_original"]).all()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_engines_on_two_devices_in_one_process():
    """The > 48 KB shared-memory opt-in is per device: an engine on cuda:1 created after one on cuda:0 must work (ADVICE r1)."""
    version = "Paramnet-360Cities-edina-centered"
    m0, _ = model(version)
    img = wg.smooth_images(1, 240, 320, 91)[0]
    a = m0.inference(img)
    m1, _ = U.make_model(version, device="cuda:1")
    b = m1.inference(img)
    c = m0.inference(img)
    for k, v in a.items():
        if not isinstance(v, str):
            assert b[k].device.index == 1
            assert torch.equal(v.cpu(), b[k].cpu()) and torch.equal(v, c[k]), k
