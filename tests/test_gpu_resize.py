"""GPU: working sizes other than 320 x 320 (``PerspectiveFields(version, resize=(H, W))``, ``pf_create_sized``).

Kernel precision: the attention core at key counts on both sides of the single-block limit (112) and of the key-block size (64),
in both precisions, against float64; the pre-process bit for bit against oracle/pillow_resize.py at rectangular working sizes;
the post-process from non-320 fields against the oracle (tests/oracle_resize.py: oracle/model.py at another working size).  End to end: all five variants at 320 x 448 and 448 x 448 against the
oracle at 1e-3, the bf16 mode within the DESIGN.md section 3 bounds, decode_only, mixed input sizes, the ``forward`` entry,
output shapes, workspace growth, and the identity of the 320 x 320 path."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_resize as ro
import pf_test_util as U
from bf16_emulation import ANGLE_KEYS, DEG_BOUND, REL_BOUND, error_table
from golden_util import golden_images
from oracle import model as om
from oracle import weights_gen as wg
from oracle.pillow_resize import resize_bilinear_u8
from perspectivefields_b200 import _native

pytestmark = pytest.mark.gpu

VERSIONS = ["Paramnet-360Cities-edina-centered", "Paramnet-360Cities-edina-uncentered", "PersNet-360Cities",
            "PersNet_Paramnet-GSV-uncentered", "PersNet_Paramnet-GSV-centered"]


def _rn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).cuda()


# ------------------------------------------------------------------------------------------------ attention core
@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("nkv", [4, 36, 96, 100, 112, 144, 192, 240, 256])
def test_attention_key_counts(nkv, bf16):
    """pf_op_attention_tc_keys against a float64 softmax.  Split precision: 5e-5 relative (the bar of the 100-key core in
    tests/test_gpu_ops.py).  bf16: against float64 on bf16-rounded q, k, v and P with the one-ulp-of-P bound of
    tests/test_gpu_bf16.py::test_attention_one_product.  The output starts as NaN: every element must be written."""
    g = torch.Generator().manual_seed(nkv)
    B, N, C, heads = 2, 300, 128, 2                # 300 queries: 5 passes of 64, the last one ragged
    q, kv = _rn(g, B, N, C, scale=2.0), _rn(g, B, nkv, 2 * C)
    out = torch.full((B, N, C), float("nan"), device="cuda")
    _native.check(_native.lib().pf_op_attention_tc_keys(q.data_ptr(), kv.data_ptr(), out.data_ptr(), B, N, nkv, C, heads, bf16, U.stream_ptr()))
    torch.cuda.synchronize()
    assert not out.isnan().any()
    if not bf16:
        qh = q.double().reshape(B, N, heads, 64).permute(0, 2, 1, 3)
        kvh = kv.double().reshape(B, nkv, 2, heads, 64).permute(2, 0, 3, 1, 4)
        ref = ((qh @ kvh[0].transpose(-2, -1)) * 0.125).softmax(-1) @ kvh[1]
        assert U.rel_err(out, ref.transpose(1, 2).reshape(B, N, C)) < 5e-5
        return
    r = lambda t: t.bfloat16().double()
    qh, kh, vh = r(q), r(kv[..., :C]), r(kv[..., C:])
    for h in range(heads):
        sl = slice(64 * h, 64 * h + 64)
        s = qh[..., sl] @ kh[..., sl].transpose(1, 2) / 8
        # P is rounded to bf16 once per key (relative error <= 2^-9); the key-block kernel rounds exp(s - m) with the running
        # maximum m of the key blocks seen so far and rescales the fp32 sums later, which can add one more such rounding: each key
        # then contributes at most 2^-8 P_i |v_i| / l, plus 1e-5 relative for fp32 accumulation
        p = torch.exp(s - s.amax(-1, keepdim=True))
        l = p.sum(-1, keepdim=True)
        ref = (p @ vh[..., sl]) / l
        bound = 2.0 ** -8 * (p @ vh[..., sl].abs()) / l + 1e-5 * ref.abs().max()
        err = (out[..., sl].double() - ref).abs()
        assert (err <= bound).all(), (err / bound).max().item()


def test_attention_rejects_unsupported_key_counts():
    L = _native.lib()
    t = torch.zeros(1, 64, 64, device="cuda")
    kv = torch.zeros(1, 300, 128, device="cuda")
    for nkv in (0, 257):
        assert L.pf_op_attention_tc_keys(t.data_ptr(), kv.data_ptr(), t.data_ptr(), 1, 64, nkv, 64, 1, 0, U.stream_ptr()) < 0


# ------------------------------------------------------------------------------------------------ pre / post-process
@pytest.mark.parametrize("net_hw", [(320, 448), (448, 320), (384, 512), (640, 384), (64, 640)])
@pytest.mark.parametrize("hw", [(480, 640), (33, 47), (721, 900)])
def test_preprocess_rectangular_is_pillow_exact(net_hw, hw):
    L = _native.lib()
    img = wg.synth_images(1, hw[0], hw[1], 7)[0]
    mean = np.array([103.53, 116.28, 123.675], np.float32)
    std = np.array([57.375, 57.12, 58.395], np.float32)
    ref = (resize_bilinear_u8(img, net_hw[0], net_hw[1]).astype(np.float32) - mean) / std
    d = torch.from_numpy(img).cuda()
    y = torch.full((net_hw[0], net_hw[1], 4), float("nan"), device="cuda")
    fp = ctypes.POINTER(ctypes.c_float)
    _native.check(L.pf_op_preprocess_sized(d.data_ptr(), hw[0], hw[1], net_hw[0], net_hw[1], mean.ctypes.data_as(fp), std.ctypes.data_as(fp),
                                           y.data_ptr(), U.stream_ptr()))
    torch.cuda.synchronize()
    got = y.cpu().numpy()
    assert np.array_equal(got[..., :3], ref) and (got[..., 3] == 0).all()


@pytest.mark.parametrize("lat_is_sin", [1, 0])
@pytest.mark.parametrize("net_hw", [(320, 448), (640, 384)])
def test_postprocess_from_non_320_fields(net_hw, lat_is_sin):
    """pf_op_postprocess_sized against the oracle's post-process (crop to and scale by the working size) for up- and
    down-sampled targets of several shapes in one call."""
    L = _native.lib()
    g = torch.Generator().manual_seed(5)
    NH, NW = net_hw
    sizes = [(480, 640), (33, 47), (NH, NW), (700, 301)]
    n = len(sizes)
    # smooth fields (as tests/test_gpu_ops.py uses at 320): F.normalize of a bilinear blend of unrelated unit vectors can come near
    # zero length, where the direction depends on the last rounding of either side
    smooth = lambda c: F.interpolate(torch.randn(n, c, 9, 9, generator=g), size=(NH, NW), mode="bicubic", align_corners=False)
    vec = F.normalize(0.3 * smooth(2) + torch.tensor([1.0, -0.6]).view(1, 2, 1, 1), dim=1)
    lat = (torch.rand(n, 1, NH, NW, generator=g) * 2 - 1) if lat_is_sin else smooth(1) * 40
    h = np.array([s[0] for s in sizes], np.int32)
    w = np.array([s[1] for s in sizes], np.int32)
    hw = h.astype(np.int64) * w
    g_off, l_off = np.zeros(n, np.int64), np.zeros(n, np.int64)
    np.cumsum(2 * hw[:-1], out=g_off[1:])
    np.cumsum(hw[:-1], out=l_off[1:])
    go = torch.full((int(2 * hw.sum()),), float("nan"), device="cuda")
    lo = torch.full((int(hw.sum()),), float("nan"), device="cuda")
    i32p, i64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    vd, ld = vec.cuda().contiguous(), lat.cuda().contiguous()
    _native.check(L.pf_op_postprocess_sized(vd.data_ptr(), ld.data_ptr(), n, NH, NW, h.ctypes.data_as(i32p), w.ctypes.data_as(i32p), go.data_ptr(),
                                            g_off.ctypes.data_as(i64p), lo.data_ptr(), l_off.ctypes.data_as(i64p), lat_is_sin, U.stream_ptr()))
    torch.cuda.synchronize()
    cfg = {"gravity": "regression", "latitude": "regression" if lat_is_sin else "classification"}
    for i, (hh, ww) in enumerate(sizes):
        rg = ro.postprocess_gravity(cfg, vec[i], hh, ww, net_hw)
        gg = go[g_off[i]:g_off[i] + 2 * hh * ww].view(2, hh, ww).cpu()
        assert (gg - rg).abs().max() < 2e-5, i
        if lat_is_sin:
            rl = torch.rad2deg(torch.asin(ro.pf_postprocess(lat[i], hh, ww, net_hw)[0]))
        else:
            rl = ro.pf_postprocess(lat[i], hh, ww, net_hw)[0]
        ll = lo[l_off[i]:l_off[i] + hh * ww].view(hh, ww).cpu()
        assert (ll - rl).abs().max() < 1e-3, i


# ------------------------------------------------------------------------------------------------ end to end
_models = {}


def model(version, resize, **kw):
    key = (version, resize, tuple(sorted(kw.items())))
    if key not in _models:
        _models[key] = U.make_model(version, model_kwargs=dict(kw, resize=resize))
    return _models[key]


def _check_against_oracle(version, out, ora, tol=1e-3):
    classification = version == "PersNet-360Cities"
    for o, r in zip(out, ora):
        assert list(o.keys()) == list(r.keys())
        for k, v in r.items():
            if isinstance(v, str):
                assert o[k] == v
                continue
            assert tuple(o[k].shape) == tuple(v.shape), (k, o[k].shape, v.shape)
            if classification and k.endswith("_original"):
                continue
            if k == "pred_latitude_original" and v.abs().max() > 75:
                # degrees = asin(sin_lat) is not Lipschitz at +-1, where the regression head clamps: the sine domain everywhere and
                # degrees away from the poles (the metric of tests/test_gpu_forward.py)
                a_, b_ = o[k].detach().cpu().double(), v.double()
                e = U.rel_err(torch.sin(torch.deg2rad(a_)), torch.sin(torch.deg2rad(b_)))
                far = b_.abs() < 75
                if far.any():
                    e = max(e, ((a_ - b_).abs()[far].max() / b_.abs().max()).item())
            else:
                e = U.rel_err(o[k], v)
            assert e < tol, (version, k, e)
        if classification:
            h, w = r["pred_latitude_original"].shape
            for key, okey, scale in (("pred_gravity", "pred_gravity_original", 1.0), ("pred_latitude", "pred_latitude_original", 90.0)):
                err = max((o[key].cpu() - r[key]).abs().max().item(), 1e-6)
                stable = U.stable_mask(r[key], err, h, w)
                assert stable.float().mean() > 0.5, okey
                d = (o[okey].cpu() - r[okey]).abs()
                d = d.amax(0) if d.ndim == 3 else d
                assert d[stable].max().item() / scale < tol, okey


@pytest.mark.parametrize("resize", [(320, 448), (448, 448)])
@pytest.mark.parametrize("version", VERSIONS)
def test_variants_against_the_oracle(version, resize):
    """Mixed input sizes in one call (the golden images: 480 x 640 and 360 x 500); 448 x 448 has 196 keys per attention
    (the key-block path), 320 x 448 has 140."""
    m, sd = model(version, resize)
    imgs = golden_images()
    out = m.inference_batch(imgs)
    ora = ro.inference_batch(sd, version, imgs, resize)
    assert tuple(out[0]["pred_gravity"].shape[1:]) == resize and tuple(out[0]["pred_latitude"].shape[1:]) == resize
    _check_against_oracle(version, out, ora)


@pytest.mark.parametrize("version", ["Paramnet-360Cities-edina-centered", "PersNet_Paramnet-GSV-uncentered"])
def test_bf16_at_a_rectangular_size(version):
    resize = (384, 512)
    m, sd = model(version, resize, precision="bf16")
    imgs = golden_images()
    out = m.inference_batch(imgs)
    ora = ro.inference_batch(sd, version, imgs, resize)
    table = error_table(out, ora)
    print(version, {k: round(v, 4) for k, v in table.items()})
    for k, e in table.items():
        assert e < (DEG_BOUND if k in ANGLE_KEYS else REL_BOUND), (version, k, e)


def test_decode_only_at_a_non_square_size():
    version, resize = "PersNet-360Cities", (320, 448)
    m, _ = model(version, resize)
    d, _ = model(version, resize, logits=False)
    imgs = golden_images()
    a, b = m.inference_batch(imgs), d.inference_batch(imgs)
    for o, r in zip(b, a):
        assert tuple(o["pred_gravity"].shape) == (2,) + resize and tuple(o["pred_latitude"].shape) == (1,) + resize
        idx_g, idx_l = r["pred_gravity"].argmax(0).cpu(), r["pred_latitude"].argmax(0).cpu()
        assert (o["pred_gravity"].cpu() - om.decode_bin(idx_g, 73)).abs().max() < 2e-6
        assert torch.equal(o["pred_latitude"].cpu()[0], om.decode_bin_latitude(idx_l, 180))
        assert torch.equal(o["pred_gravity_original"], r["pred_gravity_original"])
        assert torch.equal(o["pred_latitude_original"], r["pred_latitude_original"])


def test_forward_entry_and_single_image():
    version, resize = "Paramnet-360Cities-edina-uncentered", (448, 320)
    m, sd = model(version, resize)
    img = wg.smooth_images(1, 300, 420, 4)[0]
    one = m.inference(img)
    batch = m.inference_batch([img])[0]
    for k, v in one.items():
        if isinstance(v, torch.Tensor):
            assert torch.equal(v, batch[k]), k
    x = ro.preprocess(img, resize)
    out = m.forward([{"image": x, "height": 300, "width": 420}])[0]
    ora = ro.forward(sd, version, [{"image": x, "height": 300, "width": 420}], resize)
    _check_against_oracle(version, [out], ora)
    with pytest.raises(ValueError):
        m.forward([{"image": torch.zeros(3, 320, 320), "height": 300, "width": 420}])


def test_workspace_grows_with_the_working_area():
    L = _native.lib()
    version = "Paramnet-360Cities-edina-centered"
    sizes = [(256, 256), (320, 320), (320, 448), (512, 512)]
    ws = []
    for r in sizes:
        m, _ = model(version, r)
        eng = m._get_engine()
        assert (eng.net_h, eng.net_w) == r
        ws.append(_native.check(L.pf_workspace_bytes(eng.handle, 2, 480)))
    assert all(a < b for a, b in zip(ws, ws[1:])), ws


def test_320_identity_and_coexistence():
    """resize=(320, 320) runs exactly the default graph, and a 320 model and a 448 model alive in one process each give what they
    give alone (resize tables, tensor-map cache and workspace are per engine)."""
    version = "Paramnet-360Cities-edina-centered"
    imgs = golden_images()

    def run(mod):
        return [{k: v.clone() for k, v in o.items() if isinstance(v, torch.Tensor)} for o in mod.inference_batch(imgs)]

    def same(a, b):
        return all(torch.equal(x[k].reshape(-1).view(torch.int32), y[k].reshape(-1).view(torch.int32)) for x, y in zip(a, b) for k in x)

    d, _ = U.make_model(version)
    alone_d = run(d)
    r320, _ = U.make_model(version, model_kwargs={"resize": (320, 320)})
    assert same(run(r320), alone_d)
    big, _ = U.make_model(version, model_kwargs={"resize": (448, 448)})
    alone_big = run(big)
    assert same(run(d), alone_d) and same(run(big), alone_big)
    assert tuple(alone_big[0]["pred_gravity"].shape) == (2, 448, 448)


def test_unsupported_options_and_sizes_are_rejected():
    version = "Paramnet-360Cities-edina-centered"
    m, _ = U.make_model(version, model_kwargs={"resize": (320, 448)})
    img = wg.smooth_images(1, 100, 120, 2)[0]
    assert tuple(m.inference(img)["pred_gravity"].shape) == (2, 320, 448)
    L = _native.lib()
    desc = _native.pf_model_desc()
    desc.gravity_classes, desc.latitude_classes = 2, 1
    h = ctypes.c_void_p()
    for hw in ((320, 330), (32, 320), (672, 320), (640, 448)):
        assert L.pf_create_sized(0, ctypes.byref(desc), hw[0], hw[1], ctypes.byref(h)) < 0, hw
