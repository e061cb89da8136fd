"""GPU: every operator of libpf_b200.so, called through the C ABI, against a float64 torch restatement of the same op
on the same seeded inputs (all GEMM-shaped operators run on the TMA -> wgmma engine, the only engine since ABI 2).  Tolerances: 5e-5 relative for the bf16x3 split-precision GEMM engine (per-product error
~2^-17; the end-to-end bar is 1e-3), 1e-5 for fp32 CUDA-core ops, bit-exact for the integer resize."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pf_test_util as U

pytestmark = pytest.mark.gpu


def _rn(g, *s):
    return torch.randn(*s, generator=g)


# B, H, W, Cin, N, K, stride, pad, in_relu, act, res, res_relu
GEMM_CASES = [
    (2, 20, 20, 64, 256, 3, 1, 1, 0, 0, 0, 0),      # composed head conv shape (C1 -> 256)
    (2, 20, 20, 256, 256, 3, 1, 1, 1, 1, 0, 0),     # RCU conv1: relu prologue + relu epilogue
    (1, 23, 17, 256, 256, 3, 1, 1, 0, 0, 1, 1),     # RCU conv2: + relu(residual), ragged M
    (1, 1, 700, 320, 640, 1, 1, 0, 0, 0, 0, 0),     # kv linear (N tail: 640 = 5 x 128)
    (1, 1, 300, 96, 384, 1, 1, 0, 0, 2, 0, 0),      # ConvNeXt pwconv1 + GELU
    (1, 1, 130, 384, 96, 1, 1, 0, 0, 0, 1, 0),      # pwconv2 + residual, N = 96 (64-wide tiles)
    (2, 80, 80, 64, 64, 8, 8, 0, 0, 0, 0, 0),       # spatial-reduction conv k = s = 8
    (2, 40, 40, 64, 128, 3, 2, 1, 0, 0, 0, 0),      # overlap patch embed, stride 2
    (1, 24, 24, 64, 32, 3, 1, 1, 0, 1, 0, 0),       # conv_fuse_conv1, N = 32 tile
    (1, 16, 16, 96, 192, 2, 2, 0, 0, 0, 0, 0),      # ConvNeXt downsample
    (1, 40, 40, 320, 64, 3, 1, 1, 0, 1, 0, 0),      # conv_fuse_conv0 shape
    (1, 1, 1, 512, 512, 1, 1, 0, 0, 0, 0, 0),       # single row (M = 1)
]


@pytest.mark.parametrize("case", GEMM_CASES)
def test_conv_gemm(case):
    B, H, W, Cin, N, K, s, p, ir, act, res, rr = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x = _rn(g, B, Cin, H, W).cuda()
    w = _rn(g, N, Cin, K, K) / (Cin * K * K) ** 0.5
    b = _rn(g, N)
    ref = F.conv2d((F.relu(x) if ir else x).double(), w.double().cuda(), b.double().cuda(), stride=s, padding=p)
    ref = F.relu(ref) if act == 1 else (F.gelu(ref) if act == 2 else ref)
    r = None
    if res:
        r = _rn(g, *ref.shape).cuda()
        ref = ref + (F.relu(r) if rr else r).double()
        r = r.permute(0, 2, 3, 1).contiguous()
    y = U.conv_gemm(x.permute(0, 2, 3, 1).contiguous(), w, b, s, p, ir, act, r, rr)
    assert U.rel_err(y.permute(0, 3, 1, 2), ref) < 5e-5


def test_conv_gemm_is_deterministic_and_batch_invariant():
    g = torch.Generator().manual_seed(3)
    x = _rn(g, 3, 12, 12, 256).cuda()
    w, b = _rn(g, 256, 256, 3, 3) / 48, _rn(g, 256)
    y = U.conv_gemm(x, w, b, 1, 1)
    assert torch.equal(y, U.conv_gemm(x, w, b, 1, 1))
    assert torch.equal(y[1:2], U.conv_gemm(x[1:2].contiguous(), w, b, 1, 1))


@pytest.mark.parametrize("C", [64, 96, 128, 192, 320, 384, 512, 768])
def test_layernorm(C):
    from perspectivefields_b200 import _native

    g = torch.Generator().manual_seed(C)
    x = (_rn(g, 777, C) * 3 + 1).cuda()
    w, b = _rn(g, C).cuda(), _rn(g, C).cuda()
    y = torch.empty_like(x)
    _native.check(_native.lib().pf_op_layernorm(x.data_ptr(), y.data_ptr(), 777, C, w.data_ptr(), b.data_ptr(), 1e-6, U.stream_ptr()))
    assert U.rel_err(y, F.layer_norm(x.double(), (C,), w.double(), b.double(), 1e-6)) < 1e-5


@pytest.mark.parametrize("shape", [(2, 6400, 1), (2, 1600, 2), (1, 400, 5), (1, 100, 8), (1, 77, 2), (1, 1000, 1)])
def test_attention(shape):
    from perspectivefields_b200 import _native

    B, N, heads = shape
    C = heads * 64
    g = torch.Generator().manual_seed(N)
    q, kv = (_rn(g, B, N, C) * 2).cuda(), (_rn(g, B, 100, 2 * C) * 2).cuda()
    o = torch.empty_like(q)
    _native.check(_native.lib().pf_op_attention_tc(q.data_ptr(), kv.data_ptr(), o.data_ptr(), B, N, C, heads, U.stream_ptr()))
    qh = q.double().reshape(B, N, heads, 64).permute(0, 2, 1, 3)
    kvh = kv.double().reshape(B, 100, 2, heads, 64).permute(2, 0, 3, 1, 4)
    ref = ((qh @ kvh[0].transpose(-2, -1)) * 0.125).softmax(-1) @ kvh[1]
    assert U.rel_err(o, ref.transpose(1, 2).reshape(B, N, C)) < 5e-5


def test_depthwise_and_upsample():
    from perspectivefields_b200 import _native

    L = _native.lib()
    g = torch.Generator().manual_seed(9)
    x, w, b = _rn(g, 2, 256, 20, 20).cuda(), _rn(g, 256, 1, 3, 3).cuda(), _rn(g, 256).cuda()
    xh = x.permute(0, 2, 3, 1).contiguous()
    y = torch.empty_like(xh)
    _native.check(L.pf_op_dwconv3x3_gelu(xh.data_ptr(), y.data_ptr(), 2, 20, 20, 256, w.reshape(256, 9).t().contiguous().data_ptr(), b.data_ptr(), U.stream_ptr()))
    assert U.rel_err(y.permute(0, 3, 1, 2), F.gelu(F.conv2d(x.double(), w.double(), b.double(), padding=1, groups=256))) < 1e-5
    x, w, b = _rn(g, 2, 96, 16, 16).cuda(), _rn(g, 96, 1, 7, 7).cuda(), _rn(g, 96).cuda()
    xh = x.permute(0, 2, 3, 1).contiguous()
    y = torch.empty_like(xh)
    _native.check(L.pf_op_dwconv7x7(xh.data_ptr(), y.data_ptr(), 2, 16, 16, 96, w.reshape(96, 49).t().contiguous().data_ptr(), b.data_ptr(), U.stream_ptr()))
    assert U.rel_err(y.permute(0, 3, 1, 2), F.conv2d(x.double(), w.double(), b.double(), padding=3, groups=96)) < 1e-5
    x = _rn(g, 2, 64, 10, 13).cuda()
    xh = x.permute(0, 2, 3, 1).contiguous()
    y = torch.empty(2, 20, 26, 64, device="cuda")
    _native.check(L.pf_op_upsample2x(xh.data_ptr(), y.data_ptr(), 2, 10, 13, 64, U.stream_ptr()))
    assert U.rel_err(y.permute(0, 3, 1, 2), F.interpolate(x.double(), scale_factor=2, mode="bilinear", align_corners=False)) < 1e-6


@pytest.mark.parametrize("hw", [(480, 640), (240, 320), (320, 320), (721, 900), (1536, 2048), (33, 47), (512, 512), (320, 500), (1, 1)])
def test_preprocess_is_bit_exact_vs_pillow(hw):
    from PIL import Image

    from perspectivefields_b200 import _native

    h, w = hw
    img = np.random.RandomState(h + w).randint(0, 256, (h, w, 3), dtype=np.uint8)
    mean = np.array([103.53, 116.28, 123.675], np.float32)
    ref = np.asarray(Image.fromarray(img).resize((320, 320), Image.BILINEAR)).astype(np.float32) - mean
    d = torch.from_numpy(img).cuda()
    y = torch.empty(320, 320, 4, device="cuda")
    _native.check(_native.lib().pf_op_preprocess(d.data_ptr(), h, w, (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(1, 1, 1), y.data_ptr(), U.stream_ptr()))
    torch.cuda.synchronize()
    got = y.cpu().numpy()
    assert np.array_equal(got[..., :3], ref) and not got[..., 3].any()


# ---- more GEMM-mode / halo-mode shapes of the TMA -> wgmma engine.  The comments give the (BN, KB) the dispatcher picks on
# 132 SMs (test_host_logic.py::test_tile_dispatch_of_the_op_cases checks them); 3x3 convs with Cin % 64 == 0 run in halo mode,
# everything else in GEMM mode (strided / k > 1 convs after a patch gather)
TC_CASES = [
    (2, 20, 20, 256, 256, 3, 1, 1, 1, 1, 0, 0),     # RCU conv1, halo (256, 32)
    (1, 23, 17, 256, 256, 3, 1, 1, 0, 0, 1, 1),     # RCU conv2 + relu(residual), ragged tiles, halo (256, 32)
    (2, 16, 16, 64, 512, 3, 1, 1, 0, 0, 0, 0),      # composed proc conv, halo (256, 32): two N tiles
    (1, 1, 700, 320, 256, 1, 1, 0, 0, 0, 0, 0),     # plain linear, K = 320: (32, 64), 5 K steps
    (1, 1, 64, 32, 256, 1, 1, 0, 0, 0, 0, 0),       # single K step: (32, 32)
    (3, 40, 40, 256, 256, 3, 1, 1, 1, 0, 0, 0),     # halo (256, 32): 45 tiles, 72 K steps
    (1, 1, 700, 320, 640, 1, 1, 0, 0, 0, 0, 0),     # kv linear: (32, 64), 20 N tiles
    (1, 1, 300, 96, 384, 1, 1, 0, 0, 2, 0, 0),      # GELU, K = 96: (32, 32)
    (1, 1, 130, 384, 96, 1, 1, 0, 0, 0, 1, 0),      # + residual: (32, 64), 3 N tiles
    (2, 80, 80, 64, 64, 8, 8, 0, 0, 0, 0, 0),       # k = s = 8, K = 4096: (32, 64)
    (1, 24, 24, 64, 32, 3, 1, 1, 0, 1, 0, 0),       # halo (32, 64), resident weights
    (1, 40, 40, 320, 64, 3, 1, 1, 0, 1, 0, 0),      # halo (64, 64), K = 2880
    (2, 40, 40, 64, 128, 3, 2, 1, 0, 0, 0, 0),      # stride 2, patch gather: (32, 64)
    (1, 1, 500, 64, 320, 1, 1, 0, 0, 0, 0, 0),      # N = 320 -> ten 32-wide tiles: (32, 64)
    # large GEMM-mode launches (several tiles per CTA of the persistent grid)
    (1, 1, 12800, 320, 320, 1, 1, 0, 0, 0, 1, 0),   # MiT stage-3 proj: 100 row tiles x 2 N tiles of 160 (160, 32), + residual
    (1, 1, 20000, 96, 384, 1, 1, 0, 0, 2, 0, 0),    # ragged M (156.25 row tiles), GELU: (192, 32), 3 K steps
    (1, 1, 19000, 1280, 320, 1, 1, 0, 0, 0, 1, 1),  # K = 1280 (the ring wraps many times), relu(residual), last row tile partial: (160, 32)
    (1, 1, 25000, 64, 640, 1, 1, 0, 0, 1, 0, 0),    # N = 640 -> three N tiles of 224 (last one partial), ReLU: (224, 32)
    (1, 1, 40000, 128, 64, 1, 1, 0, 0, 0, 0, 0),    # narrow N = 64: (64, 64)
]



HALO_CASES = [
    (2, 16, 8, 64, 32, 0, 1, 0, 0),       # exactly one tile per image, conv_fuse_conv1 shape class
    (1, 80, 80, 256, 256, 1, 1, 0, 0),    # RCU conv1 at 80x80
    (2, 23, 17, 256, 256, 0, 0, 1, 1),    # ragged tiles in both directions + relu(residual)
    (1, 10, 10, 512, 512, 0, 0, 0, 0),    # proc conv at the coarsest level (tile larger than the image), two N tiles
    (1, 40, 40, 320, 64, 0, 1, 0, 0),     # conv_fuse_conv0 shape class (5 chunks)
    (3, 33, 9, 128, 128, 0, 0, 0, 0),
]



# ---- inputs are split into bf16 hi/lo planes first, exactly as the forward graph does
@pytest.mark.parametrize("case", TC_CASES)
def test_conv_gemm_tma_engine(case):
    B, H, W, Cin, N, K, s, p, ir, act, res, rr = case
    if N % 32:
        pytest.skip("TMA engine needs N % 32 == 0")
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x = _rn(g, B, Cin, H, W).cuda()
    w = _rn(g, N, Cin, K, K) / (Cin * K * K) ** 0.5
    b = _rn(g, N)
    ref = F.conv2d((F.relu(x) if ir else x).double(), w.double().cuda(), b.double().cuda(), stride=s, padding=p)
    ref = F.relu(ref) if act == 1 else (F.gelu(ref) if act == 2 else ref)
    r = None
    if res:
        r = _rn(g, *ref.shape).cuda()
        ref = ref + (F.relu(r) if rr else r).double()
        r = r.permute(0, 2, 3, 1).contiguous()
    y = U.conv_gemm(x.permute(0, 2, 3, 1).contiguous(), w, b, s, p, ir, act, r, rr)
    assert U.rel_err(y.permute(0, 3, 1, 2), ref) < 5e-5


@pytest.mark.parametrize("case", HALO_CASES)
def test_conv3x3_tma_halo(case):
    B, H, W, Cin, N, ir, act, res, rr = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x = _rn(g, B, Cin, H, W).cuda()
    w = _rn(g, N, Cin, 3, 3) / (Cin * 9) ** 0.5
    b = _rn(g, N)
    ref = F.conv2d((F.relu(x) if ir else x).double(), w.double().cuda(), b.double().cuda(), padding=1)
    ref = F.relu(ref) if act == 1 else ref
    r = None
    if res:
        r = _rn(g, *ref.shape).cuda()
        ref = ref + (F.relu(r) if rr else r).double()
        r = r.permute(0, 2, 3, 1).contiguous()
    y = U.conv_gemm(x.permute(0, 2, 3, 1).contiguous(), w, b, 1, 1, ir, act, r, rr)
    assert U.rel_err(y.permute(0, 3, 1, 2), ref) < 5e-5


# ---- classification decode: argmax + bin decode (gravity_head.py:243-244 + utils.py:114-130; latitude_head.py:205-208 + utils.py:148-162)
def _decode_ref(logits, is_gravity):
    from oracle import model as om

    nc = logits.shape[1]
    idx = logits.argmax(dim=1)
    if is_gravity:
        return torch.stack([om.decode_bin(i, nc) for i in idx])
    return torch.stack([om.decode_bin_latitude(i, nc).unsqueeze(0) for i in idx])


@pytest.mark.parametrize("nc,is_gravity", [(73, 1), (180, 0)])
def test_argmax_decode_hand_made_logits(nc, is_gravity):
    from perspectivefields_b200 import _native

    B, HW = 2, 500
    g = torch.Generator().manual_seed(nc)
    logits = _rn(g, B, nc, HW)
    # every bin wins somewhere (incl. the "no direction" bin 72 -> (0, 0)), plus exact ties (first maximal index wins)
    for c in range(nc):
        logits[0, c, c] = 50.0
    logits[1, :, 0] = 1.0                       # all equal: bin 0
    logits[1, 5, 1] = logits[1, 9, 1] = 77.0     # two-way tie: bin 5
    logits[1, nc - 1, 2] = logits[1, nc - 2, 2] = 60.0
    d = logits.cuda()
    field = torch.empty(B, 2 if is_gravity else 1, HW, device="cuda")
    _native.check(_native.lib().pf_op_argmax_decode(d.data_ptr(), field.data_ptr(), B, HW, nc, is_gravity, U.stream_ptr()))
    torch.cuda.synchronize()
    ref = _decode_ref(logits, is_gravity)
    assert (field.cpu() - ref).abs().max() < 2e-6          # cos / sin in fp32
    if is_gravity:
        assert torch.equal(field[0, :, nc - 1].cpu(), torch.zeros(2))


@pytest.mark.parametrize("nc,is_gravity", [(73, 1), (180, 0)])
def test_fused_pred_argmax_decode_equals_separate_path(nc, is_gravity):
    """Option "decode_only": 1x1 conv + argmax + decode without logits == the same decode applied to fp32 logits."""
    from perspectivefields_b200 import _native

    B, HW = 2, 1000
    g = torch.Generator().manual_seed(7 + nc)
    feat = F.relu(_rn(g, B * HW, 64))
    w, b = _rn(g, nc, 32) * 0.3, _rn(g, nc) * 0.1
    coff = 32 if not is_gravity else 0
    logits = (feat[:, coff:coff + 32].double() @ w.double().t() + b.double()).reshape(B, HW, nc).permute(0, 2, 1)
    field = torch.empty(B, 2 if is_gravity else 1, HW, device="cuda")
    fd, wd, bd = feat.cuda(), w.cuda(), b.cuda()
    _native.check(_native.lib().pf_op_pred_argmax_decode(fd.data_ptr(), 64, coff, wd.data_ptr(), bd.data_ptr(), field.data_ptr(), B, HW, nc, is_gravity,
                                                         U.stream_ptr()))
    torch.cuda.synchronize()
    ref = _decode_ref(logits.float(), is_gravity)
    top2 = logits.topk(2, dim=1).values
    stable = (top2[:, 0] - top2[:, 1]) > 1e-4                # fp32 logits vs the float64 ones above
    assert stable.float().mean() > 0.99
    diff = (field.cpu() - ref).abs().amax(dim=1)
    assert diff[stable].max() < 2e-6


@pytest.mark.parametrize("sizes", [[(480, 640)], [(33, 47), (320, 320), (240, 321)], [(768, 1024), (5, 4100)], [(1, 1), (2, 3)]])
@pytest.mark.parametrize("lat_is_sin", [1, 0])
def test_postprocess_op(sizes, lat_is_sin):
    """Resample to the original sizes + normalise / asin (gravity_head.py:246-256, latitude_head.py:209-219, utils.py:483-507)."""
    from oracle import model as om
    from perspectivefields_b200 import _native

    n = len(sizes)
    g = torch.Generator().manual_seed(len(sizes) * 10 + lat_is_sin)
    # smooth direction field (a trained head's output is smooth): neighbouring unit vectors never cancel, so the normalise after
    # the resampling stays well conditioned
    vec = F.normalize(0.3 * F.interpolate(_rn(g, n, 2, 9, 9), size=(320, 320), mode="bicubic", align_corners=False) + torch.tensor([1.0, -0.6]).view(1, 2, 1, 1), dim=1)
    lat = (torch.rand(n, 1, 320, 320, generator=g) * 2 - 1) if lat_is_sin else (_rn(g, n, 1, 320, 320) * 40)
    h = np.asarray([s[0] for s in sizes], np.int32)
    w = np.asarray([s[1] for s in sizes], np.int32)
    hw = h.astype(np.int64) * w
    g_off, l_off = np.zeros(n, np.int64), np.zeros(n, np.int64)
    np.cumsum(2 * hw[:-1], out=g_off[1:])
    np.cumsum(hw[:-1], out=l_off[1:])
    go = torch.empty(int(2 * hw.sum()), device="cuda")
    lo = torch.empty(int(hw.sum()), device="cuda")
    i32p, i64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    vd, ld = vec.cuda(), lat.cuda()
    _native.check(_native.lib().pf_op_postprocess(vd.data_ptr(), ld.data_ptr(), n, h.ctypes.data_as(i32p), w.ctypes.data_as(i32p), go.data_ptr(),
                                                  g_off.ctypes.data_as(i64p), lo.data_ptr(), l_off.ctypes.data_as(i64p), lat_is_sin, U.stream_ptr()))
    cfg = {"gravity": "regression", "latitude": "regression" if lat_is_sin else "none"}
    for i, (hh, ww) in enumerate(sizes):
        ref_g = om.postprocess_gravity(cfg, vec[i], hh, ww)
        got_g = go[g_off[i]:g_off[i] + 2 * hh * ww].view(2, hh, ww).cpu()
        assert (got_g - ref_g).abs().max() < 2e-5, (i, "gravity")
        ref_l = om.pf_postprocess(lat[i], hh, ww)[0]
        got_l = lo[l_off[i]:l_off[i] + hh * ww].view(hh, ww).cpu()
        if lat_is_sin:
            # degrees = asin(x): compare in the sine domain near the poles (asin is not Lipschitz at +-1), in degrees elsewhere
            assert (torch.sin(torch.deg2rad(got_l)) - ref_l).abs().max() < 2e-6
            far = ref_l.abs() < 0.97
            if far.any():
                assert (got_l - torch.rad2deg(torch.asin(ref_l)))[far].abs().max() < 2e-4
        else:
            assert (got_l - ref_l).abs().max() < 1e-4 * 40


@pytest.mark.parametrize("hw,new", [((480, 640), (320, 320)), ((100, 37), (64, 48)), ((320, 320), (320, 320)), ((50, 60), (200, 300)), ((1536, 2048), (320, 320))])
def test_resize_ops_match_pillow_and_aten(hw, new):
    """ResizeTransform.apply_image (perspectivefields.py:34-67): uint8 -> Pillow (bit-exact), float32 -> F.interpolate bilinear."""
    from PIL import Image

    from perspectivefields_b200 import _native

    L = _native.lib()
    h, w = hw
    nh, nw = new
    rs = np.random.RandomState(h * 7 + w)
    img = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
    d = torch.from_numpy(img).cuda()
    out = torch.empty(nh, nw, 3, dtype=torch.uint8, device="cuda")
    _native.check(L.pf_op_resize_u8(d.data_ptr(), h, w, nh, nw, out.data_ptr(), U.stream_ptr()))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), np.asarray(Image.fromarray(img).resize((nw, nh), Image.BILINEAR)))
    f = torch.from_numpy(rs.standard_normal((h, w, 3)).astype(np.float32))
    fo = torch.empty(nh, nw, 3, device="cuda")
    fd = f.cuda()
    _native.check(L.pf_op_resize_f32(fd.data_ptr(), h, w, 3, nh, nw, fo.data_ptr(), U.stream_ptr()))
    # float32 like the reference's call (the sampling positions scale * (dst + 0.5) - 0.5 are float32 quantities in ATen: a float64
    # restatement differs by ~1e-5 x the local gradient at non-dyadic ratios)
    ref = F.interpolate(f.permute(2, 0, 1)[None], (nh, nw), mode="bilinear", align_corners=False)[0].permute(1, 2, 0)
    assert (fo.cpu() - ref).abs().max() < 2e-5
