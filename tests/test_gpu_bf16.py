"""GPU: the opt-in bf16 precision mode (engine option "bf16", ``PerspectiveFields(..., precision="bf16")``).

Kernel precision: every one-product instantiation of the TMA -> wgmma engine through pf_op_tma_bf16, and the one-product
attention core through pf_op_attention_tc_bf16, against float64 restatements on the operand values the kernels multiply -- the
hi planes (bf16(x)) only.  Engine bar: 5e-5 relative, as for the split-precision engine (tests/test_gpu_engine.py); output
buffers are filled with NaN first and what a launch does not own must keep the NaN bit pattern.

End to end: the five variants with precision="bf16" against the fp32 oracle, within the bounds the CPU emulation fixed
(tests/bf16_emulation.py, DESIGN.md section 3), and switching the option on one model."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import pf_test_util as U
from bf16_emulation import ANGLE_KEYS, DEG_BOUND, REL_BOUND, error_table
from golden_util import golden_images
from oracle import model as om
from perspectivefields_b200 import _native, weights
# the split-precision engine tests' helpers: NaN-filled buffers, the launch struct, the float64 conv and the ownership checks (the
# split planes must be the exact split of relu?(C) in the one-product mode too: CUDA-core readers such as the conv1 border ring
# rebuild fp32 from hi + lo)
from test_gpu_engine import GEMM, HALO, SPARE, TOL, check_f32, check_split, conv3x3_ref, engine_variants, nan16, nan32, op_struct, rn, untouched

pytestmark = pytest.mark.gpu

LAUNCHED = set()     # (mode, bn, kb, schedule) of every successful pf_op_tma_bf16 call of this module


def split(x):
    """-> (hi, lo, hi in float64): the planes a producer writes and the value the one-product engine multiplies."""
    hi, lo = weights.split_hi_lo(x)
    return hi, lo, hi.double()


def tma_bf16(**kw):
    op = op_struct(**kw)
    _native.check(_native.lib().pf_op_tma_bf16(ctypes.byref(op), U.stream_ptr()))
    torch.cuda.synchronize()
    LAUNCHED.add((op.mode, op.picked_bn, op.picked_kb, op.picked_sched))
    return op


def halo_problem(g, B, H, W, Cin, N):
    ahi, alo, a = split(rn(g, B, H, W, Cin))
    whi, wlo, w = split(rn(g, N, 9 * Cin, scale=(9 * Cin) ** -0.5))
    bias = rn(g, N)
    return dict(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=Cin, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1), \
        conv3x3_ref(a, w, Cin) + bias.double()


# ------------------------------------------------------------------------------------------------ one product, not three
def test_one_product_runs_hi_times_hi_only():
    """The result matches hi(A) hi(W)^T at 5e-5 and is far from (hi + lo)(A) (hi + lo)(W)^T, which pf_op_tma computes: the two
    differ by about 2^-9 relative (the bf16 rounding of the operands), 50x the kernel bar."""
    g = torch.Generator().manual_seed(3)
    M, K, N = 512, 256, 128
    ahi, alo, a = split(rn(g, M, K))
    whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
    args = dict(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, ldc=N)
    C1, C3 = nan32(M, N), nan32(M, N)
    tma_bf16(C=C1, **args)
    _native.check(_native.lib().pf_op_tma(ctypes.byref(op_struct(C=C3, **args)), U.stream_ptr()))
    torch.cuda.synchronize()
    full = (ahi.double() + alo.double()) @ (whi.double() + wlo.double()).t()
    hi_only = a @ w.t()
    assert U.rel_err(C1, hi_only) < TOL
    assert U.rel_err(C1, full) > 20 * TOL, U.rel_err(C1, full)
    assert U.rel_err(C3, full) < TOL and U.rel_err(C3, hi_only) > 20 * TOL


# ------------------------------------------------------------------------------------------------ every instantiation, GEMM mode
@pytest.mark.parametrize("sched", [1, 2])
def test_gemm_instantiations_both_schedules_ragged(sched):
    """Every GEMM-mode one-product instantiation, cooperative (1) and ping-pong (2): M = 1000 (ragged last 64- and 128-row
    tile), N = 480 (a partial last N tile for most widths), K = 320; + bias, GELU, split planes.  All bit-identical."""
    g = torch.Generator().manual_seed(77)
    M, K, N, ldc, lds = 1000, 320, 480, 488, 496
    ahi, alo, a = split(rn(g, M, K))
    whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
    bias = rn(g, N)
    ref = F.gelu(a @ w.t() + bias.double())
    outs = {}
    for m, bn, kb in sorted(engine_variants()):
        if m != GEMM:
            continue
        C, shi, slo = nan32(M + SPARE, ldc), nan16(M + SPARE, lds), nan16(M + SPARE, lds)
        op = tma_bf16(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1, act=2,
                      C=C, ldc=ldc, c_coff=4, s_hi=shi, s_lo=slo, lds=lds, s_coff=8, force_bn=bn, force_kb=kb, force_sched=sched)
        assert (op.picked_bn, op.picked_kb, op.picked_sched) == (bn, kb, sched)
        check_f32(C, [(4, ref)], tol=1e-4)      # (GELU: the engine's polynomial erf is 4.4e-7 absolute)
        check_split(shi, slo, [(8, C[:M, 4:4 + N])], False)
        outs[(bn, kb)] = C
    first = next(iter(outs))
    assert all(torch.equal(v.view(torch.int32), outs[first].view(torch.int32)) for v in outs.values())


def test_layer_scale_with_in_place_residual():
    g = torch.Generator().manual_seed(5)
    M, K, N, ld = 777, 384, 96, 104
    ahi, alo, a = split(rn(g, M, K))
    whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
    bias, gamma = rn(g, N), (torch.rand(N, generator=g) * 0.4 + 0.1).cuda()
    C = nan32(M + SPARE, ld)
    C[:M, 8:8 + N] = rn(g, M, N)
    ref = (a @ w.t() + bias.double()) * gamma.double() + C[:M, 8:8 + N].double()
    tma_bf16(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1, gamma=gamma,
             res=C, ldr=ld, r_coff=8, C=C, ldc=ld, c_coff=8)
    check_f32(C, [(8, ref)])


# ------------------------------------------------------------------------------------------------ every instantiation, halo mode
HALO_MANY = [(bn, kb, cin, n) for (m, bn, kb) in sorted(engine_variants()) if m == HALO for cin, n in ((320, bn), (64, bn))] + [(256, 32, 128, 512)]


@pytest.mark.parametrize("bn,kb,cin,n", HALO_MANY)
def test_halo_instantiations_with_many_tiles_per_cta(bn, kb, cin, n):
    """Every halo-mode one-product instantiation at more than 2 x SM-count tiles, ragged in both directions: the one-plane halo
    double buffer (Cin = 320), resident weights in the deeper one-product ring (Cin = 64) and two N tiles (N = 512)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    H, W = 37, 45
    B = 2 * sms // (3 * 6 * (n // bn)) + 1
    g = torch.Generator().manual_seed(bn * 1000 + cin)
    args, ref = halo_problem(g, B, H, W, cin, n)
    M = B * H * W
    C = nan32(M + SPARE, n + 8)
    op = tma_bf16(C=C, ldc=n + 8, c_coff=4, force_bn=bn, force_kb=kb, **args)
    assert (op.picked_bn, op.picked_kb) == (bn, kb)
    check_f32(C, [(4, ref)])


def test_halo_instantiations_compute_the_same_bits():
    g = torch.Generator().manual_seed(78)
    args, ref = halo_problem(g, 2, 20, 13, 128, 256)
    outs = {}
    for m, bn, kb in sorted(engine_variants()):
        if m != HALO:
            continue
        C = nan32(2 * 20 * 13 + SPARE, 256)
        tma_bf16(C=C, ldc=256, force_bn=bn, force_kb=kb, **args)
        check_f32(C, [(0, ref)])
        outs[(bn, kb)] = C
    first = next(iter(outs))
    assert all(torch.equal(v.view(torch.int32), outs[first].view(torch.int32)) for v in outs.values())


@pytest.mark.parametrize("hw", [(10, 10), (11, 7), (2, 2)])
def test_border_class_bias_and_rectified_split(hw):
    """Nine border-class biases (bias_mode 2: class (ry * 3 + rx) of the pixel), N = 512 in two N tiles, C and split_relu planes."""
    H, W = hw
    B, Cin, N = 2, 128, 512
    g = torch.Generator().manual_seed(H * 100 + W)
    args, _ = halo_problem(g, B, H, W, Cin, N)
    bias9 = rn(g, 9 * N)
    a = args["a_hi"].double()
    w = args["w_hi"].double()
    ry = torch.ones(H, dtype=torch.long)
    ry[0], ry[-1] = 0, 2
    rx = torch.ones(W, dtype=torch.long)
    rx[0], rx[-1] = 0, 2
    cls = (ry[:, None] * 3 + rx[None, :]).reshape(-1).repeat(B).cuda()
    ref = conv3x3_ref(a, w, Cin) + bias9.view(9, N).double()[cls]
    M, ldc, lds = B * H * W, 520, 528
    C, shi, slo = nan32(M + SPARE, ldc), nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    tma_bf16(**dict(args, bias=bias9, bias_mode=2, C=C, ldc=ldc, c_coff=4, s_hi=shi, s_lo=slo, lds=lds, s_coff=8, split_relu=1))
    check_f32(C, [(4, ref)])
    check_split(shi, slo, [(8, C[:M, 4:4 + N])], True)


@pytest.mark.parametrize("shape", [(2, 20, 20), (1, 23, 17)])
def test_grouped_conv_with_two_residuals(shape):
    B, H, W = shape
    M, Cin, N = B * H * W, 256, 256
    g = torch.Generator().manual_seed(B * H * W)
    ahi, alo, a = split(rn(g, B, H, W, 512))
    whi, wlo, w = split(rn(g, 2 * N, 9 * Cin, scale=(9 * Cin) ** -0.5))
    bias = rn(g, 2 * N)
    res, res2 = rn(g, M, 544), rn(g, M, 512)
    ldc, c_coff, lds, s_coff = 560, 24, 528, 8
    C, shi, slo = nan32(M + SPARE, ldc), nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    tma_bf16(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=2, a_hi=ahi, a_lo=alo, lda=512, a_gc=256, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1,
             bias_gstride=256, res=res, ldr=544, r_coff=16, r_gcoff=256, res_relu=1, res2=res2, ldr2=512, r2_gcoff=256,
             C=C, ldc=ldc, c_coff=c_coff, c_gcoff=256, s_hi=shi, s_lo=slo, lds=lds, s_coff=s_coff, s_gcoff=256, split_relu=1)
    refs = []
    for gi in range(2):
        r = conv3x3_ref(a[..., 256 * gi:256 * gi + 256], w[N * gi:N * gi + N], Cin) + bias[N * gi:N * gi + N].double()
        r = r + F.relu(res[:, 16 + 256 * gi:16 + 256 * gi + N]).double() + res2[:, 256 * gi:256 * gi + N].double()
        refs.append((c_coff + 256 * gi, r))
    check_f32(C, refs)
    check_split(shi, slo, [(s_coff + 256 * gi, C[:M, c_coff + 256 * gi:c_coff + 256 * gi + N]) for gi in range(2)], True)


@pytest.mark.parametrize("shape", [(2, 24, 24), (1, 19, 13)])
def test_dual_source(shape):
    """Input channels 0-255 from A (group block of 256), 256-319 from A2 (hi plane only read), ReLU, split planes."""
    B, H, W = shape
    M, Cin, N = B * H * W, 320, 64
    g = torch.Generator().manual_seed(M)
    ahi, alo, a = split(rn(g, B, H, W, 512))
    a2hi, a2lo, a2 = split(rn(g, B, H, W, 64))
    whi, wlo, w = split(rn(g, 2 * N, 9 * Cin, scale=(9 * Cin) ** -0.5))
    bias = rn(g, 2 * N)
    lds = 144
    shi, slo = nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    tma_bf16(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=2, a_hi=ahi, a_lo=alo, lda=512, a_gc=256, a2_hi=a2hi, a2_lo=a2lo, lda2=64,
             c_split=256, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1, bias_gstride=N, act=1, s_hi=shi, s_lo=slo, lds=lds, s_coff=8, s_gcoff=N)
    got = (shi.double() + slo.double())[:M]
    owned = torch.zeros_like(shi, dtype=torch.bool)
    for gi in range(2):
        x = torch.cat([a[..., 256 * gi:256 * gi + 256], a2], -1)
        ref = F.relu(conv3x3_ref(x, w[N * gi:N * gi + N], Cin) + bias[N * gi:N * gi + N].double())
        c0 = 8 + N * gi
        assert U.rel_err(got[:, c0:c0 + N], ref) < TOL, gi
        owned[:M, c0:c0 + N] = True
    assert untouched(shi)[~owned].all() and untouched(slo)[~owned].all()


@pytest.mark.parametrize("bhw", [(1, 2, 2), (2, 10, 18), (2, 160, 160)])
def test_phase4_with_prediction_tails(bhw):
    """The phase-composed conv1 launch (N = 4 phases x 32 per head, groups = 2, resident weights, fused prediction tails): chunk
    ph of low-res pixel (y, x) is hi-res pixel (2y + ph / 2, 2x + ph % 2).  Restated as a 3x3 conv with the composed weights'
    hi plane on the input's hi plane, then the same tails in float64."""
    B, H, W = bhw
    H2, W2, P2 = 2 * H, 2 * W, 4 * B * H * W
    g = torch.Generator().manual_seed(B * H * W + 1)
    chi, clo, c = split(F.relu(rn(g, B, H, W, 128)))
    whi, wlo, w = split(rn(g, 256, 9 * 64, scale=(9 * 64) ** -0.5))
    bias = rn(g, 256)
    pgw, pgb, plw, plb = rn(g, 2 * 32, scale=0.3), rn(g, 2), rn(g, 32, scale=0.3), rn(g, 1)
    C = nan32(P2 + SPARE, 64)
    pg, pl = nan32(B, 2, H2, W2), nan32(B, 1, H2, W2)
    op = tma_bf16(mode=HALO, B=B, H=H, W=W, Cin=64, N=128, groups=2, a_hi=chi, a_lo=clo, lda=128, a_gc=64, w_hi=whi, w_lo=wlo, bias=bias,
                  bias_mode=1, bias_gstride=128, act=1, phase4=1, C=C, ldc=64, c_gcoff=32, pred=[(pgw, pgb, pg, 2, 1), (plw, plb, pl, 1, 2)])
    assert (op.picked_bn, op.picked_kb) == (128, 64)
    ys = []
    for gi in range(2):
        y = F.relu(conv3x3_ref(c[..., 64 * gi:64 * gi + 64], w[128 * gi:128 * gi + 128], 64) + bias[128 * gi:128 * gi + 128].double())
        ys.append(y.view(B, H, W, 2, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(B, H2, W2, 32))
    ref = torch.cat(ys, -1).reshape(P2, 64)
    check_f32(C, [(0, ref)])
    y0 = ys[0].permute(0, 3, 1, 2)
    v = F.conv2d(y0, pgw.double().view(2, 32, 1, 1), pgb.double())
    nrm = v.norm(dim=1, keepdim=True)
    ok = (nrm > 0.05 * nrm.max()).expand_as(pg)
    assert ok.float().mean() > 0.5
    assert ((pg.double() - F.normalize(v, dim=1)) * nrm / nrm.max())[ok].abs().max() < 1e-5
    lat = F.conv2d(ys[1].permute(0, 3, 1, 2), plw.double().view(1, 32, 1, 1), plb.double()).clamp(-1, 1)
    assert U.rel_err(pl, lat) < 1e-5


def test_every_one_product_instantiation_was_launched():
    """Runs after the tests above (file order): together they launched every (mode, bn, kb), GEMM mode in both schedules."""
    want = {(m, bn, kb, s) for (m, bn, kb) in engine_variants() for s in ((1, 2) if m == GEMM else (0,))}
    assert want <= LAUNCHED, sorted(want - LAUNCHED)


def test_resident_rule_follows_the_one_product_ring():
    """Cin = 64 with N = 128 in 64-wide tiles: the three-product ring (6 stages) streams the 9 taps, so two N tiles are fine; the
    one-product ring (16 stages) keeps them resident, which needs one N tile per launch: refused before anything runs."""
    L = _native.lib()
    g = torch.Generator().manual_seed(1)
    args, ref = halo_problem(g, 1, 8, 8, 64, 128)
    C = nan32(64 + SPARE, 128)
    _native.check(L.pf_op_tma(ctypes.byref(op_struct(C=C, ldc=128, force_bn=64, force_kb=64, **args)), U.stream_ptr()))
    torch.cuda.synchronize()
    C1 = nan32(64 + SPARE, 128)
    before = L.pf_kernel_launch_count()
    assert L.pf_op_tma_bf16(ctypes.byref(op_struct(C=C1, ldc=128, force_bn=64, force_kb=64, **args)), U.stream_ptr()) == -1
    assert "one N tile" in L.pf_last_error().decode()
    assert L.pf_kernel_launch_count() == before
    assert untouched(C1).all()


# ------------------------------------------------------------------------------------------------ attention core
def test_attention_one_product():
    """pf_op_attention_tc_bf16 against float64 with bf16-rounded q, k, v and P.  The kernel rounds P = exp(s - max) (fp32, before
    the 1 / l normalisation) to bf16; float64 rounding of the same P can land one bf16 ulp away where fp32's exp sits next to a
    rounding midpoint (about one element in 4000).  One such flip of key i moves the output row by at most
    ulp(P_i) |v_i| / l <= 2^-8 max|v| / l (P <= 1, so one bf16 ulp of P is at most 2^-8); the bound allows three per row, plus
    1e-5 relative for fp32 accumulation."""
    g = torch.Generator().manual_seed(9)
    B, N, C, heads = 2, 400, 128, 2
    q, kv = rn(g, B, N, C, scale=2.0), rn(g, B, 100, 2 * C)
    out = torch.empty(B, N, C, device="cuda")
    _native.check(_native.lib().pf_op_attention_tc_bf16(q.data_ptr(), kv.data_ptr(), out.data_ptr(), B, N, C, heads, U.stream_ptr()))
    torch.cuda.synchronize()
    r = lambda t: t.bfloat16().double()
    qh, kh, vh = r(q), r(kv[..., :C]), r(kv[..., C:])
    for h in range(heads):
        sl = slice(64 * h, 64 * h + 64)
        s = qh[..., sl] @ kh[..., sl].transpose(1, 2) / 8
        p = torch.exp(s - s.amax(-1, keepdim=True))
        l = p.sum(-1, keepdim=True)
        ref = (r(p) @ vh[..., sl]) / l
        bound = 3 * 2.0 ** -8 * vh[..., sl].abs().max() / l + 1e-5 * ref.abs().max()
        err = (out[..., sl].double() - ref).abs()
        assert (err <= bound).all(), (err / bound).max().item()
        # without the rounding of q, k, v and P the result is measurably elsewhere: one product ran on bf16 operands
        qf, kf, vf = q.double(), kv[..., :C].double(), kv[..., C:].double()
        ex = torch.softmax(qf[..., sl] @ kf[..., sl].transpose(1, 2) / 8, -1) @ vf[..., sl]
        assert 10 * err.mean() < (out[..., sl].double() - ex).abs().mean()


# ------------------------------------------------------------------------------------------------ end to end
_models = {}


def model(version, **kw):
    key = (version, tuple(sorted(kw.items())))
    if key not in _models:
        _models[key] = U.make_model(version, model_kwargs=dict(kw, precision="bf16"))
    return _models[key]


@pytest.mark.parametrize("version", ["Paramnet-360Cities-edina-centered", "Paramnet-360Cities-edina-uncentered",
                                     "PersNet_Paramnet-GSV-uncentered", "PersNet_Paramnet-GSV-centered"])
def test_regression_variants_within_the_emulated_bounds(version):
    """Mixed image sizes in one call (480 x 640 and 360 x 500)."""
    m, sd = model(version)
    imgs = golden_images()
    out = m.inference_batch(imgs)
    ora = om.inference_batch(sd, version, imgs)
    table = error_table(out, ora)
    print(version, {k: round(v, 4) for k, v in table.items()})
    assert {"pred_gravity", "pred_latitude", "pred_gravity_original", "pred_latitude_original", "pred_roll", "pred_pitch"} <= set(table)
    for k, e in table.items():
        assert e < (DEG_BOUND if k in ANGLE_KEYS else REL_BOUND), (version, k, e)


def _stable_decoded_fields(out, ora, err_of):
    """The argmax-decoded fields on the pixels whose top-2 logit margin exceeds 4x the logit error (pf_test_util.stable_mask).  The
    bf16 logit error is about 10x the fp32 path's, so fewer pixels qualify than in test_gpu_forward.py (0.47 of the resampled
    latitude field of the larger golden image)."""
    for o, r in zip(out, ora):
        h, w = r["pred_latitude_original"].shape
        for key, okey, scale in (("pred_gravity", "pred_gravity_original", 1.0), ("pred_latitude", "pred_latitude_original", 90.0)):
            stable = U.stable_mask(r[key], err_of(key), h, w)
            frac = stable.float().mean().item()
            assert frac > 0.25, (okey, frac)
            d = (o[okey].cpu() - r[okey]).abs()
            d = d.amax(0) if d.ndim == 3 else d
            assert d[stable].max().item() / scale < 1e-3, okey


def test_classification_variant_with_and_without_logits():
    version = "PersNet-360Cities"
    m, sd = model(version)
    imgs = golden_images()
    out = m.inference_batch(imgs)
    ora = om.inference_batch(sd, version, imgs)
    table = error_table(out, ora, classification=True)
    print(version, {k: round(v, 4) for k, v in table.items()})
    assert table["pred_gravity"] < REL_BOUND and table["pred_latitude"] < REL_BOUND
    errs = {k: max((o[k].cpu() - r[k]).abs().max().item() for o, r in zip(out, ora)) for k in ("pred_gravity", "pred_latitude")}
    _stable_decoded_fields(out, ora, errs.get)
    m2, _ = model(version, logits=False)
    dec = m2.inference_batch(imgs)
    for o, b, r in zip(dec, out, ora):
        assert tuple(o["pred_gravity"].shape) == (2, 320, 320) and tuple(o["pred_latitude"].shape) == (1, 320, 320)
        # the same bf16 forward up to the logits: the decode of its own logits, bit for bit in the resampled fields
        idx_g, idx_l = b["pred_gravity"].argmax(0).cpu(), b["pred_latitude"].argmax(0).cpu()
        assert (o["pred_gravity"].cpu() - om.decode_bin(idx_g, 73)).abs().max() < 2e-6
        assert torch.equal(o["pred_latitude"].cpu()[0], om.decode_bin_latitude(idx_l, 180))
        assert torch.equal(o["pred_gravity_original"], b["pred_gravity_original"])
        assert torch.equal(o["pred_latitude_original"], b["pred_latitude_original"])
    _stable_decoded_fields(dec, ora, errs.get)


def test_switching_precision_on_one_model():
    """default -> bf16 -> default on one engine: the default runs are bit-identical to each other and to a fresh default model,
    two bf16 runs are bit-identical to each other, and bf16 does differ from the default."""
    version = "Paramnet-360Cities-edina-centered"
    imgs = golden_images()
    m, _ = U.make_model(version)
    fresh, _ = U.make_model(version)

    def run(mod):
        return [{k: v.clone() for k, v in o.items() if isinstance(v, torch.Tensor)} for o in mod.inference_batch(imgs)]

    def same(a, b):
        return all(torch.equal(x[k].reshape(-1).view(torch.int32), y[k].reshape(-1).view(torch.int32)) for x, y in zip(a, b) for k in x)

    d1 = run(m)
    m.set_option("bf16", 1)
    b1, b2 = run(m), run(m)
    m.set_option("bf16", 0)
    d2 = run(m)
    ref = run(fresh)
    assert same(d1, d2) and same(d1, ref)
    assert same(b1, b2)
    assert not same(b1, d1)
    assert U.rel_err(b1[0]["pred_gravity"], d1[0]["pred_gravity"]) < REL_BOUND


def test_precision_survives_engine_recreation():
    """precision="bf16" is an engine option of the model: .to() / load_state_dict re-create the engine with it."""
    version = "Paramnet-360Cities-edina-centered"
    m, sd = model(version)
    imgs = golden_images()[:1]
    a = m.inference_batch(imgs)[0]["pred_gravity"].clone()
    m.load_state_dict(m.state_dict())
    b = m.inference_batch(imgs)[0]["pred_gravity"]
    assert torch.equal(a, b)
    d, _ = U.make_model(version)
    assert not torch.equal(d.inference_batch(imgs)[0]["pred_gravity"], a)
