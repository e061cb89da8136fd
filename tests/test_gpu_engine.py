"""GPU: the TMA -> wgmma engine at kernel precision, through pf_op_tma (one engine launch with every epilogue feature the forward
graph uses) and pf_op_conv1_ring, against float64 torch restatements of the same operations on the exact operand values the
kernels read (hi + lo of the split planes).  Bar: 5e-5 relative, as in test_gpu_ops.py.

Every output buffer is wider than the launch's region (row pitch > N, non-zero column offsets, spare rows at the end) and
filled with NaN first: what the launch owns must be finite and right, everything else must still hold the NaN bit pattern."""
import ctypes
import os
import re

import pytest
import torch
import torch.nn.functional as F

import pf_test_util as U
from perspectivefields_b200 import _native, weights

pytestmark = pytest.mark.gpu

TOL = 5e-5
GEMM, HALO = 0, 1
SPARE = 200          # spare rows behind every output: stores from rows past the end land there
LAUNCHED = set()     # (mode, bn, kb) of every successful pf_op_tma call of this module


def engine_variants():
    """(mode, BN, KB) of every instantiation listed in PF_TMA_VARIANTS (csrc/tma_host.cuh)."""
    src = open(os.path.join(_native.SRC_DIR, "tma_host.cuh")).read()
    body = src[src.index("#define PF_TMA_VARIANTS(X)"):]
    body = body[:body.index("\n\n")]
    return {(GEMM if m == "GEMM" else HALO, int(bn), int(kb)) for bn, m, kb in re.findall(r"X\((\d+), MODE_(GEMM|HALO), (\d+)\)", body)}


def rn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).cuda()


def split(x):
    """-> (hi, lo, hi + lo in float64): the planes a producer kernel writes and the value the engine multiplies."""
    hi, lo = weights.split_hi_lo(x)
    return hi, lo, hi.double() + lo.double()


def nan32(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def nan16(*shape):
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda")


def untouched(t):
    """Elementwise: still the NaN fill pattern (compared as bits)."""
    it = torch.int32 if t.dtype == torch.float32 else torch.int16
    return t.view(it) == torch.full_like(t, float("nan")).view(it)


def op_struct(**kw):
    op = _native.pf_tma_op()
    preds = kw.pop("pred", None)
    for k, v in kw.items():
        setattr(op, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    for g, (w, b, out, nc, mode) in enumerate(preds or []):
        op.pred[g].w, op.pred[g].b, op.pred[g].out, op.pred[g].nc, op.pred[g].mode = w.data_ptr(), b.data_ptr(), out.data_ptr(), nc, mode
    op.npred = len(preds or [])
    return op


def tma(**kw):
    op = op_struct(**kw)
    _native.check(_native.lib().pf_op_tma(ctypes.byref(op), U.stream_ptr()))
    torch.cuda.synchronize()
    LAUNCHED.add((op.mode, op.picked_bn, op.picked_kb))
    return op


def conv3x3_ref(x_nhwc, w_nk, cin):
    """x: [B, H, W, cin] float64; w: [N, 9 * cin] ordered (ky, kx, ci) -> [B * H * W, N]."""
    B, H, W, _ = x_nhwc.shape
    w = w_nk.reshape(-1, 3, 3, cin).permute(0, 3, 1, 2)
    y = F.conv2d(x_nhwc.permute(0, 3, 1, 2), w, padding=1)
    return y.permute(0, 2, 3, 1).reshape(B * H * W, -1)


def check_f32(buf, regions, tol=TOL):
    """buf: [rows, ld] fp32; regions: (first column, reference [rows', n]) pairs the launch owns (rows 0 .. rows'-1)."""
    owned = torch.zeros_like(buf, dtype=torch.bool)
    for c0, ref in regions:
        got = buf[:ref.shape[0], c0:c0 + ref.shape[1]]
        assert torch.isfinite(got).all(), "an owned element was not written"
        assert U.rel_err(got, ref) < tol, (c0, U.rel_err(got, ref))
        owned[:ref.shape[0], c0:c0 + ref.shape[1]] = True
    assert untouched(buf)[~owned].all(), "a store landed outside the launch's region"


def check_split(shi, slo, regions, relu):
    """S planes == weights.split_hi_lo(relu?(C)) bit for bit on the regions (first column, C values), NaN elsewhere."""
    owned = torch.zeros_like(shi, dtype=torch.bool)
    for c0, c in regions:
        hi, lo = weights.split_hi_lo(F.relu(c) if relu else c)
        rows, n = c.shape
        assert torch.equal(shi[:rows, c0:c0 + n].view(torch.int16), hi.view(torch.int16))
        assert torch.equal(slo[:rows, c0:c0 + n].view(torch.int16), lo.view(torch.int16))
        owned[:rows, c0:c0 + n] = True
    assert untouched(shi)[~owned].all() and untouched(slo)[~owned].all()


@pytest.fixture(scope="module")
def repacked():
    """Repacked weights of a synthetic checkpoint whose gravity head is driven by its weights (the field turns), as the forward
    loads them: weights.repack on a reference-layout state dict."""
    from oracle import weights_gen as wg
    from perspectivefields_b200.variants import VARIANTS

    version = "Paramnet-360Cities-edina-centered"
    sd = wg.synth_state_dict(version, 3, gravity_bias=(0.0, 0.0), gravity_gain=0.8)
    return sd, {k: v.cuda() for k, v in weights.repack(sd, VARIANTS[version]).items()}


# ------------------------------------------------------------------------------------------------ split output planes
@pytest.mark.parametrize("split_relu", [0, 1])
@pytest.mark.parametrize("mode", ["gemm", "halo"])
def test_split_planes_are_exact_and_independent_of_c(mode, split_relu):
    """Odd M (GEMM) / odd W and H % 16 != 0 (halo): the last row / pixel pair of the lane-pair store exchange has one valid
    partner.  S must be the exact split of relu?(C), and the same whether or not C is written."""
    g = torch.Generator().manual_seed(11 + split_relu)
    N, ldc, c_coff, lds, s_coff = 96, 136, 20, 120, 16
    if mode == "gemm":
        M, K = 333, 128
        ahi, alo, a = split(rn(g, M, K + 32))
        geo = dict(mode=GEMM, M=M, K=K, a_c0=32)
    else:
        B, H, W, K = 2, 21, 13, 64
        M = B * H * W
        ahi, alo, a = split(rn(g, B, H, W, K))
        geo = dict(mode=HALO, B=B, H=H, W=W, Cin=K)
    kk = K if mode == "gemm" else 9 * K
    whi, wlo, w = split(rn(g, N, kk, scale=kk ** -0.5))
    bias = rn(g, N)
    acc = a[:, 32:] @ w.t() if mode == "gemm" else conv3x3_ref(a, w, K)
    ref = acc + bias.double()
    C, shi, slo = nan32(M + SPARE, ldc), nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    args = dict(geo, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=ahi.shape[-1], w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1,
                ldc=ldc, c_coff=c_coff, s_hi=shi, s_lo=slo, lds=lds, s_coff=s_coff, split_relu=split_relu)
    tma(C=C, **args)
    check_f32(C, [(c_coff, ref)])
    check_split(shi, slo, [(s_coff, C[:M, c_coff:c_coff + N])], split_relu)
    shi2, slo2 = nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    tma(**dict(args, s_hi=shi2, s_lo=slo2))
    assert torch.equal(shi2.view(torch.int16), shi.view(torch.int16)) and torch.equal(slo2.view(torch.int16), slo.view(torch.int16))


# ------------------------------------------------------------------------------------------------ border-class bias
@pytest.mark.parametrize("hw", [(10, 10), (11, 7), (2, 2)])
def test_border_class_bias_of_the_composed_proc_conv(hw, repacked):
    """head.proc2 (linear_c2 o linear_c2_proc of both heads, N = 512, nine border-class biases) == conv3x3(linear(x)) with the
    768-wide intermediate in float64, as the forward launches it (C and the rectified split planes)."""
    sd, rp = repacked
    H, W = hw
    B, Cin, N = 2, 128, 512
    g = torch.Generator().manual_seed(H * 100 + W)
    ahi, alo, a = split(rn(g, B, H, W, Cin))
    ref = []
    for head in ("gravity_head", "latitude_head"):
        p = f"persformer_heads.{head}."
        t = a @ sd[p + "linear_c2.proj.weight"].double().cuda().t() + sd[p + "linear_c2.proj.bias"].double().cuda()
        y = F.conv2d(t.permute(0, 3, 1, 2), sd[p + "linear_c2_proc.weight"].double().cuda(), sd[p + "linear_c2_proc.bias"].double().cuda(), padding=1)
        ref.append(y.permute(0, 2, 3, 1).reshape(B * H * W, 256))
    ref = torch.cat(ref, 1)
    M, ldc, lds = B * H * W, 520, 528
    C, shi, slo = nan32(M + SPARE, ldc), nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    tma(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=Cin, w_hi=rp["head.proc2.whi"], w_lo=rp["head.proc2.wlo"],
        bias=rp["head.proc2.b"], bias_mode=2, C=C, ldc=ldc, c_coff=4, s_hi=shi, s_lo=slo, lds=lds, s_coff=8, split_relu=1)
    check_f32(C, [(4, ref)])
    check_split(shi, slo, [(8, C[:M, 4:4 + N])], True)


# ------------------------------------------------------------------------------------------------ grouped RCU conv
@pytest.mark.parametrize("shape", [(2, 20, 20), (1, 23, 17)])
def test_grouped_rcu_conv_with_two_residuals(shape):
    """The RefineNet conv2 of both heads in one launch (groups = 2, channel blocks of 256 in 512-wide rows): + bias, +
    relu(res), + res2, C and split_relu planes, each group against its own reference."""
    B, H, W = shape
    M, Cin, N = B * H * W, 256, 256
    g = torch.Generator().manual_seed(B * H * W)
    ahi, alo, a = split(rn(g, B, H, W, 512))
    whi, wlo, w = split(rn(g, 2 * N, 9 * Cin, scale=(9 * Cin) ** -0.5))
    bias = rn(g, 2 * N)
    res, res2 = rn(g, M, 544), rn(g, M, 512)
    ldc, c_coff, lds, s_coff = 560, 24, 528, 8
    C, shi, slo = nan32(M + SPARE, ldc), nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    tma(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=2, a_hi=ahi, a_lo=alo, lda=512, a_gc=256, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1,
        bias_gstride=256, res=res, ldr=544, r_coff=16, r_gcoff=256, res_relu=1, res2=res2, ldr2=512, r2_gcoff=256,
        C=C, ldc=ldc, c_coff=c_coff, c_gcoff=256, s_hi=shi, s_lo=slo, lds=lds, s_coff=s_coff, s_gcoff=256, split_relu=1)
    refs = []
    for gi in range(2):
        r = conv3x3_ref(a[..., 256 * gi:256 * gi + 256], w[N * gi:N * gi + N], Cin) + bias[N * gi:N * gi + N].double()
        r = r + F.relu(res[:, 16 + 256 * gi:16 + 256 * gi + N]).double() + res2[:, 256 * gi:256 * gi + N].double()
        refs.append((c_coff + 256 * gi, r))
    check_f32(C, refs)
    check_split(shi, slo, [(s_coff + 256 * gi, C[:M, c_coff + 256 * gi:c_coff + 256 * gi + N]) for gi in range(2)], True)


# ------------------------------------------------------------------------------------------------ layer scale
def test_layer_scale_with_in_place_residual():
    """ConvNeXt pwconv2: x = gamma * (h W^T + b) + x, written in place over its own residual (C == res), GELU-free."""
    g = torch.Generator().manual_seed(5)
    M, K, N, ld = 777, 384, 96, 104
    ahi, alo, a = split(rn(g, M, K))
    whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
    bias, gamma = rn(g, N), (torch.rand(N, generator=g) * 0.4 + 0.1).cuda()
    C = nan32(M + SPARE, ld)
    C[:M, 8:8 + N] = rn(g, M, N)
    ref = (a @ w.t() + bias.double()) * gamma.double() + C[:M, 8:8 + N].double()
    tma(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1, gamma=gamma,
        res=C, ldr=ld, r_coff=8, C=C, ldc=ld, c_coff=8)
    check_f32(C, [(8, ref)])


# ------------------------------------------------------------------------------------------------ dual source
@pytest.mark.parametrize("shape", [(2, 24, 24), (1, 19, 13)])
def test_dual_source_conv0(shape):
    """conv_fuse_conv0: per head, input channels 0-255 from the fused feature (group block of 256 in 512-wide rows) and 256-319
    from the low-level feature (A2, 64-wide rows, the same for both groups); ReLU; split planes only."""
    B, H, W = shape
    M, Cin, N = B * H * W, 320, 64
    g = torch.Generator().manual_seed(M)
    ahi, alo, a = split(rn(g, B, H, W, 512))
    a2hi, a2lo, a2 = split(rn(g, B, H, W, 64))
    whi, wlo, w = split(rn(g, 2 * N, 9 * Cin, scale=(9 * Cin) ** -0.5))
    bias = rn(g, 2 * N)
    lds = 144
    shi, slo = nan16(M + SPARE, lds), nan16(M + SPARE, lds)
    tma(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=2, a_hi=ahi, a_lo=alo, lda=512, a_gc=256, a2_hi=a2hi, a2_lo=a2lo, lda2=64,
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


# ------------------------------------------------------------------------------------------------ phase conv + border ring
@pytest.mark.parametrize("bhw", [(1, 2, 2), (2, 3, 3), (2, 10, 18), (2, 160, 160)])
def test_phase_conv1_and_border_ring(bhw, repacked):
    """Default conv_fuse_conv1: the phase-composed conv on the H x W grid (N = 4 phases x 32 per head, fused prediction tails),
    then conv1_ring_kernel on the same stream, in the forward's order.  Together they must equal relu(conv3x3(bilinear_x2(c0)))
    on the whole 2H x 2W grid for both heads; the ring kernel overwrites what the phase tiles wrote on the ring.  At 160 x 160,
    batch 2, each group's launch has 400 tiles, several per CTA."""
    sd, rp = repacked
    B, H, W = bhw
    H2, W2, P2 = 2 * H, 2 * W, 4 * B * H * W
    g = torch.Generator().manual_seed(B * H * W)
    chi, clo, c = split(F.relu(rn(g, B, H, W, 128)))
    C = nan32(P2 + SPARE, 64)
    pg, pl = nan32(B, 2, H2, W2), nan32(B, 1, H2, W2)
    tails = [(rp["head.pred_g.w"], rp["head.pred_g.b"], pg, 2, 1), (rp["head.pred_l.w"], rp["head.pred_l.b"], pl, 1, 2)]
    op = tma(mode=HALO, B=B, H=H, W=W, Cin=64, N=128, groups=2, a_hi=chi, a_lo=clo, lda=128, a_gc=64, w_hi=rp["head.conv1p.whi"],
             w_lo=rp["head.conv1p.wlo"], bias=rp["head.conv1p.b"], bias_mode=1, bias_gstride=128, act=1, phase4=1, C=C, ldc=64, c_gcoff=32,
             pred=tails)
    assert (op.picked_bn, op.picked_kb) == (128, 64)
    _native.check(_native.lib().pf_op_conv1_ring(chi.data_ptr(), clo.data_ptr(), B, H, W, rp["head.conv1f.w"].data_ptr(), rp["head.conv1f.b"].data_ptr(),
                                                 C.data_ptr(), rp["head.pred_g.w"].data_ptr(), rp["head.pred_g.b"].data_ptr(), pg.data_ptr(),
                                                 rp["head.pred_l.w"].data_ptr(), rp["head.pred_l.b"].data_ptr(), pl.data_ptr(), U.stream_ptr()))
    torch.cuda.synchronize()
    u = F.interpolate(c.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
    ys, raw = [], []
    for gi, (head, pred) in enumerate((("gravity_head", "linear_pred_gravity"), ("latitude_head", "linear_pred_latitude"))):
        p = f"persformer_heads.{head}."
        y = F.relu(F.conv2d(u[:, 64 * gi:64 * gi + 64], sd[p + "conv_fuse_conv1.conv.weight"].double().cuda(),
                            sd[p + "conv_fuse_conv1.conv.bias"].double().cuda(), padding=1))
        ys.append(y)
        raw.append(F.conv2d(y, sd[p + pred + ".weight"].double().cuda(), sd[p + pred + ".bias"].double().cuda()))
    ref = torch.cat(ys, 1).permute(0, 2, 3, 1).reshape(P2, 64)
    check_f32(C, [(0, ref)])
    ring = torch.ones(H2, W2, dtype=torch.bool)
    ring[2:-2, 2:-2] = False
    assert U.rel_err(C[:P2].view(B, H2, W2, 64)[:, ring], ref.view(B, H2, W2, 64)[:, ring]) < TOL     # the overwrite landed
    assert torch.isfinite(pg).all() and torch.isfinite(pl).all()                                     # every pixel written
    # F.normalize divides the error of v by |v|: pixels with a small |v| are masked, the end-to-end error is weighed by |v| / max |v|,
    # and the tail's own arithmetic is checked on the conv1 values the kernels wrote
    nrm = raw[0].norm(dim=1, keepdim=True)
    ok = (nrm > 0.05 * nrm.max()).expand_as(pg)
    assert ok.float().mean() > 0.5
    assert ((pg.double() - F.normalize(raw[0], dim=1)) * nrm / nrm.max())[ok].abs().max() < 1e-5
    y_got = C[:P2, :32].double().reshape(B, H2, W2, 32).permute(0, 3, 1, 2)
    v_got = F.conv2d(y_got, sd["persformer_heads.gravity_head.linear_pred_gravity.weight"].double().cuda(),
                     sd["persformer_heads.gravity_head.linear_pred_gravity.bias"].double().cuda())
    assert (pg.double() - F.normalize(v_got, dim=1))[ok].abs().max() < 1e-5
    assert U.rel_err(pl, raw[1].clamp(-1, 1)) < 1e-5


# ------------------------------------------------------------------------------------------------ many tiles per CTA
def halo_problem(g, B, H, W, Cin, N):
    ahi, alo, a = split(rn(g, B, H, W, Cin))
    whi, wlo, w = split(rn(g, N, 9 * Cin, scale=(9 * Cin) ** -0.5))
    bias = rn(g, N)
    return dict(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=Cin, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1), \
        conv3x3_ref(a, w, Cin) + bias.double()


HALO_MANY = [(bn, kb, cin, n) for (m, bn, kb) in sorted(engine_variants()) if m == HALO for cin, n in ((320, bn), (64, bn))] + [(256, 32, 128, 512)]


@pytest.mark.parametrize("bn,kb,cin,n", HALO_MANY)
def test_halo_instantiations_with_many_tiles_per_cta(bn, kb, cin, n):
    """Every halo-mode instantiation at more than 2 x SM-count tiles: the halo double buffer (Cin = 320: 5 chunks, its phase
    parity changes from tile to tile), the weight ring, resident weights (Cin = 64) and, for N = 512, two N tiles."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    H, W = 37, 45                                            # 3 x 6 tiles per image, ragged in both directions
    per_image = 3 * 6 * (n // bn)
    B = 2 * sms // per_image + 1
    g = torch.Generator().manual_seed(bn * 1000 + cin)
    args, ref = halo_problem(g, B, H, W, cin, n)
    M = B * H * W
    C = nan32(M + SPARE, n + 8)
    op = tma(C=C, ldc=n + 8, c_coff=4, force_bn=bn, force_kb=kb, **args)
    assert (op.picked_bn, op.picked_kb) == (bn, kb)
    check_f32(C, [(4, ref)])


# ------------------------------------------------------------------------------------------------ tiling does not change results
def test_every_instantiation_computes_the_same_bits():
    """One GEMM problem (M = 1000, K = 320, N = 480: a partial last N tile for most widths) through every GEMM-mode
    instantiation and one halo problem through every halo-mode one: each within 5e-5 of float64, and all of a mode bit-identical
    (the K order of every output is the same whatever the tile).  The suite as a whole launches every instantiation."""
    g = torch.Generator().manual_seed(77)
    M, K, N = 1000, 320, 480
    ahi, alo, a = split(rn(g, M, K))
    whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
    bias = rn(g, N)
    gemm = dict(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1)
    problems = {GEMM: (gemm, a @ w.t() + bias.double(), M), HALO: halo_problem(g, 2, 20, 13, 128, 256) + (2 * 20 * 13,)}
    variants = engine_variants()
    for mode, (args, ref, rows) in problems.items():
        outs = {}
        for m, bn, kb in sorted(variants):
            if m != mode:
                continue
            C = nan32(rows + SPARE, args["N"])
            op = tma(C=C, ldc=args["N"], force_bn=bn, force_kb=kb, **args)
            assert (op.picked_bn, op.picked_kb) == (bn, kb)
            check_f32(C, [(0, ref)])
            outs[(bn, kb)] = C
        first = next(iter(outs))
        differ = [k for k, v in outs.items() if not torch.equal(v.view(torch.int32), outs[first].view(torch.int32))]   # (NaN spare rows)
        assert not differ, f"mode {mode}: {differ} differ from {first}"
    assert LAUNCHED == variants
    print("launched (mode, bn, kb):", sorted(LAUNCHED))


# ------------------------------------------------------------------------------------------------ argument validation
def test_invalid_launches_are_refused_before_anything_runs():
    L = _native.lib()
    g = torch.Generator().manual_seed(1)
    C = nan32(4096, 64)

    def refused(text, **kw):
        before = L.pf_kernel_launch_count()
        assert L.pf_op_tma(ctypes.byref(op_struct(**kw)), U.stream_ptr()) == -1
        assert text in L.pf_last_error().decode(), L.pf_last_error()
        assert L.pf_kernel_launch_count() == before

    args, _ = halo_problem(g, 1, 8, 8, 64, 64)
    bias9 = rn(g, 9 * 64)
    for h, w in ((1, 8), (8, 1)):           # a one-pixel edge is top and bottom at once: no border class expresses it
        refused("border-class bias needs H, W >= 2", **dict(args, H=h, W=w, bias=bias9, bias_mode=2, C=C, ldc=64))
    refused("one N tile", force_bn=32, force_kb=64, C=C, ldc=64, **args)     # resident weights over two N tiles
    refused("no engine instantiation", force_bn=96, force_kb=32, C=C, ldc=64, **args)
    refused("no engine instantiation", force_bn=256, force_kb=64, C=C, ldc=64, **args)
    refused("phase4 needs N = 128", phase4=1, C=C, ldc=64, **args)
    gemm, _ = halo_problem(g, 1, 8, 8, 64, 64)
    gemm.update(mode=GEMM, M=64, K=96, lda=576)
    refused("K must be a multiple of the K step", force_bn=64, force_kb=64, C=C, ldc=64, **gemm)
    torch.cuda.synchronize()
    assert untouched(C).all()
    x = nan16(2, 1, 8, 128)
    wf, bf = nan32(2 * 9 * 64 * 32), nan32(64)
    before = L.pf_kernel_launch_count()
    for h, w in ((1, 8), (8, 1)):
        assert L.pf_op_conv1_ring(x.data_ptr(), x.data_ptr(), 2, h, w, wf.data_ptr(), bf.data_ptr(), C.data_ptr(), *([None] * 6), U.stream_ptr()) == -1
        assert "H, W >= 2" in L.pf_last_error().decode()
    assert L.pf_kernel_launch_count() == before
