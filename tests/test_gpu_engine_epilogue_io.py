"""GPU: how the TMA -> wgmma engine's epilogue moves fp32 data between registers and HBM.  The fp32 output and the residuals go
through the warpgroup's staging rows as whole row segments; these tests drive pf_op_tma through every tile-shape instantiation
of both modes and both GEMM-mode schedules, on ragged problems, and check each launch against a float64 restatement (5e-5
relative) and all launches of a problem against each other bit for bit.

Covered: fp32 output alone; fp32 output and split planes; one residual written in place (res == C) with layer scale; a
rectified residual in its own buffer; two residuals with per-group column offsets (halo mode, two groups).  Every output is
wider than the launch's region, at a column offset, with spare rows behind it, and NaN-filled: what a launch does not own must
keep the NaN bit pattern."""
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
COOP, PINGPONG = 1, 2
SPARE = 200


def variants(mode):
    """(BN, KB) of every instantiation of `mode` in PF_TMA_VARIANTS and, for GEMM mode, PF_TMA_PINGPONG_VARIANTS, with the
    schedule to force: [(sched, BN, KB)]."""
    src = open(os.path.join(_native.SRC_DIR, "tma_host.cuh")).read()

    def body(name):
        b = src[src.index(f"#define {name}(X)"):]
        return b[:b.index("\n\n")]
    name = "GEMM" if mode == GEMM else "HALO"
    out = [(COOP if mode == GEMM else 0, int(bn), int(kb))
           for bn, m, kb in re.findall(r"X\((\d+), MODE_(GEMM|HALO), (\d+)\)", body("PF_TMA_VARIANTS")) if m == name]
    if mode == GEMM:
        out += [(PINGPONG, int(bn), int(kb)) for bn, kb in re.findall(r"X\((\d+), (\d+)\)", body("PF_TMA_PINGPONG_VARIANTS"))]
    return sorted(set(out))


def rn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).cuda()


def split(x):
    hi, lo = weights.split_hi_lo(x)
    return hi, lo, hi.double() + lo.double()


def nan32(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def nan16(*shape):
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda")


def untouched(t):
    it = torch.int32 if t.dtype == torch.float32 else torch.int16
    return t.view(it) == torch.full_like(t, float("nan")).view(it)


def tma(**kw):
    op = _native.pf_tma_op()
    for k, v in kw.items():
        setattr(op, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    _native.check(_native.lib().pf_op_tma(ctypes.byref(op), U.stream_ptr()))
    torch.cuda.synchronize()
    return op


def conv3x3_ref(x_nhwc, w_nk, cin):
    """x: [B, H, W, cin] float64; w: [N, 9 * cin] ordered (ky, kx, ci) -> [B * H * W, N]."""
    B, H, W, _ = x_nhwc.shape
    w = w_nk.reshape(-1, 3, 3, cin).permute(0, 3, 1, 2)
    y = F.conv2d(x_nhwc.permute(0, 3, 1, 2), w, padding=1)
    return y.permute(0, 2, 3, 1).reshape(B * H * W, -1)


def check_f32(buf, regions):
    owned = torch.zeros_like(buf, dtype=torch.bool)
    for c0, ref in regions:
        got = buf[:ref.shape[0], c0:c0 + ref.shape[1]]
        assert torch.isfinite(got).all(), "an owned element was not written"
        assert U.rel_err(got, ref) < TOL, (c0, U.rel_err(got, ref))
        owned[:ref.shape[0], c0:c0 + ref.shape[1]] = True
    assert untouched(buf)[~owned].all(), "a store landed outside the launch's region"


def check_split(shi, slo, regions, relu):
    owned = torch.zeros_like(shi, dtype=torch.bool)
    for c0, c in regions:
        hi, lo = weights.split_hi_lo(F.relu(c) if relu else c)
        rows, n = c.shape
        assert torch.equal(shi[:rows, c0:c0 + n].view(torch.int16), hi.view(torch.int16))
        assert torch.equal(slo[:rows, c0:c0 + n].view(torch.int16), lo.view(torch.int16))
        owned[:rows, c0:c0 + n] = True
    assert untouched(shi)[~owned].all() and untouched(slo)[~owned].all()


def same_bits(outs):
    first = next(iter(outs))
    for k, bufs in outs.items():
        for a, b in zip(bufs, outs[first]):
            it = torch.int32 if a.dtype == torch.float32 else torch.int16
            assert torch.equal(a.view(it), b.view(it)), f"{k} differs from {first}"


# ------------------------------------------------------------------------------------------------ GEMM mode
GEMM_CASES = ["c", "c_split", "res_in_place", "res_relu"]


@pytest.mark.parametrize("case", GEMM_CASES)
def test_gemm_mode_epilogue_io(case):
    """M = 1000: the last 128-row tile has 104 rows and the last 64-row (ping-pong) tile 40.  N = 480: a partial last N tile for
    most widths, and a 32-column last round for the widths that are odd multiples of 32."""
    g = torch.Generator().manual_seed(GEMM_CASES.index(case) + 1)
    M, K, N = 1000, 320, 480
    # row pitches and column offsets are multiples of 16 bytes, as the engine's vector loads and stores need
    ldc, c_coff, lds, s_coff, ldr, r_coff = 520, 20, 504, 8, 496, 12
    ahi, alo, a = split(rn(g, M, K))
    whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
    bias = rn(g, N)
    args = dict(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1,
                ldc=ldc, c_coff=c_coff)
    ref = a @ w.t() + bias.double()
    resv = None
    if case == "res_in_place":
        gamma = (torch.rand(N, generator=g) * 0.4 + 0.1).cuda()
        resv = rn(g, M, N)
        ref = ref * gamma.double() + resv.double()
        args.update(gamma=gamma, ldr=ldc, r_coff=c_coff)
    elif case == "res_relu":
        res = rn(g, M, ldr)
        ref = F.relu(ref) + F.relu(res[:, r_coff:r_coff + N]).double()
        args.update(act=1, res=res, ldr=ldr, r_coff=r_coff, res_relu=1)
    outs = {}
    for sched, bn, kb in variants(GEMM):
        C = nan32(M + SPARE, ldc)
        if resv is not None:
            C[:M, c_coff:c_coff + N] = resv
            args["res"] = C
        bufs = [C]
        if case == "c_split":
            shi, slo = nan16(M + SPARE, lds), nan16(M + SPARE, lds)
            args.update(s_hi=shi, s_lo=slo, lds=lds, s_coff=s_coff)
            bufs += [shi, slo]
        op = tma(C=C, force_bn=bn, force_kb=kb, force_sched=sched, **{k: v for k, v in args.items() if k != "C"})
        assert (op.picked_sched, op.picked_bn, op.picked_kb) == (sched, bn, kb)
        check_f32(C, [(c_coff, ref)])
        if case == "c_split":
            check_split(shi, slo, [(s_coff, C[:M, c_coff:c_coff + N])], False)
        outs[(sched, bn, kb)] = bufs
    same_bits(outs)


# ------------------------------------------------------------------------------------------------ halo mode
HALO_CASES = ["c", "c_split", "res_in_place", "two_res"]


@pytest.mark.parametrize("hw", [(10, 10), (11, 7)])
@pytest.mark.parametrize("case", HALO_CASES)
def test_halo_mode_epilogue_io(case, hw):
    """Two groups of 128 input and 128 output channels (group blocks in 256-wide rows), ragged 16 x 8 tiles in both directions.
    The BN = 256 instantiation covers both groups' columns with one tile per group, half of whose columns are past N."""
    H, W = hw
    B, Cin, N, G = 2, 128, 128, 2
    M = B * H * W
    g = torch.Generator().manual_seed(100 * HALO_CASES.index(case) + H * W)
    ldc, c_coff, lds, s_coff = G * N + 24, 8, G * N + 16, 16
    ahi, alo, a = split(rn(g, B, H, W, G * Cin))
    whi, wlo, w = split(rn(g, G * N, 9 * Cin, scale=(9 * Cin) ** -0.5))
    bias = rn(g, G * N)
    args = dict(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=G, a_hi=ahi, a_lo=alo, lda=G * Cin, a_gc=Cin, w_hi=whi, w_lo=wlo,
                bias=bias, bias_mode=1, bias_gstride=N, ldc=ldc, c_coff=c_coff, c_gcoff=N)
    refs = [conv3x3_ref(a[..., Cin * gi:Cin * gi + Cin], w[N * gi:N * gi + N], Cin) + bias[N * gi:N * gi + N].double() for gi in range(G)]
    resv = None
    if case == "res_in_place":
        resv = rn(g, M, G * N)
        refs = [r + resv[:, N * gi:N * gi + N].double() for gi, r in enumerate(refs)]
        args.update(ldr=ldc, r_coff=c_coff, r_gcoff=N)
    elif case == "two_res":
        ldr, r_coff, ldr2, r2_coff = G * N + 20, 12, G * N + 8, 4
        res, res2 = rn(g, M, ldr), rn(g, M, ldr2)
        refs = [r + F.relu(res[:, r_coff + N * gi:r_coff + N * gi + N]).double() + res2[:, r2_coff + N * gi:r2_coff + N * gi + N].double()
                for gi, r in enumerate(refs)]
        args.update(res=res, ldr=ldr, r_coff=r_coff, r_gcoff=N, res_relu=1, res2=res2, ldr2=ldr2, r2_coff=r2_coff, r2_gcoff=N)
    split_out = case in ("c_split", "two_res")
    outs = {}
    for _, bn, kb in variants(HALO):
        C = nan32(M + SPARE, ldc)
        if resv is not None:
            C[:M, c_coff:c_coff + G * N] = resv
            args["res"] = C
        bufs = [C]
        if split_out:
            shi, slo = nan16(M + SPARE, lds), nan16(M + SPARE, lds)
            args.update(s_hi=shi, s_lo=slo, lds=lds, s_coff=s_coff, s_gcoff=N, split_relu=int(case == "two_res"))
            bufs += [shi, slo]
        op = tma(C=C, force_bn=bn, force_kb=kb, **{k: v for k, v in args.items() if k != "C"})
        assert (op.picked_bn, op.picked_kb) == (bn, kb)
        check_f32(C, [(c_coff + N * gi, r) for gi, r in enumerate(refs)])
        if split_out:
            check_split(shi, slo, [(s_coff + N * gi, C[:M, c_coff + N * gi:c_coff + N * gi + N]) for gi in range(G)], case == "two_res")
        outs[(bn, kb)] = bufs
    same_bits(outs)
