"""GPU: the two GEMM-mode schedules of the TMA -> wgmma engine (cooperative: 128-row tiles shared by both MMA warpgroups;
ping-pong: 64-row tiles, alternate tiles per warpgroup) through pf_op_tma's force_sched, against float64 restatements at 5e-5
and against each other bit for bit (the K order of every output is the same in both schedules and at every tile width).

Problems are sized so that CTAs run an odd number of tiles (the two ping-pong warpgroups get unequal counts) and the last
64-row tile is ragged.  Output buffers are wider than the launch's region and NaN-filled: what a launch does not own must keep
the NaN bit pattern."""
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
GEMM = 0
COOP, PINGPONG = 1, 2
SPARE = 200


def pingpong_variants():
    """(BN, KB) of every instantiation listed in PF_TMA_PINGPONG_VARIANTS (csrc/tma_host.cuh)."""
    src = open(os.path.join(_native.SRC_DIR, "tma_host.cuh")).read()
    body = src[src.index("#define PF_TMA_PINGPONG_VARIANTS(X)"):]
    body = body[:body.index("\n\n")]
    return sorted({(int(bn), int(kb)) for bn, kb in re.findall(r"X\((\d+), (\d+)\)", body)})


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


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def check_region(buf, c0, ref, tol=TOL):
    got = buf[:ref.shape[0], c0:c0 + ref.shape[1]]
    assert torch.isfinite(got).all(), "an owned element was not written"
    assert U.rel_err(got, ref) < tol, U.rel_err(got, ref)
    owned = torch.zeros_like(buf, dtype=torch.bool)
    owned[:ref.shape[0], c0:c0 + ref.shape[1]] = True
    assert untouched(buf)[~owned].all(), "a store landed outside the launch's region"


def odd_tile_rows(n, bn, sms):
    """Rows M such that cdiv(M, 64) x N tiles = about 2.5 x the SM count (CTAs run 2 or 3 ping-pong tiles, 1 or 2 cooperative
    ones) and the last 64-row tile holds 47 rows."""
    n_tiles = -(-n // bn)
    t = -(-5 * sms // (2 * n_tiles))
    return 64 * t - 17


def test_every_pingpong_instantiation_matches_the_cooperative_bits():
    """K = 320, N = 480 (a partial last N tile for most widths) through every (bn, kb) in both schedules: each within 5e-5 of
    float64, and the two schedules bit-identical for every instantiation; one common M: every width gives the same bits."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    K, N = 320, 480
    g = torch.Generator().manual_seed(5)
    whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
    bias = rn(g, N)
    variants = pingpong_variants()
    assert len(variants) == 10
    Mc = 1000 + 13
    ahi_c, alo_c, a_c = split(rn(g, Mc, K))
    ref_c = a_c @ w.t() + bias.double()
    common = {}
    for bn, kb in variants:
        M = odd_tile_rows(N, bn, sms)
        ahi, alo, a = split(rn(g, M, K))
        ref = a @ w.t() + bias.double()
        outs = {}
        for sched in (COOP, PINGPONG):
            C = nan32(M + SPARE, N + 8)
            op = tma(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1,
                     C=C, ldc=N + 8, c_coff=4, force_bn=bn, force_kb=kb, force_sched=sched)
            assert (op.picked_bn, op.picked_kb, op.picked_sched) == (bn, kb, sched)
            check_region(C, 4, ref)
            outs[sched] = C
            Cc = nan32(Mc + SPARE, N)
            tma(mode=GEMM, M=Mc, K=K, N=N, groups=1, a_hi=ahi_c, a_lo=alo_c, lda=K, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1,
                C=Cc, ldc=N, force_bn=bn, force_kb=kb, force_sched=sched)
            check_region(Cc, 0, ref_c)
            common[(bn, kb, sched)] = Cc
        assert torch.equal(bits(outs[COOP]), bits(outs[PINGPONG])), (bn, kb)
    first = next(iter(common))
    differ = [k for k, v in common.items() if not torch.equal(bits(v), bits(common[first]))]
    assert not differ, f"{differ} differ from {first}"


FEATURES = {
    "bias_relu_split_only": dict(act=1, split=True, c=False),
    "gelu_split_and_c": dict(act=2, split=True, c=True, split_relu=1),
    "gamma_inplace_residual": dict(gamma=True, res="inplace"),
    "relu_residual_split": dict(res="relu", split=True, c=True),
    "no_bias_c_only": dict(bias=False),
}


@pytest.mark.parametrize("feature", sorted(FEATURES))
def test_pingpong_epilogue_features(feature):
    """Each GEMM-mode epilogue feature the forward uses, in the ping-pong schedule at the widest and a narrow tile: + bias, ReLU /
    GELU, layer scale, in-place residual, relu(residual), split planes (rectified or not) with and without C.  Within 5e-5 of
    float64, S the exact split of relu?(C), and bit-identical to the cooperative schedule."""
    f = FEATURES[feature]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    K, N = 192, 256
    ldc, c_coff, lds, s_coff, ldr, r_coff = N + 24, 8, N + 16, 16, N + 40, 32
    for bn, kb in ((256, 32), (64, 64)):
        M = odd_tile_rows(N, bn, sms)
        g = torch.Generator().manual_seed(bn + len(feature))
        ahi, alo, a = split(rn(g, M, K))
        whi, wlo, w = split(rn(g, N, K, scale=K ** -0.5))
        ref = a @ w.t()
        args = dict(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K, w_hi=whi, w_lo=wlo, force_bn=bn, force_kb=kb)
        if f.get("bias", True):
            bias = rn(g, N)
            args.update(bias=bias, bias_mode=1)
            ref = ref + bias.double()
        if f.get("act") == 1:
            ref = F.relu(ref)
        elif f.get("act") == 2:
            ref = F.gelu(ref)
        args["act"] = f.get("act", 0)
        if f.get("gamma"):
            gamma = rn(g, N)
            args["gamma"] = gamma
            ref = ref * gamma.double()
        res = None
        if f.get("res") == "relu":
            res = rn(g, M, ldr)
            args.update(res=res, ldr=ldr, r_coff=r_coff, res_relu=1)
            ref = ref + F.relu(res[:, r_coff:r_coff + N]).double()
        elif f.get("res") == "inplace":
            res = rn(g, M, N)
            ref = ref + res.double()
        outs = {}
        for sched in (COOP, PINGPONG):
            run = dict(args, force_sched=sched)
            C = shi = slo = None
            if f.get("c", True):
                C = nan32(M + SPARE, ldc)
                run.update(C=C, ldc=ldc, c_coff=c_coff)
                if f.get("res") == "inplace":
                    C[:M, c_coff:c_coff + N] = res
                    run.update(res=C, ldr=ldc, r_coff=c_coff)
            if f.get("split"):
                shi, slo = nan16(M + SPARE, lds), nan16(M + SPARE, lds)
                run.update(s_hi=shi, s_lo=slo, lds=lds, s_coff=s_coff, split_relu=f.get("split_relu", 0))
            op = tma(**run)
            assert (op.picked_bn, op.picked_kb, op.picked_sched) == (bn, kb, sched)
            if C is not None:
                check_region(C, c_coff, ref)
            if shi is not None:
                v = C[:M, c_coff:c_coff + N] if C is not None else ref.float()
                hi, lo = weights.split_hi_lo(F.relu(v) if f.get("split_relu") else v)
                if C is not None:
                    assert torch.equal(bits(shi[:M, s_coff:s_coff + N]), bits(hi)) and torch.equal(bits(slo[:M, s_coff:s_coff + N]), bits(lo))
                else:
                    got = shi[:M, s_coff:s_coff + N].double() + slo[:M, s_coff:s_coff + N].double()
                    assert U.rel_err(got, ref) < TOL
                owned = torch.zeros_like(shi, dtype=torch.bool)
                owned[:M, s_coff:s_coff + N] = True
                assert untouched(shi)[~owned].all() and untouched(slo)[~owned].all()
            outs[sched] = [t for t in (C, shi, slo) if t is not None]
        for x, y in zip(outs[COOP], outs[PINGPONG]):
            assert torch.equal(bits(x), bits(y)), (feature, bn, kb)


def test_schedule_override_is_validated():
    """force_sched outside 0..2, or a schedule override on a halo-mode launch, is refused before anything is launched."""
    L = _native.lib()
    g = torch.Generator().manual_seed(3)
    ahi, alo, _ = split(rn(g, 8, 8, 8, 64))
    whi, wlo, _ = split(rn(g, 64, 9 * 64))
    C = nan32(1024, 64)
    for mode, sched in ((GEMM, 3), (GEMM, -1), (1, PINGPONG)):
        op = _native.pf_tma_op()
        geo = dict(mode=GEMM, M=64, K=64) if mode == GEMM else dict(mode=1, B=1, H=8, W=8, Cin=64)
        for k, v in dict(geo, N=64, groups=1, a_hi=ahi, a_lo=alo, lda=64, w_hi=whi, w_lo=wlo, C=C, ldc=64, force_sched=sched).items():
            setattr(op, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
        before = L.pf_kernel_launch_count()
        assert L.pf_op_tma(ctypes.byref(op), U.stream_ptr()) == -1
        assert "force_sched" in L.pf_last_error().decode()
        assert L.pf_kernel_launch_count() == before
    torch.cuda.synchronize()
    assert untouched(C).all()
