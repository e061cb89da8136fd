"""GPU: the forward graph's tensor-core launches, one at a time, at every shape, tile and epilogue form the graph runs them with,
against float64 -- the counterpart of test_gpu_forward_ops.py for the TMA -> wgmma engine (GEMM and halo mode), the gathered
stride-2 patch embeddings, the mma.sync attention core and conv_fuse_conv1's border ring.

``graph_tc_launches`` / ``paramnet_tc_launches`` restate every ``tgemm`` / ``thalo`` / ``tconv_gather`` /
``attention_mma_launch`` / ``conv1_ring_kernel`` call of ``run_forward`` and ``fwd_paramnet`` (``pf_b200.cu``) with its shape
and the exact epilogue form (``Fwd::Epi``) the graph gives it.  ``test_restatement_matches_the_graph`` pins the restatement to
the graph through the engine's per-launch profile at every sweep size; ``test_sweep_reaches_every_engine_configuration``
asserts that the sweep reaches every (launch, mode, tile, schedule) any legal working size at batches 1..64 reaches, and the
edges where the kernels go wrong (M < 64, ragged ping-pong tiles, halo grids below one tile or ragged in both directions, both
attention paths with a ragged last query pass).

Each distinct launch runs alone through the entry point that calls the graph's own helper (``pf_op_tma`` / ``pf_op_tma_bf16``,
``pf_op_conv_gemm``, ``pf_op_attention_tc_keys``, ``pf_op_conv1_ring``), in both precisions, against float64 on the operand
values the kernels multiply (hi + lo in split precision, hi in bf16).  Bars: 5e-5 for the engine in both modes (as in
test_gpu_engine.py / test_gpu_bf16.py) and for the split-precision attention core; the per-element one-ulp-of-P bound of
test_gpu_resize.py::test_attention_key_counts for the bf16 core; the bars of test_gpu_engine.py::test_phase_conv1_and_border_ring
for the ring and the fused prediction tails.

Every output sits in a NaN-filled buffer with spare rows and columns: the owned region must come back finite, everything else must
keep NaN's bit pattern.  Inputs carry NaN after the last image and in the columns past K (Cin) of a wider row pitch, so a tensor
map whose extent is too large poisons a checked output.  In-place residuals run in place.  Every case runs twice, bit-identical;
every GEMM-mode case runs again under the other schedule, bit-identical; the picked tile and schedule must be the dispatcher's."""
import collections
import csv
import ctypes
import os
import tempfile

import pytest
import torch
import torch.nn.functional as F

import oracle_resize as ro
import pf_test_util as U
from golden_util import golden_images
from perspectivefields_b200 import _native, weights
from test_gpu_engine import GEMM, HALO, TOL, check_split, conv3x3_ref, op_struct
from test_gpu_forward_ops import CNX_DIMS, GRAPH_SIZES as CORE_GRAPH_SIZES, MIT_DIMS, MIT_SR, PF_PARAM_CENTERED, PF_PARAM_UNCENTERED, bits, gen

pytestmark = pytest.mark.gpu

MIT_HEADS, MIT_DEPTHS, CNX_DEPTHS = (1, 2, 5, 8), (3, 4, 18, 3), (3, 3, 9, 3)
AM_KEYS_PAD, AM_QTILE = 112, 64         # attention_mma.cuh: single-block key limit, queries per pass
HT_TILE_H, HT_TILE_W = 16, 8            # tc_ptx.cuh: halo-mode output tile
PP_KMAX = 512                           # tma_host.cuh: kPingPongKMax
SPARE = 67                              # spare output rows behind every region (row pitches keep 16 spare columns: 16 B aligned)
PAD = 64                                # NaN columns past K / Cin in every input row
GEMM_KINDS = ("llenc", "embed1", "embed", "sr", "kv", "q", "proj", "fc1", "fc2", "pn_ds", "pw1", "pw2")
HALO_KINDS = ("proc", "rcu", "conv0", "conv1")


def L():
    return _native.lib()


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ the graph's launches
def graph_tc_launches(NH, NW, n, classification=False):
    """(kind, form, shape) of every tensor-core launch of run_forward at working size NH x NW and batch n, in the graph's order
    (one entry per launch: a block's launches repeat once per block).  GEMM mode: M x K -> N; ``embed`` is the gathered 3x3 / 2
    conv of tconv_gather on the previous stage's B x H x W x Cin map; halo mode: B x H x W x Cin -> N per group.  Regression heads
    fuse the prediction tails into conv_fuse_conv1 and the ring, classification heads write conv1's fp32 output."""
    RH, RW = [NH >> (s + 2) for s in range(4)], [NW >> (s + 2) for s in range(4)]
    nkv = RH[3] * RW[3]
    LH, LW = NH // 2, NW // 2
    out = [("llenc", "split+relu", dict(M=n * LH * LW, K=160, N=64))]
    for s in range(4):
        C, sr, heads, N = MIT_DIMS[s], MIT_SR[s], MIT_HEADS[s], RH[s] * RW[s]
        rows = n * N
        if s == 0:
            out.append(("embed1", "c", dict(M=rows, K=160, N=64)))
        else:
            out.append(("embed", "gather", dict(B=n, H=RH[s - 1], W=RW[s - 1], Cin=MIT_DIMS[s - 1], N=C)))
        block = []
        if sr > 1:
            block += [("sr", "c", dict(M=n * nkv, K=sr * sr * C, N=C)), ("kv", "split", dict(M=n * nkv, K=C, N=2 * C))]
        block.append(("q", "split", dict(M=rows, K=C, N=C)))
        if sr == 1:
            block.append(("kv", "split", dict(M=rows, K=C, N=2 * C)))
        block += [("attn", "", dict(B=n, N=N, nkv=nkv, C=C, heads=heads)), ("proj", "res_inplace", dict(M=rows, K=C, N=C)),
                  ("fc1", "c", dict(M=rows, K=C, N=4 * C)), ("fc2", "res_inplace", dict(M=rows, K=4 * C, N=C))]
        out += block * MIT_DEPTHS[s]
    for lvl in (4, 3, 2, 1):
        g = dict(B=n, H=RH[lvl - 1], W=RW[lvl - 1])
        out.append(("proc", "border+c+split_relu", dict(g, Cin=MIT_DIMS[lvl - 1], N=512, groups=1)))
        rcu = dict(g, Cin=256, N=256, groups=2)
        if lvl < 4:
            out += [("rcu", "relu_split", rcu), ("rcu", "c+split_relu+res_relu+res2", rcu)]
        out += [("rcu", "relu_split", rcu), ("rcu", "c+res_relu", rcu)]
    g = dict(B=n, H=LH, W=LW)
    out.append(("conv0", "dual_src", dict(g, Cin=320, N=64, groups=2)))
    out.append(("conv1", "phase4+c" if classification else "phase4+pred", dict(g, Cin=64, N=128, groups=2)))
    out.append(("ring", "c" if classification else "pred", g))
    return out


def paramnet_tc_launches(NH, NW, n, kind, size, training=False):
    """fwd_paramnet's GEMM launches on fields at NH x NW (ConvNeXt on NH x NW when centred, size x size otherwise): per stage
    the 2x2 / 2 downsample (stages 1-3, K = 4 C of the previous stage), then per block pw1 (GELU, split planes only) and pw2
    (layer scale + residual: in place in inference, out of place when training keeps every block's input)."""
    SH, SW = (NH, NW) if kind == PF_PARAM_CENTERED else (size, size)
    rh, rw = SH // 4, SW // 4
    out = []
    for s in range(4):
        C = CNX_DIMS[s]
        if s > 0:
            rh, rw = rh // 2, rw // 2
            out.append(("pn_ds", "c", dict(M=n * rh * rw, K=4 * CNX_DIMS[s - 1], N=C)))
        rows = n * rh * rw
        out += [("pw1", "gelu+split", dict(M=rows, K=C, N=4 * C)),
                ("pw2", "scale+res" if training else "scale+res_inplace", dict(M=rows, K=4 * C, N=C))] * CNX_DEPTHS[s]
    return out


def engine_mode(kind):
    return GEMM if kind in GEMM_KINDS else HALO if kind in HALO_KINDS else None


def gemm_mkn(kind, p):
    """(M, K, N) of a GEMM-mode launch (the gathered conv: OH = H / 2 rows of the im2col matrix per image row pair)"""
    if kind == "embed":
        return p["B"] * (p["H"] // 2) * (p["W"] // 2), 9 * p["Cin"], p["N"]
    return p["M"], p["K"], p["N"]


def profile_key(kind, p):
    """(engine_cfg, M, N, K, Cin, groups) of the engine's per-launch profile (Fwd::launch_tma), None for other kernels"""
    if engine_mode(kind) == GEMM:
        M, K, N = gemm_mkn(kind, p)
        return (5, M, N, K, K, 1)
    if engine_mode(kind) == HALO:
        return (6, p["B"] * p["H"] * p["W"], p["N"], 9 * p["Cin"], p["Cin"], p["groups"])
    return None


def pick(kind, p, sms):
    """(bn, kb, schedule) the dispatcher picks for a launch of the restatement"""
    if engine_mode(kind) == GEMM:
        M, K, N = gemm_mkn(kind, p)
        return pick_tile(GEMM, M, K, N, sms)
    return pick_tile(HALO, p["B"] * p["H"] * p["W"], 9 * p["Cin"], p["N"], sms)


def pick_tile(mode, M, K, N, sms):
    """pf_tma_pick_tile and the ping-pong rule (tma_pick_pingpong): (bn, kb, schedule), schedule 1 cooperative, 2 ping-pong,
    0 in halo mode"""
    bn, kb = ctypes.c_int(), ctypes.c_int()
    _native.check(L().pf_tma_pick_tile(mode, M, N, K, sms, ctypes.byref(bn), ctypes.byref(kb)))
    if mode == HALO:
        return bn.value, kb.value, 0
    return bn.value, kb.value, 2 if K <= PP_KMAX and cdiv(M, 64) * cdiv(N, bn.value) >= 2 * sms else 1


# Working sizes: test_gpu_forward_ops.py's (stage-4 grids 2 x 2 .. 16 x 16, a batch of 22 at 320 x 320), then 64 x 64 and
# 64 x 640 at batch 1 (M = 4 kv / sr GEMMs; a 2 x 20 level-4 grid).  ParamNet: centred at three of them, uncentred at the
# variants' INPUT_SIZE (64) at batches 1 and 64, and training's out-of-place pw2.
GRAPH_SIZES = CORE_GRAPH_SIZES + [(64, 64, 1), (64, 640, 1)]
PARAMNET_SIZES = [(320, 320, 22, PF_PARAM_CENTERED, 0, False), (96, 160, 3, PF_PARAM_CENTERED, 0, False), (64, 64, 1, PF_PARAM_CENTERED, 0, False),
                  (320, 320, 1, PF_PARAM_UNCENTERED, 64, False), (320, 320, 64, PF_PARAM_UNCENTERED, 64, False),
                  (320, 320, 4, PF_PARAM_UNCENTERED, 64, True)]
# Single launch kinds of other (NH, NW, n), where the sizes above leave an engine configuration or an edge of
# test_sweep_reaches_every_engine_configuration unreached on 132 SMs (H100 SXM): the cheapest launches that reach them.
GRAPH_EXTRA = [(64, 64, 22, 'fc1'), (64, 64, 33, 'embed1'), (64, 64, 33, 'fc1'), (64, 64, 33, 'proj'), (64, 64, 33, 'q'),
               (64, 96, 11, 'fc1'), (64, 160, 35, 'fc1'), (64, 160, 53, 'fc2'), (64, 224, 19, 'embed'), (64, 224, 19, 'fc1'),
               (64, 288, 58, 'proj'), (64, 288, 58, 'q'), (64, 352, 19, 'fc1'), (64, 480, 47, 'proj'), (64, 480, 47, 'q'),
               (64, 544, 17, 'fc1'), (96, 96, 29, 'fc2'), (96, 352, 1, 'llenc'), (96, 448, 55, 'kv'), (96, 544, 54, 'kv'),
               (96, 640, 47, 'kv'), (128, 512, 1, 'attn'), (160, 160, 59, 'kv'), (160, 480, 41, 'kv'), (160, 544, 49, 'kv'),
               (160, 576, 37, 'sr'), (192, 608, 1, 'attn'), (192, 640, 47, 'embed'), (192, 640, 47, 'fc2'), (192, 640, 47, 'proj'),
               (192, 640, 47, 'q'), (256, 544, 41, 'proj'), (256, 544, 41, 'q'), (416, 416, 25, 'embed'), (416, 416, 25, 'fc2'),
               (416, 416, 25, 'proj'), (416, 416, 25, 'q'), (416, 416, 50, 'sr'), (416, 480, 43, 'kv'), (416, 480, 43, 'proj'),
               (416, 480, 43, 'q')]
PARAMNET_EXTRA = [(64, 64, 6, 'pw1'), (64, 64, 11, 'pw1'), (64, 64, 22, 'pw1'), (64, 64, 22, 'pw2'), (64, 64, 33, 'pw2'),
                  (64, 64, 45, 'pw1'), (64, 96, 11, 'pw1'), (64, 96, 29, 'pn_ds'), (64, 96, 59, 'pn_ds'), (64, 160, 35, 'pn_ds'),
                  (64, 352, 1, 'pw1'), (96, 160, 35, 'pn_ds'), (96, 640, 47, 'pn_ds'), (96, 640, 47, 'pw2'), (160, 544, 1, 'pw1'),
                  (416, 416, 25, 'pn_ds'), (416, 416, 25, 'pw2')]


def case_id(kind, form, p):
    return "-".join([kind] + ([form] if form else []) + [f"{k}{v}" for k, v in p.items()])


def sweep():
    cases = {}
    for NH, NW, n in GRAPH_SIZES:
        for classification in (False, True):
            for c in graph_tc_launches(NH, NW, n, classification):
                cases.setdefault(case_id(*c), c)
    for NH, NW, n, kind, size, training in PARAMNET_SIZES:
        for c in paramnet_tc_launches(NH, NW, n, kind, size, training):
            cases.setdefault(case_id(*c), c)
    for extra, launches in ((GRAPH_EXTRA, graph_tc_launches), (PARAMNET_EXTRA, lambda NH, NW, n: paramnet_tc_launches(NH, NW, n, PF_PARAM_CENTERED, 0))):
        for NH, NW, n, kind in extra:
            for c in launches(NH, NW, n):
                if c[0] == kind:
                    cases.setdefault(case_id(*c), c)
    return cases


SWEEP = sweep()


# ------------------------------------------------------------------------------------------------ coverage of the sweep
def legal_sizes():
    return [(h, w) for h in range(64, 641, 32) for w in range(64, 641, 32) if (h // 32) * (w // 32) <= 256]


def features(launches, sms, memo):
    """the properties the sweep must reach, of a list of launches: engine configurations, and edge tuples"""
    out = set()
    for kind, form, p in launches:
        key = (kind, form, tuple(p.values()))
        if key in memo:
            out |= memo[key]
            continue
        f = set()
        mode = engine_mode(kind)
        if mode is not None:
            bn, kb, sched = pick(kind, p, sms)
            f.add(("cfg", kind, mode, bn, kb, sched))
        if mode == GEMM:
            M = gemm_mkn(kind, p)[0]
            if M < 64:
                f.add(("gemm M < 64", form))
            if sched == 2 and M % 64:
                f.add(("ragged ping-pong tile", kind))
        elif mode == HALO:
            H, W = p["H"], p["W"]
            if H < HT_TILE_H and W < HT_TILE_W:
                f.add(("halo below one tile", kind))
            if H > HT_TILE_H and W > HT_TILE_W and H % HT_TILE_H and W % HT_TILE_W:
                f.add(("halo ragged both ways", kind))
        elif kind == "attn":
            f.add(("attention", p["C"], p["heads"], p["nkv"] > AM_KEYS_PAD, p["N"] % AM_QTILE != 0))
        memo[key] = f
        out |= f
    return out


def reachable(sms):
    """features of every legal working size at batches 1..64: the graph (the head kinds share their shapes), ParamNet centred at the working
    size and uncentred at the variants' INPUT_SIZE (64)"""
    memo, out = {}, set()
    for NH, NW in legal_sizes():
        for n in range(1, 65):
            out |= features(graph_tc_launches(NH, NW, n), sms, memo)
            out |= features(paramnet_tc_launches(NH, NW, n, PF_PARAM_CENTERED, 0), sms, memo)
    for n in range(1, 65):
        for training in (False, True):
            out |= features(paramnet_tc_launches(64, 64, n, PF_PARAM_UNCENTERED, 64, training), sms, memo)
    return out


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_sweep_reaches_every_engine_configuration():
    sms = sm_count()
    got = features(list(SWEEP.values()), sms, {})
    want = reachable(sms)
    assert want <= got, sorted(want - got)
    # the edges named in the docstring are reachable (so the inclusion above asserts them)
    gemm_forms = {f for k, f, _ in SWEEP.values() if engine_mode(k) == GEMM}
    assert {("gemm M < 64", f) for f in gemm_forms - {"split+relu"}} <= got      # (ll_enc: M = n NH NW / 4 >= 1024)
    assert any(f[0] == "ragged ping-pong tile" for f in got)
    assert {("halo below one tile", k) for k in ("proc", "rcu")} <= got
    assert {("halo ragged both ways", k) for k in ("proc", "rcu")} <= got     # (conv0 / conv1 run on NH / 2 rows: whole tiles)
    for C, heads in zip(MIT_DIMS, MIT_HEADS):
        assert ("attention", C, heads, False, False) in got or ("attention", C, heads, False, True) in got
        assert ("attention", C, heads, True, False) in got or ("attention", C, heads, True, True) in got


# ------------------------------------------------------------------------------------------------ the restatement is the graph
def profiled_launches(m, imgs):
    """the (engine_cfg, M, N, K, Cin, groups) multiset of one inference_batch, from the engine's per-launch profile"""
    eng = m._get_engine()
    buf = (ctypes.c_double * 21)()
    path = os.path.join(tempfile.mkdtemp(), "launches.csv")
    eng.L.pf_profile_enable(eng.handle, 1)
    try:
        torch.cuda.synchronize()
        _native.check(eng.L.pf_profile_read(eng.handle, buf))
        m.inference_batch(imgs)
        torch.cuda.synchronize()
        os.environ["PF_PROFILE_CSV"] = path
        try:
            _native.check(eng.L.pf_profile_read(eng.handle, buf))
        finally:
            del os.environ["PF_PROFILE_CSV"]
    finally:
        eng.L.pf_profile_enable(eng.handle, 0)
    with open(path) as f:
        rows = list(csv.DictReader(f))
    os.remove(path)
    return collections.Counter(tuple(int(r[k]) for k in ("engine_cfg", "M", "N", "K", "Cin", "groups")) for r in rows)


def restated(launches):
    return collections.Counter(k for k in (profile_key(kind, p) for kind, _, p in launches) if k is not None)


@pytest.mark.parametrize("NH,NW,n", GRAPH_SIZES)
def test_restatement_matches_the_graph(NH, NW, n):
    """The engine launches of one batch through the product API equal the restatement's, launch for launch: the regression
    variant with the centred ParamNet at the working size, and the classification variant (no ParamNet)."""
    from oracle import weights_gen as wg

    imgs = wg.smooth_images(n, 48, 64, NH + NW)
    for version, pn in (("Paramnet-360Cities-edina-centered", True), ("PersNet-360Cities", False)):
        m, _ = U.make_model(version, model_kwargs={"resize": (NH, NW)})
        want = graph_tc_launches(NH, NW, n, not pn) + (paramnet_tc_launches(NH, NW, n, PF_PARAM_CENTERED, 0) if pn else [])
        got = profiled_launches(m, imgs)
        assert got == restated(want), (version, sorted((got - restated(want)).items()), sorted((restated(want) - got).items()))
        del m
    torch.cuda.empty_cache()


def test_uncentred_paramnet_matches_the_graph():
    from oracle import weights_gen as wg

    NH, NW, n = 96, 160, 3
    m, _ = U.make_model("Paramnet-360Cities-edina-uncentered", model_kwargs={"resize": (NH, NW)})
    want = graph_tc_launches(NH, NW, n) + paramnet_tc_launches(NH, NW, n, PF_PARAM_UNCENTERED, 64)
    assert profiled_launches(m, wg.smooth_images(n, 48, 64, 5)) == restated(want)


# ------------------------------------------------------------------------------------------------ buffers and checks
def rnd(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def untouched(t):
    return bits(t) == bits(torch.full((1,), float("nan"), dtype=t.dtype, device=t.device))


def operand(x, prec):
    """(hi, lo) planes of x and the value the engine multiplies: hi + lo (split precision) or hi (bf16)"""
    hi, lo = weights.split_hi_lo(x)
    return hi, lo, (hi.double() + lo.double()) if prec == "split" else hi.double()


def padded_planes(x, prec, ld):
    """split planes of x [..., c] in rows of pitch ld (NaN in the columns past c) with one NaN image / row block behind them"""
    hi, lo, v = operand(x, prec)
    lead = x.shape[:-1]
    extra = (1,) + lead[1:] if len(lead) > 1 else (SPARE,)
    ph, pl = nan(*((lead[0] + extra[0],) + lead[1:] + (ld,)), dtype=torch.bfloat16), nan(*((lead[0] + extra[0],) + lead[1:] + (ld,)), dtype=torch.bfloat16)
    ph[:lead[0], ..., :x.shape[-1]] = hi
    pl[:lead[0], ..., :x.shape[-1]] = lo
    return ph, pl, v


def owned_region(buf, rows, regions):
    """check that nothing outside [0, rows) x the (c0, n) column regions of buf [R, ld] was written"""
    owned = torch.zeros_like(buf, dtype=torch.bool)
    for c0, n in regions:
        owned[:rows, c0:c0 + n] = True
    assert untouched(buf)[~owned].all(), "a store landed outside the launch's region"


def check_c(C, regions, tol=TOL):
    """C [R, ld]: regions (c0, reference [rows, n]) within tol, finite; NaN elsewhere"""
    for c0, ref in regions:
        got = C[:ref.shape[0], c0:c0 + ref.shape[1]]
        assert torch.isfinite(got).all(), "an owned element was not written"
        assert U.rel_err(got, ref) < tol, (c0, U.rel_err(got, ref))
    owned_region(C, regions[0][1].shape[0], [(c0, r.shape[1]) for c0, r in regions])


def check_s(shi, slo, regions, tol=TOL):
    """split planes of a launch that writes no fp32 C: hi + lo within tol of the references (the split itself is exact to
    2^-17 relative), NaN elsewhere"""
    for c0, ref in regions:
        h, l = shi[:ref.shape[0], c0:c0 + ref.shape[1]], slo[:ref.shape[0], c0:c0 + ref.shape[1]]
        y = h.double() + l.double()
        assert torch.isfinite(y).all(), "an owned element was not written"
        assert U.rel_err(y, ref) < tol, (c0, U.rel_err(y, ref))
    for t in (shi, slo):
        owned_region(t, regions[0][1].shape[0], [(c0, r.shape[1]) for c0, r in regions])


def same_bits(a, b, what):
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(bits(x), bits(y)), what


def run_tma(prec, outs, **kw):
    """one pf_op_tma(_bf16) launch on fresh copies of the NaN-filled output buffers outs (name -> tensor); in-place residuals
    (res is C) follow the copy.  Returns (op, {name: written copy})."""
    fresh = {k: v.clone() for k, v in outs.items()}
    args = dict(kw)
    for k, v in list(args.items()):
        for name, t in outs.items():
            if v is t:
                args[k] = fresh[name]
    args.update({k: v for k, v in fresh.items() if k not in args})
    op = op_struct(**args)
    fn = L().pf_op_tma_bf16 if prec == "bf16" else L().pf_op_tma
    _native.check(fn(ctypes.byref(op), U.stream_ptr()))
    torch.cuda.synchronize()
    return op, fresh


def engine_case(kind, prec, outs, **kw):
    """the launch twice (bit-identical), its picked tile and schedule against the dispatcher's, and in GEMM mode once more under the
    other schedule (bit-identical).  Returns the written outputs."""
    op, a = run_tma(prec, outs, **kw)
    _, b = run_tma(prec, outs, **kw)
    same_bits([a[k] for k in outs], [b[k] for k in outs], "two identical launches differ")
    M, K = (kw["B"] * kw["H"] * kw["W"], 9 * kw["Cin"]) if kw["mode"] == HALO else (kw["M"], kw["K"])
    want = pick_tile(kw["mode"], M, K, kw["N"], sm_count())
    assert (op.picked_bn, op.picked_kb, op.picked_sched) == want, (kind, (op.picked_bn, op.picked_kb, op.picked_sched), want)
    if kw["mode"] == GEMM:
        other = 3 - op.picked_sched
        op2, c = run_tma(prec, outs, force_sched=other, **kw)
        assert op2.picked_sched == other and (op2.picked_bn, op2.picked_kb) == (op.picked_bn, op.picked_kb)
        same_bits([a[k] for k in outs], [c[k] for k in outs], "the other schedule computes different bits")
    return a


# ------------------------------------------------------------------------------------------------ GEMM mode
def gemm_case(kind, form, M, K, N, prec):
    g = gen((kind, form, M, K, N, prec))
    ahi, alo, a = padded_planes(rnd(g, M, K), prec, K + PAD)
    whi, wlo, w = operand(rnd(g, N, K, scale=K ** -0.5), prec)
    bias = rnd(g, N, scale=0.5)
    acc = a @ w.t() + bias.double()
    kw = dict(mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K + PAD, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1)
    ldc, lds, c0, s0 = N + 16, N + 24, 4, 8
    if form in ("split+relu", "split", "gelu+split"):
        act = {"split+relu": 1, "split": 0, "gelu+split": 2}[form]
        ref = F.relu(acc) if act == 1 else F.gelu(acc) if act == 2 else acc
        o = engine_case(kind, prec, dict(s_hi=nan(M + SPARE, lds, dtype=torch.bfloat16), s_lo=nan(M + SPARE, lds, dtype=torch.bfloat16)),
                        lds=lds, s_coff=s0, act=act, **kw)
        check_s(o["s_hi"], o["s_lo"], [(s0, ref)])
    elif form == "c":
        o = engine_case(kind, prec, dict(C=nan(M + SPARE, ldc)), ldc=ldc, c_coff=c0, **kw)
        check_c(o["C"], [(c0, acc)])
    elif form in ("res_inplace", "scale+res_inplace", "scale+res"):
        res = rnd(g, M, N)
        gamma = (torch.rand(N, generator=g, device="cuda") * 0.4 + 0.1) if form.startswith("scale") else None
        ref = (acc * gamma.double() if gamma is not None else acc) + res.double()
        C = nan(M + SPARE, ldc)
        extra = dict(gamma=gamma) if gamma is not None else {}
        if form.endswith("inplace"):
            C[:M, c0:c0 + N] = res
            o = engine_case(kind, prec, dict(C=C), ldc=ldc, c_coff=c0, res=C, ldr=ldc, r_coff=c0, **extra, **kw)
        else:
            R = nan(M + SPARE, N + 24)
            R[:M, 16:16 + N] = res
            o = engine_case(kind, prec, dict(C=C), ldc=ldc, c_coff=c0, res=R, ldr=N + 24, r_coff=16, **extra, **kw)
            assert torch.equal(R[:M, 16:16 + N], res), "the out-of-place residual was written"
        check_c(o["C"], [(c0, ref)])
    else:
        raise AssertionError(form)


def gather_case(p, prec):
    """embed2..4: the 3x3 / 2 / pad 1 conv of the previous stage's map.  Split precision: pf_op_conv_gemm, which splits x and runs
    the graph's tconv_gather (im2col_split_kernel + tgemm).  bf16: the same GEMM through pf_op_tma_bf16 on the im2col matrix (the
    gather is precision independent: it copies planes)."""
    B, H, W, Cin, N = p["B"], p["H"], p["W"], p["Cin"], p["N"]
    OH, OW = H // 2, W // 2
    M, K = B * OH * OW, 9 * Cin
    g = gen(("gather", B, H, W, Cin, N, prec))
    x = rnd(g, B, H, W, Cin)
    whi, wlo, w = operand(rnd(g, N, K, scale=K ** -0.5), prec)
    bias = rnd(g, N, scale=0.5)
    if prec == "bf16":
        cols = F.unfold(x.permute(0, 3, 1, 2), 3, padding=1, stride=2)              # (c, ky, kx) -> the engine's (ky, kx, c)
        a = cols.view(B, Cin, 9, OH * OW).permute(0, 3, 2, 1).reshape(M, K)
        return gemm_case_on(a, whi, wlo, w, bias, prec)
    xs = torch.full((B * H * W * Cin + 4 * Cin,), float("nan"), device="cuda")
    xs[:B * H * W * Cin] = x.reshape(-1)
    xv = xs[:B * H * W * Cin].view(B, H, W, Cin)
    hi, lo = weights.split_hi_lo(x)
    ref = F.conv2d((hi.double() + lo.double()).permute(0, 3, 1, 2), w.view(N, 3, 3, Cin).permute(0, 3, 1, 2), bias.double(), stride=2, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(M, N)

    def run():
        y = nan(M + SPARE, N)
        _native.check(L().pf_op_conv_gemm(xv.data_ptr(), B, H, W, Cin, whi.data_ptr(), wlo.data_ptr(), bias.data_ptr(), N, 3, 3, 2, 1, 0, 0,
                                          None, 0, y.data_ptr(), U.stream_ptr()))
        torch.cuda.synchronize()
        return y
    y = run()
    assert torch.equal(bits(y), bits(run())), "two identical launches differ"
    check_c(y, [(0, ref)])


def gemm_case_on(a32, whi, wlo, w, bias, prec):
    M, K = a32.shape
    N = w.shape[0]
    ahi, alo, a = padded_planes(a32, prec, K + PAD)
    ldc = N + 16
    o = engine_case("embed", prec, dict(C=nan(M + SPARE, ldc)), mode=GEMM, M=M, K=K, N=N, groups=1, a_hi=ahi, a_lo=alo, lda=K + PAD,
                    w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1, ldc=ldc, c_coff=4)
    check_c(o["C"], [(4, a @ w.t() + bias.double())])


# ------------------------------------------------------------------------------------------------ halo mode
def border_classes(B, H, W):
    ry = torch.ones(H, dtype=torch.long)
    ry[0], ry[-1] = 0, 2
    rx = torch.ones(W, dtype=torch.long)
    rx[0], rx[-1] = 0, 2
    return (ry[:, None] * 3 + rx[None, :]).reshape(-1).repeat(B).cuda()


def halo_case(kind, form, p, prec):
    B, H, W, Cin, N, groups = (p[k] for k in ("B", "H", "W", "Cin", "N", "groups"))
    M = B * H * W
    g = gen((kind, form, B, H, W, prec))
    geo = dict(mode=HALO, B=B, H=H, W=W, Cin=Cin, N=N, groups=groups)
    if kind == "proc":
        ahi, alo, a = padded_planes(rnd(g, B, H, W, Cin), prec, Cin + PAD)
        whi, wlo, w = operand(rnd(g, N, 9 * Cin, scale=(9 * Cin) ** -0.5), prec)
        bias9 = rnd(g, 9 * N, scale=0.5)
        ref = conv3x3_ref(a, w, Cin) + bias9.view(9, N).double()[border_classes(B, H, W)]
        ldc, lds = N + 16, N + 24
        o = engine_case(kind, prec, dict(C=nan(M + SPARE, ldc), s_hi=nan(M + SPARE, lds, dtype=torch.bfloat16), s_lo=nan(M + SPARE, lds, dtype=torch.bfloat16)),
                        a_hi=ahi, a_lo=alo, lda=Cin + PAD, w_hi=whi, w_lo=wlo, bias=bias9, bias_mode=2, ldc=ldc, c_coff=4, lds=lds, s_coff=8, split_relu=1, **geo)
        check_c(o["C"], [(4, ref)])
        check_split(o["s_hi"], o["s_lo"], [(8, o["C"][:M, 4:4 + N])], True)
        return
    if kind == "rcu":
        # both heads in one launch: group g reads channels 256 g .. of 512-wide rows, writes its block of 256 columns
        ahi, alo, a = padded_planes(rnd(g, B, H, W, 512), prec, 512 + PAD)
        whi, wlo, w = operand(rnd(g, 2 * N, 9 * Cin, scale=(9 * Cin) ** -0.5), prec)
        bias = rnd(g, 2 * N, scale=0.5)
        accs = [conv3x3_ref(a[..., 256 * gi:256 * gi + 256], w[N * gi:N * gi + N], Cin) + bias[N * gi:N * gi + N].double() for gi in range(2)]
        kw = dict(geo, a_hi=ahi, a_lo=alo, lda=512 + PAD, a_gc=256, w_hi=whi, w_lo=wlo, bias=bias, bias_mode=1, bias_gstride=256)
        ldc, lds = 512 + 16, 512 + 24
        S = dict(s_hi=nan(M + SPARE, lds, dtype=torch.bfloat16), s_lo=nan(M + SPARE, lds, dtype=torch.bfloat16))
        if form == "relu_split":
            o = engine_case(kind, prec, S, lds=lds, s_coff=8, s_gcoff=256, act=1, **kw)
            check_s(o["s_hi"], o["s_lo"], [(8 + 256 * gi, F.relu(accs[gi])) for gi in range(2)])
            return
        res = rnd(g, M, 512 + 32)
        kw.update(res=res, ldr=512 + 32, r_coff=16, r_gcoff=256, res_relu=1, ldc=ldc, c_coff=4, c_gcoff=256)
        refs = [accs[gi] + F.relu(res[:, 16 + 256 * gi:16 + 256 * gi + N]).double() for gi in range(2)]
        outs = dict(C=nan(M + SPARE, ldc))
        if form == "c+split_relu+res_relu+res2":
            res2 = rnd(g, M, 512)
            kw.update(res2=res2, ldr2=512, r2_gcoff=256, lds=lds, s_coff=8, s_gcoff=256, split_relu=1)
            refs = [refs[gi] + res2[:, 256 * gi:256 * gi + N].double() for gi in range(2)]
            outs.update(S)
        else:
            assert form == "c+res_relu", form
        o = engine_case(kind, prec, outs, **kw)
        check_c(o["C"], [(4 + 256 * gi, refs[gi]) for gi in range(2)])
        if "s_hi" in o:
            check_split(o["s_hi"], o["s_lo"], [(8 + 256 * gi, o["C"][:M, 4 + 256 * gi:4 + 256 * gi + N]) for gi in range(2)], True)
        return
    if kind == "conv0":
        # per head: input channels 0-255 from the fused feature (group block of 256 in 512-wide rows), 256-319 from ll (A2)
        ahi, alo, a = padded_planes(rnd(g, B, H, W, 512), prec, 512 + PAD)
        a2hi, a2lo, a2 = padded_planes(rnd(g, B, H, W, 64), prec, 64 + PAD)
        whi, wlo, w = operand(rnd(g, 2 * N, 9 * Cin, scale=(9 * Cin) ** -0.5), prec)
        bias = rnd(g, 2 * N, scale=0.5)
        lds = 2 * N + 24
        o = engine_case(kind, prec, dict(s_hi=nan(M + SPARE, lds, dtype=torch.bfloat16), s_lo=nan(M + SPARE, lds, dtype=torch.bfloat16)),
                        a_hi=ahi, a_lo=alo, lda=512 + PAD, a_gc=256, a2_hi=a2hi, a2_lo=a2lo, lda2=64 + PAD, c_split=256, w_hi=whi, w_lo=wlo,
                        bias=bias, bias_mode=1, bias_gstride=N, act=1, lds=lds, s_coff=8, s_gcoff=N, **geo)
        refs = [(8 + N * gi, F.relu(conv3x3_ref(torch.cat([a[..., 256 * gi:256 * gi + 256], a2], -1), w[N * gi:N * gi + N], Cin)
                                    + bias[N * gi:N * gi + N].double())) for gi in range(2)]
        check_s(o["s_hi"], o["s_lo"], refs)
        return
    assert kind == "conv1", kind
    phase_case(form, B, H, W, prec, g)


def phase_case(form, B, H, W, prec, g):
    """conv_fuse_conv1 composed with the x2 upsample: N = 4 phases x 32 per head on the H x W grid, chunk ph of pixel (y, x) is
    pixel (2y + ph / 2, 2x + ph % 2) of the 2H x 2W output.  Restated as a 3x3 conv with the composed weights; the prediction
    tails in float64 on the launch's own conv1 values (bounds of test_gpu_engine.py::test_phase_conv1_and_border_ring)."""
    H2, W2, P2 = 2 * H, 2 * W, 4 * B * H * W
    chi, clo, c = padded_planes(F.relu(rnd(g, B, H, W, 128)), prec, 128 + PAD)
    whi, wlo, w = operand(rnd(g, 256, 9 * 64, scale=(9 * 64) ** -0.5), prec)
    bias = rnd(g, 256, scale=0.5)
    ys = []
    for gi in range(2):
        y = F.relu(conv3x3_ref(c[..., 64 * gi:64 * gi + 64], w[128 * gi:128 * gi + 128], 64) + bias[128 * gi:128 * gi + 128].double())
        ys.append(y.view(B, H, W, 2, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(B, H2, W2, 32))
    kw = dict(mode=HALO, B=B, H=H, W=W, Cin=64, N=128, groups=2, a_hi=chi, a_lo=clo, lda=128 + PAD, a_gc=64, w_hi=whi, w_lo=wlo, bias=bias,
              bias_mode=1, bias_gstride=128, act=1, phase4=1)
    if form == "phase4+c":
        o = engine_case("conv1", prec, dict(C=nan(P2 + SPARE, 64 + 8)), ldc=64 + 8, c_gcoff=32, **kw)
        check_c(o["C"], [(0, torch.cat(ys, -1).reshape(P2, 64))])
        return
    pgw, pgb, plw, plb = rnd(g, 2 * 32, scale=0.3), rnd(g, 2), rnd(g, 32, scale=0.3), rnd(g, 1)
    n2 = B * H2 * W2

    def run(with_c):
        """the graph's form (the tails alone), or the same launch also writing conv1's output C"""
        pg, pl = nan(2 * n2 + SPARE), nan(n2 + SPARE)
        C = nan(P2 + SPARE, 64 + 8) if with_c else None
        op = op_struct(pred=[(pgw, pgb, pg, 2, 1), (plw, plb, pl, 1, 2)], **(dict(kw, C=C, ldc=64 + 8, c_gcoff=32) if with_c else kw))
        _native.check((L().pf_op_tma_bf16 if prec == "bf16" else L().pf_op_tma)(ctypes.byref(op), U.stream_ptr()))
        torch.cuda.synchronize()
        return op, pg, pl, C
    op, pg, pl, _ = run(False)
    _, pg2, pl2, _ = run(False)
    same_bits((pg, pl), (pg2, pl2), "two identical launches differ")
    assert (op.picked_bn, op.picked_kb, op.picked_sched) == pick("conv1", dict(B=B, H=H, W=W, Cin=64, N=128), sm_count())
    assert untouched(pg[2 * n2:]).all() and untouched(pl[n2:]).all(), "a store landed behind the prediction outputs"
    # conv1's values: within the engine's bar of float64, and the tails' own arithmetic on them (the 1e-5 bars of the tails
    # bound the 1x1 conv + normalise / clamp, not the 32-term amplification of conv1's error by the tail weights)
    _, pgc, plc, C = run(True)
    same_bits((pg, pl), (pgc, plc), "the tails depend on whether C is written")
    check_c(C, [(0, torch.cat(ys, -1).reshape(P2, 64))])
    y = C[:P2, :64].double().view(B, H2, W2, 64)
    check_tails(pg[:2 * n2].view(B, 2, H2, W2), pl[:n2].view(B, 1, H2, W2), [y[..., :32], y[..., 32:]], (pgw, pgb, plw, plb),
                torch.ones(H2, W2, dtype=torch.bool))


def check_tails(pg, pl, ys, tails, mask):
    """the fused prediction tails on the pixels of mask [H2, W2]: F.normalize of the gravity 1x1 conv weighed by |v| / max |v| on
    the pixels whose |v| is not small, and the clamped latitude conv, in float64 on the conv1 output ys (per head, [B, H2, W2, 32])"""
    pgw, pgb, plw, plb = tails
    y0, y1 = ys[0].permute(0, 3, 1, 2), ys[1].permute(0, 3, 1, 2)
    v = F.conv2d(y0, pgw.double().view(2, 32, 1, 1), pgb.double())[..., mask]
    lat = F.conv2d(y1, plw.double().view(1, 32, 1, 1), plb.double()).clamp(-1, 1)[..., mask]
    pg, pl = pg[..., mask], pl[..., mask]
    assert torch.isfinite(pg).all() and torch.isfinite(pl).all(), "a pixel of the tails was not written"
    nrm = v.norm(dim=1, keepdim=True)
    ok = (nrm > 0.05 * nrm.max()).expand_as(pg)
    assert ok.float().mean() > 0.5
    assert ((pg.double() - F.normalize(v, dim=1)) * nrm / nrm.max())[ok].abs().max() < 1e-5
    assert U.rel_err(pl, lat) < 1e-5


# ------------------------------------------------------------------------------------------------ conv1's border ring
def ring_case(form, p):
    """conv1_ring_kernel alone on conv_fuse_conv0's split output: relu(conv3x3(bilinear_x2(c0))) per head on the two outermost rows
    and columns of the 2H x 2W output (fp32 CUDA-core arithmetic on hi + lo, in both precision modes); nothing else written"""
    B, H, W = p["B"], p["H"], p["W"]
    H2, W2, P2 = 2 * H, 2 * W, 4 * B * H * W
    g = gen(("ring", form, B, H, W))
    c = F.relu(rnd(g, B, H, W, 128))
    hi, lo = weights.split_hi_lo(c)
    chi, clo = nan(B * H * W * 128 + 1024, dtype=torch.bfloat16), nan(B * H * W * 128 + 1024, dtype=torch.bfloat16)
    chi[:hi.numel()], clo[:lo.numel()] = hi.reshape(-1), lo.reshape(-1)
    cv = hi.double() + lo.double()
    wf = rnd(g, 2, 9, 64, 32, scale=(9 * 64) ** -0.5)          # [head][tap = 3 ky + kx][ci][o]
    bias = rnd(g, 64, scale=0.5)
    u = F.interpolate(cv.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
    ys = [F.relu(F.conv2d(u[:, 64 * gi:64 * gi + 64], wf[gi].double().view(3, 3, 64, 32).permute(3, 2, 0, 1), bias[32 * gi:32 * gi + 32].double(),
                          padding=1)).permute(0, 2, 3, 1) for gi in range(2)]
    ring = torch.ones(H2, W2, dtype=torch.bool, device="cuda")
    ring[2:-2, 2:-2] = False
    tails = (rnd(g, 2 * 32, scale=0.3), rnd(g, 2), rnd(g, 32, scale=0.3), rnd(g, 1))

    def run():
        out = nan(P2 + SPARE, 64) if form == "c" else None
        pg, pl = (nan(B * 2 * H2 * W2 + SPARE), nan(B * H2 * W2 + SPARE)) if form == "pred" else (None, None)
        t = [tails[0], tails[1], pg, tails[2], tails[3], pl] if form == "pred" else [None] * 6
        _native.check(L().pf_op_conv1_ring(chi.data_ptr(), clo.data_ptr(), B, H, W, wf.data_ptr(), bias.data_ptr(), None if out is None else out.data_ptr(),
                                           *[None if x is None else x.data_ptr() for x in t], U.stream_ptr()))
        torch.cuda.synchronize()
        return out, pg, pl
    a = run()
    same_bits(a, run(), "two identical launches differ")
    out, pg, pl = a
    n2 = B * H2 * W2
    if form == "c":
        got = out[:P2].view(B, H2, W2, 64)
        ref = torch.cat(ys, -1)
        assert torch.isfinite(got[:, ring]).all()
        assert U.rel_err(got[:, ring], ref[:, ring]) < TOL, U.rel_err(got[:, ring], ref[:, ring])
        assert untouched(got[:, ~ring]).all() and untouched(out[P2:]).all(), "the ring kernel wrote outside the ring"
        return
    pgv, plv = pg[:2 * n2].view(B, 2, H2, W2), pl[:n2].view(B, 1, H2, W2)
    assert untouched(pgv[..., ~ring]).all() and untouched(plv[..., ~ring]).all() and untouched(pg[2 * n2:]).all() and untouched(pl[n2:]).all()
    check_tails(pgv, plv, ys, tails, ring)


# ------------------------------------------------------------------------------------------------ attention core
def attention_case(p, prec):
    """pf_op_attention_tc_keys at the graph's (B, N queries, keys, C, heads).  Split precision: 5e-5 against a float64 softmax on
    hi + lo of q and kv; bf16: the per-element bound of test_gpu_resize.py::test_attention_key_counts on the hi planes."""
    B, N, nkv, C, heads = p["B"], p["N"], p["nkv"], p["C"], p["heads"]
    g = gen(("attn", B, N, nkv, C, prec))
    q, kv = rnd(g, B, N, C, scale=2.0), rnd(g, B, nkv, 2 * C)
    qg, kvg = nan(B * N * C + 4096), nan(B * nkv * 2 * C + 4096)          # NaN after the last image
    qg[:q.numel()], kvg[:kv.numel()] = q.reshape(-1), kv.reshape(-1)

    def run():
        out = nan(B * N * C + SPARE)
        _native.check(L().pf_op_attention_tc_keys(qg.data_ptr(), kvg.data_ptr(), out.data_ptr(), B, N, nkv, C, heads, int(prec == "bf16"), U.stream_ptr()))
        torch.cuda.synchronize()
        return (out,)
    out, = run()
    same_bits((out,), run(), "two identical launches differ")
    assert untouched(out[B * N * C:]).all(), "a store landed behind the output"
    out = out[:B * N * C].view(B, N, C)
    assert torch.isfinite(out).all(), "an owned element was not written"
    _, _, qv = operand(q, prec)
    _, _, kvv = operand(kv, prec)
    for h in range(heads):
        sl = slice(64 * h, 64 * h + 64)
        qh, kh, vh = qv[..., sl], kvv[..., sl.start:sl.stop], kvv[..., C + sl.start:C + sl.stop]
        s = qh @ kh.transpose(1, 2) / 8
        pr = torch.exp(s - s.amax(-1, keepdim=True))
        l = pr.sum(-1, keepdim=True)
        ref = (pr @ vh) / l
        if prec == "split":
            assert U.rel_err(out[..., sl], ref) < TOL, (h, U.rel_err(out[..., sl], ref))
        else:
            bound = 2.0 ** -8 * (pr @ vh.abs()) / l + 1e-5 * ref.abs().max()
            err = (out[..., sl].double() - ref).abs()
            assert (err <= bound).all(), (h, (err / bound).max().item())


# ------------------------------------------------------------------------------------------------ the sweep
def precisions(kind):
    return ["split"] if kind == "ring" else ["split", "bf16"]


CASES = [pytest.param(case, prec, id=f"{case}-{prec}") for case, (kind, _, _) in SWEEP.items() for prec in precisions(kind)]


@pytest.mark.parametrize("case,prec", CASES)
def test_graph_launch(case, prec):
    kind, form, p = SWEEP[case]
    if kind == "embed":
        gather_case(p, prec)
    elif engine_mode(kind) == GEMM:
        gemm_case(kind, form, p["M"], p["K"], p["N"], prec)
    elif engine_mode(kind) == HALO:
        halo_case(kind, form, p, prec)
    elif kind == "attn":
        attention_case(p, prec)
    elif kind == "ring":
        ring_case(form, p)
    else:
        raise AssertionError(kind)


# ------------------------------------------------------------------------------------------------ whole-graph taps
@pytest.mark.parametrize("resize", [(64, 64), (96, 160), (640, 384)])
@pytest.mark.parametrize("version", ["Paramnet-360Cities-edina-centered", "PersNet_Paramnet-GSV-uncentered"])
def test_every_layer_tap_matches_oracle_at_other_sizes(version, resize):
    """Every layer tap against tests/oracle_resize.py at 1e-3 (the bar of test_gpu_forward.py::test_every_layer_tap_matches_oracle):
    arena aliasing, strides and group offsets at working sizes the per-launch cases cannot see together."""
    m, sd = U.make_model(version, model_kwargs={"resize": resize})
    imgs = golden_images()
    m.debug_taps(True)
    try:
        m.inference_batch(imgs)
        taps = m.read_taps()
    finally:
        m.debug_taps(False)
    otaps = {}
    ro.inference_batch(sd, version, imgs, resize, otaps)
    checked = 0
    for name, t in taps.items():
        if name.startswith("mit."):
            ref = otaps[name]
        elif name == "ll" or name.startswith("cnx.s"):
            ref = otaps[name].permute(0, 2, 3, 1)
        elif name in ("head.raw_g", "head.raw_l"):
            ref = otaps["g.raw" if name.endswith("_g") else "l.raw"]
        elif name.startswith("head."):
            k = name[5:]
            ref = torch.cat([otaps["g." + k], otaps["l." + k]], 1).permute(0, 2, 3, 1)
        else:
            continue
        e = U.rel_err(t, ref.contiguous().reshape(-1))
        assert e < 1e-3, (name, e)
        checked += 1
    assert checked > 72 and "head.raw_g" in taps and "head.raw_l" in taps
