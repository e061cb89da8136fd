"""GPU: ParamNet training's backward, one piece at a time (the ``pf_op_pn_*`` entry points, each through the host helper
``pf_param_backward`` runs it with), against a float64 restatement of the same operation.

The end-to-end check of ``test_gpu_paramnet_train.py`` bounds each gradient tensor normwise; here every kernel meets its own
reference elementwise: 5e-5 relative (max error over max reference) for the weight-gradient GEMMs on the split-bf16 engine,
1e-5 for the fp32 CUDA-core kernels, bit for bit where the operation is a permutation, an exact product or an integer sum.

Coverage is asserted, not assumed: the weight-gradient cases check the chunk plan (S, chunk) the entry point reports against a
restatement of the planner and assert which of its bounds binds; the depthwise and stem cases check the rows per block the
entry point reports and assert the multi-row and ragged-last-block partitions.

Every output is wider than its region and NaN-filled: the region must come back finite and the rest must keep NaN's bit
pattern.  The scratch inside each call is NaN-filled too, so a read of memory no kernel wrote poisons the result.  Every case
runs twice and the two results must be bit-identical (the reductions use no atomics)."""
import ctypes
import functools
import math

import pytest
import torch
import torch.nn.functional as F

import pf_test_util as U
from perspectivefields_b200 import _native, weights

pytestmark = pytest.mark.gpu

PF_ERR_ARG = -1
TOL_GEMM = 5e-5
TOL_F32 = 1e-5
PAD = 67            # NaN floats behind every output region
NAN_BITS = torch.tensor(float("nan")).view(torch.int32).item()
CNX_DIMS = (96, 192, 384, 768)
TAIL = 768 * 2 + 5 * 768 + 5


def L():
    return _native.lib()


def cdiv(a, b):
    return -(-a // b)


def ptr(t):
    return None if t is None else t.data_ptr()


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def rn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


def out_buf(numel, dtype=torch.float32):
    return torch.full((numel + PAD,), float("nan"), dtype=dtype, device="cuda")


def region(buf, numel, shape=None):
    """the owned part of an output buffer: finite, and the padding behind it still NaN's bit pattern"""
    got = buf[:numel]
    assert torch.isfinite(got).all(), "an owned element was not written (or read unwritten scratch)"
    tail = buf[numel:]
    it = torch.int32 if buf.dtype == torch.float32 else torch.int16
    want = torch.full_like(tail, float("nan")).view(it)
    assert torch.equal(tail.view(it), want), "an element outside the region was written"
    return got.view(shape) if shape is not None else got


def twice(run):
    """run(outputs...) twice on fresh outputs; the two results must be bit-identical.  Returns the first."""
    a, b = run(), run()
    for x, y in zip(a, b):
        it = torch.int32 if x.dtype == torch.float32 else torch.int16
        assert torch.equal(x.view(it), y.view(it)), "two identical calls differ"
    return a


def launches():
    return L().pf_kernel_launch_count()


def ok(status):
    _native.check(status)


# ------------------------------------------------------------------------------------------------ weight-gradient GEMMs
def pick_bn(n):
    """tma_pick_bn(n, GEMM mode): the widest tile of at most 256 columns that splits n evenly, rounded up to 32"""
    return cdiv(cdiv(n, cdiv(n, 256)), 32) * 32


def wg_plan(R, N, K, sms):
    """pn_wg_plan restated: (S, chunk, Rp, S wanted by the SM fill)"""
    tiles = cdiv(N, 128) * cdiv(K, pick_bn(K))
    s_fill = cdiv(2 * sms, tiles)
    S = max(1, min(min(s_fill, max(1, R // 1024)), 256))
    chunk = cdiv(cdiv(R, S), 64) * 64
    S = cdiv(R, chunk)
    return S, chunk, S * chunk, s_fill


# (form, C, R, regimes).  Forms, as the backward calls them: "pw2" (R, C, 4C) on GELU(u) (op 1); "pw1" (R, 4C, C) on split
# planes; "ds" (R, C, 4Cp) on split planes (the downsamples, Cp the previous stage's width); "sq" (R, 96, 96) on an fp32 source,
# a shape of one output tile that no layer has, the only way to make the 256-chunk cap bind.
WG_CASES = [
    ("pw2", 96, 1, {"R1", "S1"}),
    ("pw2", 96, 100, {"S1", "padded"}),
    ("pw2", 96, 4095, {"64k-1", "ragged", "rcap"}),
    ("pw2", 96, 200001, {"ragged", "fill"}),
    ("pw2", 192, 8191, {"64k-1", "ragged", "rcap"}),
    ("pw2", 384, 2049, {"64k+1", "ragged", "rcap"}),
    ("pw2", 768, 1025, {"64k+1", "S1", "padded"}),
    ("pw1", 96, 65537, {"64k+1", "ragged", "rcap"}),
    ("pw1", 192, 1, {"R1", "S1"}),
    ("pw1", 384, 3000, {"ragged", "rcap"}),
    ("pw1", 768, 63, {"64k-1", "S1", "padded"}),
    ("ds", 192, 20000, {"ragged", "rcap"}),
    ("ds", 192, 80000, {"ragged", "fill"}),
    ("ds", 384, 127, {"64k-1", "S1", "padded"}),
    ("ds", 768, 5121, {"64k+1", "ragged", "rcap"}),
    ("sq", 96, 300000, {"ragged", "cap256"}),
]


def wg_shape(form, C):
    """(N, K, op, split source)"""
    return {"pw2": (C, 4 * C, 1, False), "pw1": (4 * C, C, 0, True), "ds": (C, 4 * CNX_DIMS[max(0, CNX_DIMS.index(C) - 1)], 0, True),
            "sq": (C, C, 0, False)}[form]


@pytest.mark.parametrize("form,C,R,regimes", WG_CASES, ids=[f"{f}-C{c}-R{r}" for f, c, r, _ in WG_CASES])
def test_wgrad(form, C, R, regimes):
    N, K, op, split = wg_shape(form, C)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S_want, chunk_want, Rp, s_fill = wg_plan(R, N, K, sms)
    # the case covers what it claims
    binding = min(s_fill, max(1, R // 1024))
    claims = {
        "R1": R == 1, "S1": S_want == 1, "padded": S_want == 1 and Rp > R, "64k-1": R % 64 == 63, "64k+1": R % 64 == 1,
        "ragged": 1 < S_want < 256 and R % chunk_want != 0,
        "rcap": R // 1024 > 1 and R // 1024 < s_fill and binding <= 256,
        "fill": s_fill < R // 1024 and s_fill <= 256,
        "cap256": binding > 256,
    }
    assert all(claims[r] for r in regimes), {r: claims[r] for r in regimes}
    g = gen(R + N + K)
    dy = rn(g, R, N)
    if split:
        hi, lo = weights.split_hi_lo(rn(g, R, K))
        x_ref = hi.double() + lo.double()
        x = None
    else:
        x = rn(g, R, K, scale=1.5)
        hi = lo = None
        x_ref = x.double()
        if op == 1:
            x_ref = 0.5 * x_ref * (1.0 + torch.erf(x_ref / math.sqrt(2.0)))
    ref = dy.double().T @ x_ref
    S, chunk = ctypes.c_int(), ctypes.c_int()

    def run():
        out = out_buf(N * K)
        ok(L().pf_op_pn_wgrad(ptr(dy), N, ptr(x), ptr(hi), ptr(lo), op, K, R, N, K, ptr(out), ctypes.byref(S), ctypes.byref(chunk),
                              U.stream_ptr()))
        return (out,)
    out, = twice(run)
    assert (S.value, chunk.value) == (S_want, chunk_want)
    got = region(out, N * K, (N, K))
    assert U.rel_err(got, ref) < TOL_GEMM, U.rel_err(got, ref)


# ------------------------------------------------------------------------------------------------ column sums
# 524545 rows: 257 rows per partial (the 2048-partial bound binds, rpb > 256), the last partial ragged
@pytest.mark.parametrize("C", [96, 384, 3072])
@pytest.mark.parametrize("R", [1, 255, 256, 257, 524545])
def test_colsum(R, C):
    src = rn(gen(R * 7 + C), R, C) + 0.25
    # fp32 partial sums of at most ~300 terms in sequence (rows per warp, warps, partials per group, groups); the rounding errors
    # are independent, so the error stays near sqrt(300) * 2^-24 of the sum, well inside 1e-5
    ref = torch.sum(src, 0, dtype=torch.float64)

    def run():
        out = out_buf(C)
        ok(L().pf_op_pn_colsum(ptr(src), R, C, ptr(out), U.stream_ptr()))
        return (out,)
    out, = twice(run)
    assert U.rel_err(region(out, C), ref) < TOL_F32


# ------------------------------------------------------------------------------------------------ LayerNorm backward
def ln_ref(x, dy, w):
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    bd = torch.zeros_like(wd, requires_grad=True)
    (F.layer_norm(xd, (x.shape[1],), wd, bd, eps=1e-6) * dy.double()).sum().backward()
    return xd.grad, wd.grad, bd.grad


def ln_run(x, dy, w):
    R, C = x.shape

    def run():
        dx, gw = out_buf(R * C), out_buf(2 * C)
        ok(L().pf_op_pn_ln_bwd(ptr(x), ptr(dy), R, C, ptr(w), ptr(dx), ptr(gw), U.stream_ptr()))
        return dx, gw
    dx, gw = twice(run)
    return region(dx, R * C, (R, C)), region(gw, 2 * C)


# 140001 rows: 69 rows per block (rpb > 64), the last block ragged
@pytest.mark.parametrize("C", [96, 192, 384, 768])
@pytest.mark.parametrize("R", [1, 63, 64, 65, 140001])
def test_ln_bwd(R, C):
    g = gen(R + C)
    x = rn(g, R, C, scale=2.0) + rn(g, R, 1)
    dy = rn(g, R, C)
    w = 1.0 + rn(g, C, scale=0.1)
    dx, gw = ln_run(x, dy, w)
    rdx, rw, rb = ln_ref(x, dy, w)
    assert U.rel_err(dx, rdx) < TOL_F32
    assert U.rel_err(gw[:C], rw) < TOL_F32
    assert U.rel_err(gw[C:], rb) < TOL_F32


# Constant rows (variance 0, rstd = 1 / sqrt(eps) = 1000): x_hat is exactly 0, but the fp32 mean of a row of v is off from v
# by up to (C / 32 + 6) * 2^-24 |v| (C / 32 sequential adds per lane, five shuffle levels, the rounded 1 / C), and rstd
# amplifies that into x_hat.  The exact d weight (sum of dy * x_hat) is 0; ours is bounded by the sum over rows of
# |dy| (C / 32 + 6) 2^-24 |v_r| 1000.  dx = rstd (g - mean(g) - x_hat mean(g x_hat)) and d bias do not see it: 1e-5.
@pytest.mark.parametrize("C", [96, 768])
def test_ln_bwd_constant_rows(C):
    R = 4099
    g = gen(C + 1)
    v = rn(g, R, 1)
    x = v.expand(R, C).contiguous()
    dy = rn(g, R, C)
    w = 1.0 + rn(g, C, scale=0.1)
    dx, gw = ln_run(x, dy, w)
    rdx, rw, rb = ln_ref(x, dy, w)
    assert U.rel_err(dx, rdx) < TOL_F32
    assert U.rel_err(gw[C:], rb) < TOL_F32
    bound = (C / 32 + 6) * 2.0 ** -24 * 1000 * (dy.double().abs() * v.double().abs()).sum(0)
    assert (gw[:C].double() - rw).abs().le(bound).all()


# Rows at a large common offset m (std 1): the fp32 mean is off by a few units of 2^-24 m (the sum's rounding and 1/C), which
# shifts every x_hat of the row by delta ~ 4 * 2^-24 m; dx moves by rstd * delta * mean(g x_hat) ~ delta / sqrt(C) relative and
# d weight by delta * |sum dy| / |sum dy x_hat| ~ delta.  Bound: 16 * 2^-24 * m (4x margin).
@pytest.mark.parametrize("C", [96, 768])
def test_ln_bwd_large_offset(C):
    m, R = 1000.0, 4099
    g = gen(C)
    x = rn(g, R, C) + m
    dy = rn(g, R, C)
    w = 1.0 + rn(g, C, scale=0.1)
    dx, gw = ln_run(x, dy, w)
    rdx, rw, rb = ln_ref(x, dy, w)
    bound = 16 * 2.0 ** -24 * m
    assert U.rel_err(dx, rdx) < bound
    assert U.rel_err(gw[:C], rw) < bound
    assert U.rel_err(gw[C:], rb) < TOL_F32


# ------------------------------------------------------------------------------------------------ depthwise 7x7 backward
@functools.lru_cache(maxsize=None)
def rotated_kernels():
    """{C: (w [C, 1, 7, 7], w_rot [49, C])} from weights.param_net_train_weights on a state dict whose block-0 depthwise
    kernels of stages 0 and 3 are random (everything else zero)."""
    pn = weights.PN
    g = gen(77)
    sd = {pn + "norm.weight": torch.zeros(768, device="cuda")}
    for k in (1, 2, 3):
        sd[f"{pn}downsample_layers.{k}.1.weight"] = torch.zeros(CNX_DIMS[k], CNX_DIMS[k - 1], 2, 2, device="cuda")
    for s, C in enumerate(CNX_DIMS):
        for j in range((3, 3, 9, 3)[s]):
            k = f"{pn}stages.{s}.{j}."
            sd[k + "pwconv1.weight"] = torch.zeros(4 * C, C, device="cuda")
            sd[k + "pwconv2.weight"] = torch.zeros(C, 4 * C, device="cuda")
            sd[k + "dwconv.weight"] = rn(g, C, 1, 7, 7, scale=0.2)
    out = weights.param_net_train_weights(sd, {})
    return {C: (sd[f"{pn}stages.{s}.0.dwconv.weight"], out[f"pn.s{s}.b0.dw.wr"]) for s, C in ((0, 96), (3, 768))}


def rows_per_block(rows):
    return max(1, cdiv(rows, 1024))


DW_CASES = [(2, h, w, C) for h, w in [(1, 1), (2, 2), (3, 5), (7, 7), (8, 8), (9, 13), (10, 10), (16, 16), (64, 96), (80, 80)]
            for C in (96, 768)]
# batches past 1024 image rows: two rows per block, every block full; three rows per block, a ragged last block (one row)
DW_CASES += [(13, 80, 80, 96), (26, 80, 80, 96), (301, 7, 7, 768)]


@pytest.mark.parametrize("B,H,W,C", DW_CASES)
def test_dw7_bwd(B, H, W, C):
    rows = B * H
    if B > 2:
        rpb_want = rows_per_block(rows)
        assert rpb_want > 1
        assert (rows % rpb_want != 0) == (B != 13)
    wt, w_rot = rotated_kernels()[C]
    g = gen(B * H * W + C)
    x = rn(g, B, H, W, C)
    dt = rn(g, B, H, W, C)
    n = B * H * W * C
    rpb = ctypes.c_int()

    def run():
        dw, dx = out_buf(50 * C), out_buf(n)
        ok(L().pf_op_pn_dw7_bwd(ptr(x), ptr(dt), B, H, W, C, ptr(w_rot), ptr(dw), ptr(dx), ctypes.byref(rpb), U.stream_ptr()))
        return dw, dx
    dw, dx = twice(run)
    assert rpb.value == rows_per_block(rows)
    dw, dx = region(dw, 50 * C, (50, C)), region(dx, n, (B, H, W, C))
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    wd = wt.double().requires_grad_(True)
    bd = torch.zeros(C, dtype=torch.float64, device="cuda", requires_grad=True)
    (F.conv2d(xd, wd, bd, padding=3, groups=C) * dt.double().permute(0, 3, 1, 2)).sum().backward()
    assert U.rel_err(dw[:49], wd.grad.reshape(C, 49).T) < TOL_F32
    assert U.rel_err(dw[49], bd.grad) < TOL_F32
    assert U.rel_err(dx, xd.grad.permute(0, 2, 3, 1)) < TOL_F32


# ------------------------------------------------------------------------------------------------ stem backward
# (B, OH, OW): uncentred 64 x 64 input; two rows per block (B = 13 at 80 x 80); three rows per block with a ragged last block
# (B = 26); rectangular; the smallest (32 x 32 input)
STEM_CASES = [(2, 16, 16), (13, 80, 80), (26, 80, 80), (2, 64, 96), (3, 8, 8)]


@pytest.mark.parametrize("B,OH,OW", STEM_CASES)
def test_stem_bwd(B, OH, OW):
    rows = B * OH
    rpb_want = rows_per_block(rows)
    if B >= 13:
        assert rpb_want > 1
        assert (rows % rpb_want != 0) == (B == 26)
    g = gen(B * OH * OW)
    pin = rn(g, B, 4 * OH, 4 * OW, 4)
    dS = rn(g, B, OH, OW, 96)
    wt = rn(g, 96, 3, 4, 4, scale=0.1)                             # [co, ci, ky, kx]
    w = wt.permute(2, 3, 1, 0).reshape(48, 96).contiguous()        # the engine's [(ky, kx, ci)][co]
    npin = B * 16 * OH * OW * 4
    rpb = ctypes.c_int()

    def run():
        dw, dpin = out_buf(49 * 96), out_buf(npin)
        ok(L().pf_op_pn_stem_bwd(ptr(pin), ptr(dS), ptr(w), B, OH, OW, ptr(dw), ptr(dpin), ctypes.byref(rpb), U.stream_ptr()))
        return dw, dpin
    dw, dpin = twice(run)
    assert rpb.value == rpb_want
    dw = region(dw, 49 * 96, (49, 96))
    # channel 3 of the packed input has no gradient and is not written
    dpin = dpin[:npin].view(B, 4 * OH, 4 * OW, 4)
    assert torch.equal(dpin[..., 3].contiguous().view(torch.int32), torch.full_like(dpin[..., 3], float("nan")).view(torch.int32))
    assert torch.isfinite(dpin[..., :3]).all()
    pd = pin[..., :3].double().permute(0, 3, 1, 2).requires_grad_(True)
    wd = wt.double().requires_grad_(True)
    bd = torch.zeros(96, dtype=torch.float64, device="cuda", requires_grad=True)
    (F.conv2d(pd, wd, bd, stride=4) * dS.double().permute(0, 3, 1, 2)).sum().backward()
    assert U.rel_err(dw[:48], wd.grad.permute(2, 3, 1, 0).reshape(48, 96)) < TOL_F32
    assert U.rel_err(dw[48], bd.grad) < TOL_F32
    assert U.rel_err(dpin[..., :3], pd.grad.permute(0, 2, 3, 1)) < TOL_F32


# ------------------------------------------------------------------------------------------------ fields gradient
def fields_grad(B, IH, IW, OH, OW, seed):
    """(ours, autograd of F.interpolate(mode="nearest")): integer-valued dpin, so every sum is exact in fp32"""
    dpin = torch.randint(-8, 9, (B, OH, OW, 4), generator=gen(seed), device="cuda").float()
    ng = B * 2 * IH * IW

    def run():
        dg, dl = out_buf(ng), out_buf(ng // 2)
        ok(L().pf_op_pn_fields_grad(ptr(dpin), B, IH, IW, OH, OW, ptr(dg), ptr(dl), U.stream_ptr()))
        return dg, dl
    dg, dl = twice(run)
    src = torch.zeros(B, 3, IH, IW, requires_grad=True)
    F.interpolate(src, (OH, OW), mode="nearest").backward(dpin[..., :3].permute(0, 3, 1, 2).cpu())
    got = torch.cat((region(dg, ng, (B, 2, IH, IW)), region(dl, ng // 2, (B, 1, IH, IW))), 1).cpu()
    return got, src.grad


NET_SIDES = list(range(64, 641, 32))
PN_SIDES = list(range(32, 321, 32))


@pytest.mark.parametrize("net", NET_SIDES)
def test_fields_grad_every_side_pair(net):
    # the map is separable: rows run net -> ParamNet side, columns ParamNet -> net side, so both directions of every pair
    for pn in PN_SIDES:
        got, ref = fields_grad(1, net, pn, pn, net, seed=net * 1000 + pn)
        assert torch.equal(got, ref), (net, pn)
        assert torch.equal(got == 0, ref == 0)


@pytest.mark.parametrize("B,IH,IW,OH,OW", [(3, 640, 64, 32, 320), (2, 96, 608, 320, 32), (2, 256, 384, 256, 384),
                                           (3, 384, 256, 96, 160), (1, 64, 64, 320, 320), (2, 480, 640, 224, 224)])
def test_fields_grad_rectangular(B, IH, IW, OH, OW):
    got, ref = fields_grad(B, IH, IW, OH, OW, seed=IH + IW)
    assert torch.equal(got, ref)
    assert torch.equal(got == 0, ref == 0)


# ------------------------------------------------------------------------------------------------ tail backward
@pytest.mark.parametrize("n", [1, 3, 300])
@pytest.mark.parametrize("HW", [1, 4, 96, 100])
def test_tail_bwd(HW, n):
    g = gen(HW * 1000 + n)
    feat = rn(g, n, HW, 768) + rn(g, n, 1, 768, scale=0.5)
    nw, nb = 1.0 + rn(g, 768, scale=0.1), rn(g, 768, scale=0.1)
    hw, draw = rn(g, 5, 768, scale=0.05), rn(g, n, 5)

    def run():
        dx, gr = out_buf(n * HW * 768), out_buf(TAIL)
        ok(L().pf_op_pn_tail_bwd(ptr(feat), n, HW, ptr(nw), ptr(nb), ptr(hw), ptr(draw), ptr(dx), ptr(gr), U.stream_ptr()))
        return dx, gr
    dx, gr = twice(run)
    dx, gr = region(dx, n * HW * 768, (n, HW, 768)), region(gr, TAIL)
    f = feat.double().requires_grad_(True)
    p = [t.double().requires_grad_(True) for t in (nw, nb, hw)]
    hb = torch.zeros(5, dtype=torch.float64, device="cuda", requires_grad=True)
    raw = F.layer_norm(f.mean(1), (768,), p[0], p[1], eps=1e-6) @ p[2].T + hb
    (raw * draw.double()).sum().backward()
    assert U.rel_err(dx, f.grad) < TOL_F32
    for got, want in ((gr[:768], p[0].grad), (gr[768:1536], p[1].grad), (gr[1536:1536 + 3840], p[2].grad.reshape(-1)), (gr[-5:], hb.grad)):
        assert U.rel_err(got, want) < TOL_F32


# ------------------------------------------------------------------------------------------------ pwconv2 gradients, GELU', split, col2im
@pytest.mark.parametrize("C", [96, 768])
def test_pw2_grads(C):
    K = 4 * C
    g = gen(C)
    G, sdy, gamma, b = rn(g, C, K), rn(g, C), rn(g, C, scale=0.1), rn(g, C, scale=0.1)
    whi, wlo = weights.split_hi_lo(rn(g, C, K, scale=0.05))

    def run():
        dW, db, dgam = out_buf(C * K), out_buf(C), out_buf(C)
        ok(L().pf_op_pn_pw2_grads(ptr(G), ptr(sdy), C, K, ptr(gamma), ptr(whi), ptr(wlo), ptr(b), ptr(dW), ptr(db), ptr(dgam), U.stream_ptr()))
        return dW, db, dgam
    dW, db, dgam = twice(run)
    # one fp32 product each: the correctly rounded float64 product, bit for bit
    assert torch.equal(region(dW, C * K, (C, K)), (gamma.double()[:, None] * G.double()).float())
    assert torch.equal(region(db, C), (gamma.double() * sdy.double()).float())
    W = whi.double() + wlo.double()
    assert U.rel_err(region(dgam, C), (W * G.double()).sum(1) + b.double() * sdy.double()) < TOL_F32


def test_gelu_bwd():
    g = gen(5)
    special = torch.tensor([0.0, 6.0, -6.0, 10.0, -10.0, 40.0, -40.0], device="cuda")
    u0 = torch.cat((special, rn(g, 1 << 20, scale=3.0), torch.linspace(-12, 12, 100003, device="cuda")))
    n = u0.numel()
    dh = rn(g, n)

    def run():
        u = torch.cat((u0, torch.full((PAD,), float("nan"), device="cuda")))
        hi, lo = out_buf(n, torch.bfloat16), out_buf(n, torch.bfloat16)
        ok(L().pf_op_pn_gelu_bwd(ptr(dh), ptr(u), n, ptr(hi), ptr(lo), U.stream_ptr()))
        return u, hi, lo
    u, hi, lo = twice(run)
    got = region(u, n)
    x = u0.double()
    d = 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    ref = dh.double() * d
    # GELU' is at most ~1.13: 1e-5 of |dh| per element
    assert ((got.double() - ref).abs() <= TOL_F32 * dh.double().abs()).all()
    assert torch.equal(got[0], dh[0] * 0.5)                                  # GELU'(0) = 1/2
    assert torch.equal(got[5], dh[5]) and got[6].item() == 0.0              # GELU'(40) = 1, GELU'(-40) = 0
    want_hi, want_lo = weights.split_hi_lo(got)
    assert torch.equal(region(hi, n), want_hi) and torch.equal(region(lo, n), want_lo)


@pytest.mark.parametrize("scaled", [False, True])
def test_scale_split(scaled):
    R, C = 1001, 384
    g = gen(11)
    src, scale = rn(g, R, C), (rn(g, C) if scaled else None)

    def run():
        hi, lo = out_buf(R * C, torch.bfloat16), out_buf(R * C, torch.bfloat16)
        ok(L().pf_op_pn_scale_split(ptr(src), ptr(scale), R * C, C, ptr(hi), ptr(lo), U.stream_ptr()))
        return hi, lo
    hi, lo = twice(run)
    v = src * scale if scaled else src                       # one fp32 product, as the kernel
    want_hi, want_lo = weights.split_hi_lo(v)
    assert torch.equal(region(hi, R * C, (R, C)), want_hi)
    assert torch.equal(region(lo, R * C, (R, C)), want_lo)


@pytest.mark.parametrize("B,H,W,C", [(2, 10, 6, 96), (1, 2, 2, 192), (3, 40, 40, 96), (2, 20, 14, 384)])
def test_col2im2(B, H, W, C):
    dP = rn(gen(H * W + C), B * (H // 2) * (W // 2), 4 * C)
    n = B * H * W * C

    def run():
        out = out_buf(n)
        ok(L().pf_op_pn_col2im2(ptr(dP), B, H, W, C, ptr(out), U.stream_ptr()))
        return (out,)
    out, = twice(run)
    # the patch gather: row (b, y / 2, x / 2), column ((y % 2) * 2 + x % 2) * C + c
    want = dP.view(B, H // 2, W // 2, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)
    assert torch.equal(region(out, n, (B, H, W, C)), want)


# ------------------------------------------------------------------------------------------------ rejected arguments
def test_rejected_arguments_launch_nothing():
    t = torch.zeros(1 << 16, device="cuda")
    p, q = t.data_ptr(), t[1:].data_ptr()                        # q: 4-byte aligned only
    h = t.view(torch.bfloat16).data_ptr()
    S, ch, rpb = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    s = U.stream_ptr()
    bad = [
        lambda: L().pf_op_pn_wgrad(None, 96, p, None, None, 0, 96, 64, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),
        lambda: L().pf_op_pn_wgrad(p, 96, p, h, h, 0, 96, 64, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),      # two sources
        lambda: L().pf_op_pn_wgrad(p, 96, None, None, None, 0, 96, 64, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),  # none
        lambda: L().pf_op_pn_wgrad(p, 96, None, h, None, 0, 96, 64, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),     # half a pair
        lambda: L().pf_op_pn_wgrad(p, 96, None, h, h, 1, 96, 64, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),        # GELU of planes
        lambda: L().pf_op_pn_wgrad(p, 96, p, None, None, 2, 96, 64, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),
        lambda: L().pf_op_pn_wgrad(p, 96, p, None, None, 0, 96, 0, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),
        lambda: L().pf_op_pn_wgrad(p, 95, p, None, None, 0, 96, 64, 96, 96, p, ctypes.byref(S), ctypes.byref(ch), s),
        lambda: L().pf_op_pn_wgrad(p, 96, p, None, None, 0, 96, 64, 96, 96, p, None, ctypes.byref(ch), s),
        lambda: L().pf_op_pn_colsum(p, 0, 96, p, s),
        lambda: L().pf_op_pn_colsum(None, 4, 96, p, s),
        lambda: L().pf_op_pn_ln_bwd(p, p, 4, 100, p, p, p, s),
        lambda: L().pf_op_pn_ln_bwd(p, p, 4, 800, p, p, p, s),
        lambda: L().pf_op_pn_ln_bwd(p, p, 0, 96, p, p, p, s),
        lambda: L().pf_op_pn_ln_bwd(p, p, 4, 96, None, p, p, s),
        lambda: L().pf_op_pn_dw7_bwd(p, p, 1, 4, 4, 48, p, p, p, ctypes.byref(rpb), s),
        lambda: L().pf_op_pn_dw7_bwd(p, p, 0, 4, 4, 96, p, p, p, ctypes.byref(rpb), s),
        lambda: L().pf_op_pn_dw7_bwd(q, p, 1, 4, 4, 96, p, p, p, ctypes.byref(rpb), s),
        lambda: L().pf_op_pn_dw7_bwd(p, p, 1, 4, 4, 96, None, p, p, ctypes.byref(rpb), s),
        lambda: L().pf_op_pn_stem_bwd(q, p, p, 1, 4, 4, p, p, ctypes.byref(rpb), s),
        lambda: L().pf_op_pn_stem_bwd(p, p, p, 1, 0, 4, p, p, ctypes.byref(rpb), s),
        lambda: L().pf_op_pn_stem_bwd(p, p, None, 1, 4, 4, p, p, ctypes.byref(rpb), s),
        lambda: L().pf_op_pn_fields_grad(p, 0, 8, 8, 8, 8, p, p, s),
        lambda: L().pf_op_pn_fields_grad(q, 1, 8, 8, 8, 8, p, p, s),
        lambda: L().pf_op_pn_fields_grad(p, 1, 8, 8, 8, 8, p, None, s),
        lambda: L().pf_op_pn_tail_bwd(p, 0, 4, p, p, p, p, p, p, s),
        lambda: L().pf_op_pn_tail_bwd(p, 1, 0, p, p, p, p, p, p, s),
        lambda: L().pf_op_pn_tail_bwd(p, 1, 4, p, p, p, None, p, p, s),
        lambda: L().pf_op_pn_pw2_grads(p, p, 0, 384, p, h, h, p, p, p, p, s),
        lambda: L().pf_op_pn_pw2_grads(p, p, 96, 384, p, h, None, p, p, p, p, s),
        lambda: L().pf_op_pn_gelu_bwd(p, p, 0, None, None, s),
        lambda: L().pf_op_pn_gelu_bwd(p, p, 64, h, None, s),
        lambda: L().pf_op_pn_scale_split(p, None, 100, 96, h, h, s),
        lambda: L().pf_op_pn_scale_split(p, None, 96, 96, h, None, s),
        lambda: L().pf_op_pn_col2im2(p, 1, 3, 4, 96, p, s),
        lambda: L().pf_op_pn_col2im2(p, 1, 4, 4, 0, p, s),
    ]
    for i, call in enumerate(bad):
        before = launches()
        assert call() == PF_ERR_ARG, i
        assert launches() == before, i
