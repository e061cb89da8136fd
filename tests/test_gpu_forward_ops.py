"""GPU: the forward graph's CUDA-core kernels (``csrc/layers.cuh``), one launch at a time, against a float64 restatement of the
same operation, in every output form and at every shape the graph launches them with.

Each entry point (``pf_op_layernorm_ex``, ``pf_op_dwconv3x3_gelu_ex``, ``pf_op_dwconv7x7``, ``pf_op_upsample2x_ex``,
``pf_op_stem_gather``, ``pf_op_pn_stem``, ``pf_op_pack_fields``, ``pf_op_param_tail``, ``pf_op_pred_tail``) calls the ``Fwd``
helper ``pf_forward`` launches the kernel with, so it runs the graph's grid, block and arguments.  The shapes come from
``graph_launches`` / ``paramnet_launches``, a restatement of the shape arithmetic of ``run_forward`` and ``fwd_paramnet``
(``pf_b200.cu``), over working sizes chosen to reach the kernels' partition edges; ``test_sweep_reaches_every_partition_edge``
asserts that they do.

Bounds: 1e-5 (max error over max reference) for fp32 CUDA-core arithmetic, 1e-6 for the upsample (two taps of 1/4 and 3/4 per
direction), bit for bit for gathers and splits.  A split output is checked bit for bit against the fp32 output of the same
launch: hi = bf16(y) and lo = bf16(y - hi), both round-to-nearest-even like the kernel's ``__float2bfloat16_rn``, and the
graph's split-only launch must produce the same bits.

Every output sits at the start of a NaN-filled buffer: the owned region must come back finite and the rest must keep NaN's
bit pattern.  Every input sits between NaN guards, so a read past either end poisons the result.  Every case runs twice and
the two results must be bit-identical."""
import ctypes
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

import pf_test_util as U
from perspectivefields_b200 import _native

pytestmark = pytest.mark.gpu

PF_ERR_ARG = -1
PF_PARAM_CENTERED, PF_PARAM_UNCENTERED = _native.PF_PARAM_CENTERED, _native.PF_PARAM_UNCENTERED
TOL_F32 = 1e-5
TOL_UP = 1e-6
PAD = 67            # NaN elements behind every output region
GUARD = 64          # NaN floats before and after every input (256 bytes: the input stays 16-byte aligned)
MIT_DIMS, MIT_SR = (64, 128, 320, 512), (8, 4, 2, 1)
CNX_DIMS = (96, 192, 384, 768)
EW_THREADS = 132 * 32 * 256     # one pass of a grid-stride loop: ew_grid's block cap (common.cuh) x 256 threads
PX = 4                          # PF_DW3_PX = PF_DW7_PX: output pixels per thread along x


def L():
    return _native.lib()


def ptr(t):
    return None if t is None else t.data_ptr()


def gen(key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(str(key).encode()))


def rn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


def ok(status):
    _native.check(status)


def launches():
    return L().pf_kernel_launch_count()


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def out_buf(numel, dtype=torch.float32):
    return torch.full((numel + PAD,), float("nan"), dtype=dtype, device="cuda")


def guarded(t):
    """a copy of t between NaN guards"""
    flat = t.reshape(-1)
    buf = torch.full((flat.numel() + 2 * GUARD,), float("nan"), dtype=t.dtype, device="cuda")
    buf[GUARD:GUARD + flat.numel()] = flat
    return buf[GUARD:GUARD + flat.numel()].view(t.shape)


def region(buf, shape, chans=None, finite=True):
    """the owned part of an output buffer of the given shape (channels chans = (c0, c1) of the last dimension when only those
    are owned): finite, and every other element still NaN's bit pattern"""
    numel = math.prod(shape)
    full = buf[:numel].view(shape)
    owned = full if chans is None else full[..., chans[0]:chans[1]]
    if finite:
        assert torch.isfinite(owned).all(), "an owned element was not written (or read unwritten memory)"
    nan = bits(torch.full((1,), float("nan"), dtype=buf.dtype, device="cuda"))
    assert (bits(buf[numel:]) == nan).all(), "an element behind the region was written"
    if chans is not None:
        rest = torch.cat((full[..., :chans[0]].reshape(-1), full[..., chans[1]:].reshape(-1)))
        assert (bits(rest) == nan).all(), "a channel outside the region was written"
    return owned


def twice(run):
    """run() twice on fresh outputs; the two results must be bit-identical.  Returns the first."""
    a, b = run(), run()
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(bits(x), bits(y)), "two identical calls differ"
    return a


def rel(got, ref):
    """max |got - ref| over max |ref| (on the device)"""
    return ((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def check_split(y, hi, lo):
    want_hi = y.bfloat16()
    assert torch.equal(bits(hi), bits(want_hi)), "hi plane != bf16(y)"
    assert torch.equal(bits(lo), bits((y - want_hi.float()).bfloat16())), "lo plane != bf16(y - hi)"


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def dw_ref(x, w, b, k):
    """float64 depthwise k x k conv (pad k // 2) + bias on NHWC x; w [k * k][C] taps (ky, kx)"""
    B, H, W, C = x.shape
    p = k // 2
    xp = F.pad(x.double(), (0, 0, p, p, p, p))
    out = b.double().expand(B, H, W, C).clone()
    for ky in range(k):
        for kx in range(k):
            out += xp[:, ky:ky + H, kx:kx + W, :] * w[ky * k + kx].double()
    return out


# ------------------------------------------------------------------------------------------------ the graph's launches
def graph_launches(NH, NW, n):
    """(kernel, form, shape) of the CUDA-core launches of run_forward (pf_b200.cu) at working size NH x NW and batch n:
    the stage grids are NH / 4 .. NH / 32 (RH[s] = NH >> (s + 2)), the attention keys nkv = RH[3] RW[3], the head levels run on the
    stage grids (level l on stage l - 1's), and the prediction tails on NH x NW."""
    RH, RW = [NH >> (s + 2) for s in range(4)], [NW >> (s + 2) for s in range(4)]
    nkv = RH[3] * RW[3]
    out = [("stem_gather", "split", dict(B=n, IH=NH, IW=NW, stride=2)),        # ll_enc conv 7x7 / 2
           ("stem_gather", "split", dict(B=n, IH=NH, IW=NW, stride=4))]        # patch_embed1 7x7 / 4
    for s in range(4):
        C, sr, rows = MIT_DIMS[s], MIT_SR[s], n * RH[s] * RW[s]
        out.append(("ln", "fp32", dict(rows=rows, C=C, eps=1e-5)))           # the patch embedding's LayerNorm
        if sr > 1:
            # ln1, also written as the im2col matrix of the spatial-reduction conv; the reduced tokens' LayerNorm
            out.append(("ln", "split+patch", dict(rows=rows, C=C, eps=1e-6, RH=RH[s], RW=RW[s], sr=sr)))
            out.append(("ln", "split", dict(rows=n * nkv, C=C, eps=1e-5)))
        out.append(("ln", "split", dict(rows=rows, C=C, eps=1e-6)))          # ln1 (sr 1), ln2, the stage norm
        out.append(("dw3", "split", dict(B=n, H=RH[s], W=RW[s], C=4 * C)))   # Mix-FFN depthwise conv, into fc2's split planes
    for lvl in (4, 3, 2, 1):   # fusion upsample: fp32 at levels 4..2, split planes (conv_fuse_conv0's input) at level 1
        out.append(("up", "fp32" if lvl > 1 else "split", dict(B=n, H=RH[lvl - 1], W=RW[lvl - 1], C=512, ldi=512, icoff=0, ldo=512, ocoff=0)))
    # prediction tails on conv_fuse_conv1's output [n * NH * NW, 64] (gravity channels 0-31, latitude 32-63): the 73 / 180 logits
    # of classification heads, normalise / clamp of a regression head whose partner classifies
    HW = NH * NW
    out += [("pred", "", dict(B=n, HW=HW, NC=73, mode=0, coff=0)), ("pred", "", dict(B=n, HW=HW, NC=180, mode=0, coff=32)),
            ("pred", "", dict(B=n, HW=HW, NC=2, mode=1, coff=0)), ("pred", "", dict(B=n, HW=HW, NC=1, mode=2, coff=32))]
    return out


def paramnet_launches(NH, NW, n, kind, size):
    """fwd_paramnet's CUDA-core launches: the fields at NH x NW packed to SH x SW (the working size when centred, size x size
    otherwise), the 4x4 / 4 stem and its LayerNorm, per stage the downsample's LayerNorm in 2x2 patch order (stages 1-3), the
    depthwise 7x7 and the block LayerNorm, and the tail on the last stage's grid"""
    SH, SW = (NH, NW) if kind == PF_PARAM_CENTERED else (size, size)
    rh, rw = SH // 4, SW // 4
    out = [("pack", "", dict(B=n, IH=NH, IW=NW, OH=SH, OW=SW)), ("pn_stem", "", dict(B=n, SH=SH, SW=SW)),
           ("ln", "fp32", dict(rows=n * rh * rw, C=96, eps=1e-6))]
    for s in range(4):
        if s > 0:
            out.append(("ln", "patch", dict(rows=n * rh * rw, C=CNX_DIMS[s - 1], eps=1e-6, RH=rh, RW=rw, sr=2)))
            rh, rw = rh // 2, rw // 2
        out.append(("dw7", "fp32", dict(B=n, H=rh, W=rw, C=CNX_DIMS[s])))
        out.append(("ln", "split", dict(rows=n * rh * rw, C=CNX_DIMS[s], eps=1e-6)))
    out.append(("tail", "", dict(n=n, HW=rh * rw, kind=kind)))
    return out


# Working sizes: 64 x 64 (stage-4 grid 2 x 2, 4 keys), 96 x 160 (3 x 5), 224 x 352 (7 x 11), 320 x 320 at a batch whose stage-1
# depthwise conv, level-1 upsample and ll_enc gather need more than one grid-stride pass, and the largest side (640) and key
# count (16 x 16) at batch 1.  ParamNet: uncentred at 32 (grids down to 1 x 1, fields resampled down) and 224 (resampled up),
# centred at 320 (a batch whose stage-0 7x7 needs two passes), 224 x 352 and 96 x 160.
GRAPH_SIZES = [(64, 64, 16), (96, 160, 3), (224, 352, 2), (320, 320, 22), (640, 384, 1), (512, 512, 1)]
PARAMNET_SIZES = [(96, 160, 4, PF_PARAM_UNCENTERED, 32), (64, 64, 2, PF_PARAM_UNCENTERED, 224), (320, 320, 60, PF_PARAM_CENTERED, 0),
                  (224, 352, 2, PF_PARAM_CENTERED, 0), (96, 160, 3, PF_PARAM_CENTERED, 0)]


def case_id(kernel, form, p):
    return "-".join([kernel] + ([form] if form else []) + [f"{k}{v}" for k, v in p.items()])


def sweep():
    cases = {}
    for NH, NW, n in GRAPH_SIZES:
        for c in graph_launches(NH, NW, n):
            cases.setdefault(case_id(*c), c)
    for NH, NW, n, kind, size in PARAMNET_SIZES:
        for c in paramnet_launches(NH, NW, n, kind, size):
            cases.setdefault(case_id(*c), c)
    return cases


SWEEP = sweep()


def ln_rows_per_block(C):
    """layernorm_launch: 8 warps x (32 / LANES) lane groups x NR rows in flight"""
    return 64 if C <= 64 else 32 if C <= 128 else 8


def dw_threads(B, H, W, C):
    return B * ((H + 1) // 2) * ((W + PX - 1) // PX) * (C // 4)


def test_sweep_reaches_every_partition_edge():
    cases = list(SWEEP.values())

    def shapes(kernel):
        return [p for k, _, p in cases if k == kernel]
    # LayerNorm: every instantiation (C <= 64, <= 128, <= 384, > 384) with an exact and a ragged last block, in every form
    ln = shapes("ln")
    for lo, hi in ((0, 64), (64, 128), (128, 384), (384, 768)):
        rows = [p["rows"] % ln_rows_per_block(p["C"]) for p in ln if lo < p["C"] <= hi]
        assert 0 in rows and any(r != 0 for r in rows), (lo, hi)
    assert {p["C"] for p in ln} == set(MIT_DIMS) | set(CNX_DIMS)
    assert {f for k, f, _ in cases if k == "ln"} == {"fp32", "split", "split+patch", "patch"}
    assert {p["sr"] for k, f, p in cases if k == "ln" and "patch" in f} == {2, 4, 8}
    assert any(p["RH"] // p["sr"] == 1 and p["RW"] // p["sr"] == 1 for k, f, p in cases if f == "patch")   # down to a 1 x 1 map
    # depthwise convs: every residue of W mod the 4-pixel groups, odd heights (a half-empty two-row tile), a 1 x 1 grid
    for kernel in ("dw3", "dw7"):
        assert {p["W"] % PX for p in shapes(kernel)} == {0, 1, 2, 3}, kernel
        assert any(p["H"] % 2 for p in shapes(kernel)), kernel
    assert any(p["H"] == p["W"] == 1 for p in shapes("dw7"))
    # upsample: odd widths (the last pair of low-resolution columns has one)
    assert any(p["W"] % 2 for p in shapes("up"))
    # grid-stride loops that need more than one pass
    assert any(dw_threads(p["B"], p["H"], p["W"], p["C"]) > EW_THREADS for p in shapes("dw3"))
    assert any(dw_threads(p["B"], p["H"], p["W"], p["C"]) > EW_THREADS for p in shapes("dw7"))
    assert any(p["B"] * p["H"] * ((p["W"] + 1) // 2) * 128 > EW_THREADS for p in shapes("up"))
    assert any(p["B"] * ((p["IH"] - 1) // p["stride"] + 1) * ((p["IW"] - 1) // p["stride"] + 1) * 20 > EW_THREADS for p in shapes("stem_gather"))
    # nearest resample of the fields: up, down and identity
    pk = shapes("pack")
    assert any(p["OH"] > p["IH"] for p in pk) and any(p["OH"] < p["IH"] for p in pk) and any(p["OH"] == p["IH"] for p in pk)
    assert {p["kind"] for p in shapes("tail")} == {PF_PARAM_CENTERED, PF_PARAM_UNCENTERED}
    assert {(p["mode"], p["NC"]) for p in shapes("pred")} == {(0, 73), (0, 180), (1, 2), (2, 1)}


# ------------------------------------------------------------------------------------------------ LayerNorm
def run_ln(x, w, b, eps, outs, RH=0, RW=0, sr=0):
    """outs: which of "y", "split", "patch" to write.  Returns (y, hi, lo, phi, plo), None for the ones not written."""
    rows, C = x.shape
    n = rows * C
    y = out_buf(n) if "y" in outs else None
    hi, lo = (out_buf(n, torch.bfloat16), out_buf(n, torch.bfloat16)) if "split" in outs else (None, None)
    phi, plo = (out_buf(n, torch.bfloat16), out_buf(n, torch.bfloat16)) if "patch" in outs else (None, None)
    ok(L().pf_op_layernorm_ex(ptr(x), ptr(y), ptr(hi), ptr(lo), ptr(phi), ptr(plo), rows, C, ptr(w), ptr(b), eps, RH, RW, sr, U.stream_ptr()))
    return y, hi, lo, phi, plo


def ln_params(g, C):
    return 1.0 + rn(g, C, scale=0.2), rn(g, C, scale=0.2)


def check_ln(x, w, b, eps, form, RH=0, RW=0, sr=0, ref=None, tol=TOL_F32):
    """every output at once (fp32 against float64, the planes against the fp32 bits), then the graph's form alone (same bits)"""
    rows, C = x.shape
    patch = "patch" in form
    full = ("y", "split", "patch") if patch else ("y", "split")
    y, hi, lo, phi, plo = twice(lambda: run_ln(x, w, b, eps, full, RH, RW, sr))
    y = region(y, (rows, C))
    hi, lo = region(hi, (rows, C)), region(lo, (rows, C))
    if ref is None:
        ref = F.layer_norm(x.double(), (C,), w.double(), b.double(), eps)
    assert rel(y, ref) < tol, rel(y, ref)
    check_split(y, hi, lo)
    if patch:
        # token (b, y, x) -> row (b, y / sr, x / sr), column ((y % sr) sr + x % sr) C + c
        B = rows // (RH * RW)
        phi, plo = region(phi, (rows, C)), region(plo, (rows, C))
        for plane, row_plane in ((phi, hi), (plo, lo)):
            want = row_plane.view(B, RH // sr, sr, RW // sr, sr, C).permute(0, 1, 3, 2, 4, 5).reshape(rows, C)
            assert torch.equal(bits(plane), bits(want)), "patch-order plane != permuted row-order plane"
    graph = {"fp32": ("y",), "split": ("split",), "split+patch": ("split", "patch"), "patch": ("patch",)}[form]
    got = twice(lambda: run_ln(x, w, b, eps, graph, RH, RW, sr))
    for a, want in zip(got, (y, hi, lo, phi, plo)):
        if a is not None:
            assert torch.equal(bits(region(a, (rows, C))), bits(want)), "the graph's form differs from the full launch"
    return y


def ln_case(p, form):
    rows, C = p["rows"], p["C"]
    g = gen((rows, C, form))
    x = guarded(rn(g, rows, C, scale=2.0) + rn(g, rows, 1, scale=3.0))
    w, b = ln_params(g, C)
    check_ln(x, w, b, p["eps"], form, p.get("RH", 0), p.get("RW", 0), p.get("sr", 0))


# Constant rows: the float64 LayerNorm returns b exactly, ours returns b + w (v - mean) rstd with the fp32 mean of C copies of v
# off by at most (C / 32 + 8) units of 2^-24 |v| (per lane two quad adds and up to six sequential ones, five shuffle levels, the
# rounded 1 / C and its product) and rstd = 1 / sqrt(var + eps) <= 1 / sqrt(eps); plus the final rounding of b.
@pytest.mark.parametrize("C", [64, 96, 320, 768])
def test_layernorm_constant_rows(C):
    rows, eps = 333, 1e-6
    g = gen(("const", C))
    v = rn(g, rows, 1, scale=4.0)
    x = guarded(v.expand(rows, C).contiguous())
    w, b = ln_params(g, C)
    y, hi, lo, _, _ = twice(lambda: run_ln(x, w, b, eps, ("y", "split")))
    y = region(y, (rows, C))
    check_split(y, region(hi, (rows, C)), region(lo, (rows, C)))
    bound = (C / 32 + 8) * 2.0 ** -24 * v.double().abs() * w.double().abs() / math.sqrt(eps) + 2.0 ** -24 * b.double().abs()
    assert ((y.double() - b.double()).abs() <= bound).all()


# Rows at a large common offset m (unit spread): the fp32 mean is off by at most (C / 32 + 8) 2^-24 m (as above), which shifts
# every normalised value of the row by that much times rstd ~ 1, so y moves by |w| times it; the rest is the 1e-5 of fp32 arithmetic.
@pytest.mark.parametrize("C", [64, 128, 384, 768])
def test_layernorm_large_offset(C):
    rows, m, eps = 1001, 1000.0, 1e-6
    g = gen(("offset", C))
    x = guarded(rn(g, rows, C) + m)
    w, b = ln_params(g, C)
    ref = F.layer_norm(x.double(), (C,), w.double(), b.double(), eps)
    y, _, _, _, _ = twice(lambda: run_ln(x, w, b, eps, ("y",)))
    y = region(y, (rows, C))
    bound = (C / 32 + 8) * 2.0 ** -24 * m * 1.01 * w.double().abs() + TOL_F32 * ref.abs().max()
    assert ((y.double() - ref).abs() <= bound).all()


# ------------------------------------------------------------------------------------------------ depthwise 3x3 + GELU, 7x7
def dw3_case(p):
    B, H, W, C = p["B"], p["H"], p["W"], p["C"]
    g = gen(("dw3", B, H, W, C))
    x = guarded(rn(g, B, H, W, C))
    w, bias = guarded(rn(g, 9, C, scale=0.3)), guarded(rn(g, C, scale=0.1))
    n = B * H * W * C

    def run(fp32, split):
        y = out_buf(n) if fp32 else None
        hi, lo = (out_buf(n, torch.bfloat16), out_buf(n, torch.bfloat16)) if split else (None, None)
        ok(L().pf_op_dwconv3x3_gelu_ex(ptr(x), B, H, W, C, ptr(w), ptr(bias), ptr(y), ptr(hi), ptr(lo), U.stream_ptr()))
        return y, hi, lo
    y, hi, lo = twice(lambda: run(True, True))
    y, hi, lo = (region(t, (B, H, W, C)) for t in (y, hi, lo))
    err = rel(y, gelu64(dw_ref(x, w, bias, 3)))
    assert err < TOL_F32, err
    check_split(y, hi, lo)
    _, hs, ls = twice(lambda: run(False, True))                 # the graph's form: the planes only
    assert torch.equal(bits(region(hs, (B, H, W, C))), bits(hi)) and torch.equal(bits(region(ls, (B, H, W, C))), bits(lo))
    yf, _, _ = twice(lambda: run(True, False))                  # fp32 only (pf_op_dwconv3x3_gelu's form)
    assert torch.equal(bits(region(yf, (B, H, W, C))), bits(y))


def dw7_case(p):
    B, H, W, C = p["B"], p["H"], p["W"], p["C"]
    g = gen(("dw7", B, H, W, C))
    x = guarded(rn(g, B, H, W, C))
    w, bias = guarded(rn(g, 49, C, scale=0.2)), guarded(rn(g, C, scale=0.1))

    def run():
        y = out_buf(B * H * W * C)
        ok(L().pf_op_dwconv7x7(ptr(x), ptr(y), B, H, W, C, ptr(w), ptr(bias), U.stream_ptr()))
        return (y,)
    y, = twice(run)
    err = rel(region(y, (B, H, W, C)), dw_ref(x, w, bias, 7))
    assert err < TOL_F32, err


# ------------------------------------------------------------------------------------------------ x2 bilinear upsample
def up_case(p, form):
    B, H, W, C, ldi, icoff, ldo, ocoff = (p[k] for k in ("B", "H", "W", "C", "ldi", "icoff", "ldo", "ocoff"))
    g = gen(("up", B, H, W, C, ldi, icoff, ldo, ocoff))
    x = guarded(rn(g, B, H, W, ldi))
    shape, chans = (B, 2 * H, 2 * W, ldo), (ocoff, ocoff + C)
    n = math.prod(shape)

    def run(fp32, split):
        y = out_buf(n) if fp32 else None
        hi, lo = (out_buf(n, torch.bfloat16), out_buf(n, torch.bfloat16)) if split else (None, None)
        ok(L().pf_op_upsample2x_ex(ptr(x), ldi, icoff, ptr(y), ldo, ocoff, ptr(hi), ptr(lo), B, H, W, C, U.stream_ptr()))
        return y, hi, lo
    y, hi, lo = twice(lambda: run(True, True))
    y, hi, lo = (region(t, shape, chans) for t in (y, hi, lo))
    ref = F.interpolate(x[..., icoff:icoff + C].permute(0, 3, 1, 2).double(), scale_factor=2, mode="bilinear", align_corners=False)
    err = rel(y, ref.permute(0, 2, 3, 1))
    assert err < TOL_UP, err
    check_split(y.contiguous(), hi.contiguous(), lo.contiguous())
    yo, ho, lo_ = twice(lambda: run(form == "fp32", form == "split"))     # the graph's form alone
    for a, want in ((yo, y), (ho, hi), (lo_, lo)):
        if a is not None:
            assert torch.equal(bits(region(a, shape, chans)), bits(want))


# ------------------------------------------------------------------------------------------------ stem patch gather
def stem_gather_case(p):
    B, IH, IW, stride = p["B"], p["IH"], p["IW"], p["stride"]
    OH, OW = (IH - 1) // stride + 1, (IW - 1) // stride + 1
    g = gen(("gather", B, IH, IW, stride))
    x0 = rn(g, B, IH, IW, 4)
    x0[..., 3] = float("nan")                    # the fourth channel of the normalised input is never read
    x0 = guarded(x0)
    M = B * OH * OW

    def run():
        hi, lo = out_buf(M * 160, torch.bfloat16), out_buf(M * 160, torch.bfloat16)
        ok(L().pf_op_stem_gather(ptr(x0), B, IH, IW, stride, ptr(hi), ptr(lo), U.stream_ptr()))
        return hi, lo
    hi, lo = twice(run)
    hi, lo = region(hi, (M, 160)), region(lo, (M, 160))
    # unfold gives columns (c, ky, kx); the engine's K order is (ky, kx, c), padded 147 -> 160 with zeros
    cols = F.unfold(x0[..., :3].permute(0, 3, 1, 2), 7, padding=3, stride=stride)
    v = F.pad(cols.view(B, 3, 49, OH * OW).permute(0, 3, 2, 1).reshape(M, 147), (0, 13))
    check_split(v, hi, lo)
    assert (bits(hi[:, 147:]) == 0).all() and (bits(lo[:, 147:]) == 0).all()


# ------------------------------------------------------------------------------------------------ ParamNet stem, field packing
def pn_stem_case(p):
    B, SH, SW = p["B"], p["SH"], p["SW"]
    g = gen(("stem", B, SH, SW))
    pin = rn(g, B, SH, SW, 4)
    pin[..., 3] = float("nan")                   # the packed input's fourth channel is never read
    pin = guarded(pin)
    wt = rn(g, 96, 3, 4, 4, scale=0.2)
    w, bias = guarded(wt.permute(2, 3, 1, 0).reshape(48, 96)), guarded(rn(g, 96, scale=0.1))
    shape = (B, SH // 4, SW // 4, 96)

    def run():
        out = out_buf(math.prod(shape))
        ok(L().pf_op_pn_stem(ptr(pin), B, SH, SW, ptr(w), ptr(bias), ptr(out), U.stream_ptr()))
        return (out,)
    out, = twice(run)
    ref = F.conv2d(pin[..., :3].permute(0, 3, 1, 2).double(), wt.double(), bias.double(), stride=4).permute(0, 2, 3, 1)
    err = rel(region(out, shape), ref)
    assert err < TOL_F32, err


def pack_case(p):
    B, IH, IW, OH, OW = p["B"], p["IH"], p["IW"], p["OH"], p["OW"]
    g = gen(("pack", B, IH, IW, OH, OW))
    grav, lat = guarded(rn(g, B, 2, IH, IW)), guarded(rn(g, B, 1, IH, IW))

    def run():
        out = out_buf(B * OH * OW * 4)
        ok(L().pf_op_pack_fields(ptr(grav), ptr(lat), B, IH, IW, OH, OW, ptr(out), U.stream_ptr()))
        return (out,)
    out, = twice(run)
    out = region(out, (B, OH, OW, 4))
    # ATen's nearest resize in fp32 on the device: src = min(floor(dst * (float)in / out), in - 1)
    want = F.interpolate(torch.cat((grav, lat), 1), (OH, OW), mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(bits(out[..., :3].contiguous()), bits(want.contiguous()))
    assert (bits(out[..., 3]) == 0).all()


# ------------------------------------------------------------------------------------------------ ParamNet tail
def tail_scaling(raw, kind, gvfov):
    """param_network.py's scaling of the raw outputs in float64 ([n, 5] -> [n, 8]) and f^2 of the closed form (kind 2).
    gvfov: the general vfov in degrees the focal length is solved from (the kernel solves it from the fp32 x2 * 90)."""
    x = raw.double()
    p = torch.zeros(x.shape[0], 8, dtype=torch.float64, device=x.device)
    p[:, 0], p[:, 1], p[:, 2], p[:, 6] = x[:, 0] * 90, x[:, 1] * 90, x[:, 2] * 90, x[:, 2]
    if kind == PF_PARAM_CENTERED:
        p[:, 5] = 0.5 / torch.tan(x[:, 2])
        return p, None
    cx, cy = x[:, 3], x[:, 4]
    p[:, 3], p[:, 4] = cx, cy
    c = torch.cos(gvfov.double() * (math.pi / 180.0))
    s2 = 1.0 - c * c
    rt = torch.sqrt(torch.clamp(1.0 - s2 * (1.0 + 4.0 * c * c * cy * cy), min=0.0))
    A = torch.where(c >= 0, 1.0 + rt, 1.0 - rt) / (2.0 * s2)
    f2 = A - cx * cx - cy * cy - 0.25
    p[:, 5] = torch.sqrt(f2)                      # NaN where the equation has no real root
    return p, f2


def check_tail(n, HW, kind):
    g = gen(("tail", n, HW, kind))
    feat = guarded(rn(g, n, HW, 768) + rn(g, n, 1, 768, scale=0.5))
    nw, nb = 1.0 + rn(g, 768, scale=0.1), rn(g, 768, scale=0.1)
    hw, hb = rn(g, 5, 768, scale=0.05), rn(g, 5, scale=0.1)

    def run(with_raw):
        params, raw = out_buf(n * 8), (out_buf(n * 5) if with_raw else None)
        ok(L().pf_op_param_tail(ptr(feat), n, HW, ptr(nw), ptr(nb), ptr(hw), ptr(hb), kind, ptr(params), ptr(raw), U.stream_ptr()))
        return params, raw
    params, raw = twice(lambda: run(True))
    params, raw = region(params, (n, 8), finite=False), region(raw, (n, 5))
    p_noraw, _ = twice(lambda: run(False))
    assert torch.equal(bits(region(p_noraw, (n, 8), finite=False)), bits(params)), "params depend on whether raw is written"
    # pool -> LayerNorm(1e-6) -> Linear in float64
    ln = F.layer_norm(feat.double().mean(1), (768,), nw.double(), nb.double(), eps=1e-6)
    raw_ref = ln @ hw.double().T + hb.double()
    assert rel(raw, raw_ref) < TOL_F32, rel(raw, raw_ref)
    # the scaling, restated in float64 on the kernel's own raw outputs (the kernel scales them in fp32, solves the focal length in
    # float64 from the fp32 vfov): the products by 90 and the copies are exact, tan and the closed form agree to 1e-5 relative
    want, f2 = tail_scaling(raw, kind, raw[:, 2] * 90.0)
    exact = [0, 1, 2, 3, 4, 6, 7]
    assert torch.equal(params[:, exact].double(), want[:, exact].float().double())
    nan = torch.isnan(params[:, 5])
    assert torch.isfinite(params[:, exact]).all()
    assert torch.equal(nan, torch.isnan(want[:, 5]))
    f = ~nan
    if kind == PF_PARAM_UNCENTERED:
        f &= f2.abs() > 1e-6 * (f2.abs() + 1.0)      # away from the root at f^2 = 0, where sqrt amplifies the last bits
    assert ((params[f, 5].double() - want[f, 5]).abs() <= TOL_F32 * want[f, 5].abs()).all()
    if kind == PF_PARAM_UNCENTERED:
        # no real root at the same images as the float64 chain (away from f^2 = 0, where 1e-5 on raw can move the sign)
        _, f2_ref = tail_scaling(raw_ref, kind, (raw_ref[:, 2] * 90.0).float())
        clear = f2_ref.abs() > 1e-3
        assert torch.equal(nan[clear], (f2_ref < 0)[clear])
        return int(nan.sum())
    return 0


@pytest.mark.parametrize("kind", [PF_PARAM_CENTERED, PF_PARAM_UNCENTERED])
@pytest.mark.parametrize("HW", [1, 4, 15, 100, 400])
def test_param_tail(HW, kind):
    nans = check_tail(64, HW, kind)
    if kind == PF_PARAM_UNCENTERED:
        assert 0 < nans < 64          # both branches of the closed form: a real root and none


# ------------------------------------------------------------------------------------------------ prediction tail
def check_pred(B, HW, NC, mode, coff, ld=64, zero=False):
    g = gen(("pred", B, HW, NC, mode, coff, zero))
    feat = rn(g, B * HW, ld)
    w, bias = rn(g, NC, 32, scale=0.3), rn(g, NC, scale=0.1)
    if zero:     # F.normalize's eps branch: an all-zero feature vector and bias give (0, 0)
        feat[::7, coff:coff + 32] = 0.0
        bias.zero_()
    feat = guarded(feat)
    shape = (B, NC, HW)

    def run():
        out = out_buf(math.prod(shape))
        ok(L().pf_op_pred_tail(ptr(feat), ld, coff, ptr(w), ptr(bias), ptr(out), B, HW, NC, mode, U.stream_ptr()))
        return (out,)
    out, = twice(run)
    out = region(out, shape)
    f = feat[:, coff:coff + 32].double()
    v = f @ w.double().T + bias.double()
    if mode == 1:
        # v / |v| amplifies the dot products' error by 1 / |v|: each fp32 fma chain of 32 products and the bias is off by at
        # most 33 * 2^-24 * S (S = the sum of the magnitudes of its terms), which moves the unit vector by at most
        # 2 * 33 * 2^-24 * |S| / |v|; the norm, the square root and the divisions add a few units of 2^-24
        S = (f.abs() @ w.double().abs().T + bias.double().abs()).norm(dim=1, keepdim=True)
        nrm = v.norm(dim=1, keepdim=True)
        v = v / nrm.clamp_min(1e-12)
        bound = (TOL_F32 + 66 * 2.0 ** -24 * S / nrm.clamp_min(1e-30)).view(B, HW, 1).permute(0, 2, 1)
        ref = v.view(B, HW, NC).permute(0, 2, 1)
        assert ((out.double() - ref).abs() <= bound).all()
    else:
        if mode == 2:
            v = v.clamp(-1.0, 1.0)
        ref = v.view(B, HW, NC).permute(0, 2, 1)
        assert rel(out, ref) < TOL_F32, rel(out, ref)
    if zero:
        assert (bits(out.permute(0, 2, 1).reshape(B * HW, NC)[::7]) == 0).all()


def test_pred_tail_zero_vector():
    check_pred(2, 1000, 2, 1, 0, zero=True)


@pytest.mark.parametrize("ld,coff", [(36, 4), (128, 96)])
def test_pred_tail_channel_window(ld, coff):
    # outside the graph (which reads 32 of 64 channels): other pitches and offsets of the 32-channel window
    check_pred(3, 333, 73, 0, coff, ld=ld)


# ------------------------------------------------------------------------------------------------ the sweep
@pytest.mark.parametrize("case", list(SWEEP))
def test_graph_launch(case):
    kernel, form, p = SWEEP[case]
    if kernel == "ln":
        ln_case(p, form)
    elif kernel == "dw3":
        dw3_case(p)
    elif kernel == "dw7":
        dw7_case(p)
    elif kernel == "up":
        up_case(p, form)
    elif kernel == "stem_gather":
        stem_gather_case(p)
    elif kernel == "pn_stem":
        pn_stem_case(p)
    elif kernel == "pack":
        pack_case(p)
    elif kernel == "tail":
        check_tail(p["n"], p["HW"], p["kind"])
    elif kernel == "pred":
        check_pred(p["B"], p["HW"], p["NC"], p["mode"], p["coff"])
    else:
        raise AssertionError(kernel)


# Shapes outside the graph: the upsample on channel windows of wider tensors (the graph reads and writes all 512 channels), both
# forms at once; the 7x7 and 3x3 on grids the graph does not run (1 x W and H x 1 rows, an odd width past one group)
@pytest.mark.parametrize("H,W,C,ldi,icoff,ldo,ocoff", [(5, 7, 256, 512, 256, 384, 64), (3, 2, 64, 64, 0, 128, 64), (1, 1, 4, 12, 8, 8, 4)])
def test_upsample_channel_windows(H, W, C, ldi, icoff, ldo, ocoff):
    up_case(dict(B=2, H=H, W=W, C=C, ldi=ldi, icoff=icoff, ldo=ldo, ocoff=ocoff), "fp32")
    up_case(dict(B=2, H=H, W=W, C=C, ldi=ldi, icoff=icoff, ldo=ldo, ocoff=ocoff), "split")


@pytest.mark.parametrize("H,W", [(1, 9), (9, 1), (2, 5)])
def test_depthwise_thin_grids(H, W):
    dw3_case(dict(B=2, H=H, W=W, C=256))
    dw7_case(dict(B=2, H=H, W=W, C=96))


# ------------------------------------------------------------------------------------------------ rejected arguments
def test_rejected_arguments_launch_nothing():
    t = torch.zeros(1 << 20, device="cuda")
    p, q = t.data_ptr(), t[1:].data_ptr()                        # q: 4-byte aligned only
    h = t.view(torch.bfloat16).data_ptr()
    s = U.stream_ptr()
    big = 1 << 16
    bad = [
        # LayerNorm
        lambda: L().pf_op_layernorm(p, p, 64, 102, p, p, 1e-6, s),                               # C % 4
        lambda: L().pf_op_layernorm(p, p, 64, 772, p, p, 1e-6, s),                               # C > 768
        lambda: L().pf_op_layernorm(p, p, 0, 64, p, p, 1e-6, s),
        lambda: L().pf_op_layernorm(None, p, 64, 64, p, p, 1e-6, s),
        lambda: L().pf_op_layernorm(p, p, 1 << 27, 128, p, p, 1e-6, s),                          # rows C / 4 = 2^32
        lambda: L().pf_op_layernorm_ex(p, None, None, None, None, None, 64, 64, p, p, 1e-6, 0, 0, 0, s),   # no output
        lambda: L().pf_op_layernorm_ex(p, None, h, None, None, None, 64, 64, p, p, 1e-6, 0, 0, 0, s),      # half a pair
        lambda: L().pf_op_layernorm_ex(p, p, None, None, None, None, 64, 64, None, p, 1e-6, 0, 0, 0, s),
        lambda: L().pf_op_layernorm_ex(q, p, None, None, None, None, 64, 64, p, p, 1e-6, 0, 0, 0, s),      # unaligned
        lambda: L().pf_op_layernorm_ex(p, p, None, None, None, None, 64, 64, p, p, 0.0, 0, 0, 0, s),       # eps
        lambda: L().pf_op_layernorm_ex(p, None, None, None, h, h, 64, 64, p, p, 1e-6, 8, 6, 2, s),          # rows != B RH RW
        lambda: L().pf_op_layernorm_ex(p, None, None, None, h, h, 72, 64, p, p, 1e-6, 6, 6, 4, s),          # sr does not divide
        lambda: L().pf_op_layernorm_ex(p, None, None, None, h, h, 64, 64, p, p, 1e-6, 8, 8, 0, s),
        # depthwise 3x3 + GELU
        lambda: L().pf_op_dwconv3x3_gelu(p, p, 1, 4, 4, 6, p, p, s),
        lambda: L().pf_op_dwconv3x3_gelu(p, p, 0, 4, 4, 64, p, p, s),
        lambda: L().pf_op_dwconv3x3_gelu(p, p, 1, 0, 4, 64, p, p, s),
        lambda: L().pf_op_dwconv3x3_gelu(p, None, 1, 4, 4, 64, p, p, s),
        lambda: L().pf_op_dwconv3x3_gelu_ex(p, 1, 4, 4, 64, p, p, None, None, None, s),
        lambda: L().pf_op_dwconv3x3_gelu_ex(p, 1, 4, 4, 64, p, p, None, h, None, s),
        lambda: L().pf_op_dwconv3x3_gelu_ex(q, 1, 4, 4, 64, p, p, p, None, None, s),
        lambda: L().pf_op_dwconv3x3_gelu_ex(p, 1, 4, 4, 64, None, p, p, None, None, s),
        lambda: L().pf_op_dwconv3x3_gelu_ex(p, 64, big, 64, 2048, p, p, p, None, None, s),      # B H W C / 4 = 2^31
        # depthwise 7x7
        lambda: L().pf_op_dwconv7x7(p, p, 1, 4, 4, 6, p, p, s),
        lambda: L().pf_op_dwconv7x7(p, p, 1, 4, 0, 96, p, p, s),
        lambda: L().pf_op_dwconv7x7(p, q, 1, 4, 4, 96, p, p, s),
        lambda: L().pf_op_dwconv7x7(p, p, 1, 4, 4, 96, None, p, s),
        lambda: L().pf_op_dwconv7x7(p, p, 64, big, 64, 2048, p, p, s),
        # upsample
        lambda: L().pf_op_upsample2x(p, p, 1, 4, 4, 6, s),
        lambda: L().pf_op_upsample2x(p, p, 1, 0, 4, 64, s),
        lambda: L().pf_op_upsample2x(None, p, 1, 4, 4, 64, s),
        lambda: L().pf_op_upsample2x_ex(p, 512, 256, p, 512, 0, None, None, 1, 4, 4, 512, s),  # window past ldi
        lambda: L().pf_op_upsample2x_ex(p, 512, 0, p, 512, 2, None, None, 1, 4, 4, 64, s),     # ocoff % 4
        lambda: L().pf_op_upsample2x_ex(p, 64, 0, None, 64, 0, None, None, 1, 4, 4, 64, s),    # no output
        lambda: L().pf_op_upsample2x_ex(p, 64, 0, None, 64, 0, h, None, 1, 4, 4, 64, s),
        lambda: L().pf_op_upsample2x_ex(p, 64, 0, q, 64, 0, None, None, 1, 4, 4, 64, s),
        lambda: L().pf_op_upsample2x_ex(p, 512, 0, p, 512, 0, None, None, 16, 512, 512, 512, s),   # 4 B H W ldo / 4 = 2^31
        # stem gather
        lambda: L().pf_op_stem_gather(p, 1, 64, 64, 3, h, h, s),
        lambda: L().pf_op_stem_gather(p, 0, 64, 64, 2, h, h, s),
        lambda: L().pf_op_stem_gather(p, 1, 64, 64, 2, h, None, s),
        lambda: L().pf_op_stem_gather(None, 1, 64, 64, 2, h, h, s),
        lambda: L().pf_op_stem_gather(p, 1, 64, 64, 2, t[2:].view(torch.bfloat16).data_ptr(), h, s),
        lambda: L().pf_op_stem_gather(p, 128, 4096, 1024, 2, h, h, s),                           # 4 B IH IW = 2^31
        # ParamNet stem, packing, tail
        lambda: L().pf_op_pn_stem(p, 1, 3, 8, p, p, p, s),
        lambda: L().pf_op_pn_stem(p, 0, 8, 8, p, p, p, s),
        lambda: L().pf_op_pn_stem(p, 1, 8, 8, None, p, p, s),
        lambda: L().pf_op_pn_stem(p, 128, 4096, 1024, p, p, p, s),
        lambda: L().pf_op_pack_fields(p, p, 1, 8, 8, 0, 8, p, s),
        lambda: L().pf_op_pack_fields(p, p, 0, 8, 8, 8, 8, p, s),
        lambda: L().pf_op_pack_fields(p, None, 1, 8, 8, 8, 8, p, s),
        lambda: L().pf_op_pack_fields(p, p, 1, 8, 8, 8, 8, q, s),
        lambda: L().pf_op_pack_fields(p, p, 1, big, big, 8, 8, p, s),                            # IH IW = 2^32
        lambda: L().pf_op_param_tail(p, 1, 4, p, p, p, p, 0, p, p, s),
        lambda: L().pf_op_param_tail(p, 1, 4, p, p, p, p, 3, p, p, s),
        lambda: L().pf_op_param_tail(p, 0, 4, p, p, p, p, 1, p, p, s),
        lambda: L().pf_op_param_tail(p, 1, 0, p, p, p, p, 1, p, p, s),
        lambda: L().pf_op_param_tail(p, 1, 4, p, p, p, p, 1, None, p, s),
        lambda: L().pf_op_param_tail(p, 1, 4, p, None, p, p, 1, p, p, s),
        # prediction tail
        lambda: L().pf_op_pred_tail(p, 64, 0, p, p, p, 1, 16, 3, 1, s),                          # normalise needs NC 2
        lambda: L().pf_op_pred_tail(p, 64, 0, p, p, p, 1, 16, 2, 3, s),
        lambda: L().pf_op_pred_tail(p, 64, 0, p, p, p, 1, 16, 257, 0, s),
        lambda: L().pf_op_pred_tail(p, 64, 0, p, p, p, 1, 16, 0, 0, s),
        lambda: L().pf_op_pred_tail(p, 64, 34, p, p, p, 1, 16, 73, 0, s),                        # window past ld
        lambda: L().pf_op_pred_tail(p, 62, 0, p, p, p, 1, 16, 73, 0, s),                         # ld % 4
        lambda: L().pf_op_pred_tail(p, 64, 2, p, p, p, 1, 16, 73, 0, s),                         # coff % 4
        lambda: L().pf_op_pred_tail(q, 64, 0, p, p, p, 1, 16, 73, 0, s),
        lambda: L().pf_op_pred_tail(p, 64, 0, p, None, p, 1, 16, 73, 0, s),
        lambda: L().pf_op_pred_tail(p, 64, 0, p, p, p, 0, 16, 73, 0, s),
        lambda: L().pf_op_pred_tail(p, 64, 0, p, p, p, 2, 1 << 30, 2, 1, s),                     # B HW = 2^31
    ]
    for i, call in enumerate(bad):
        before = launches()
        assert call() == PF_ERR_ARG, i
        assert launches() == before, i
