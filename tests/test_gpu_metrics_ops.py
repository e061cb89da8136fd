"""GPU: the scoring kernels of csrc/metrics.cuh one C-ABI call at a time -- pf_encode_fields (encode_fields_kernel),
pf_head_losses (cross_entropy_kernel or regression_loss_kernel, then loss_finish_kernel) and pf_field_errors
(field_errors_kernel, then field_stats_kernel) -- against the float64 oracle tests/oracle_metrics.py, at the shapes, class
counts and values where the kernels' partitions and arithmetic have edges.  test_gpu_metrics.py covers the same kernels end to
end through the Python API on the golden fixtures.

Bars, each from what the kernel computes:
- median, counts, fractions: exact.  The median is the mean of two float32 order statistics of the map, which float64 adds and
  halves exactly, as np.median does; a fraction is one float64 quotient of two exact counts, as numpy's mean of booleans is.
- mean: 1e-12 relative, against the float64 mean of the GPU's own map.  Every term is >= 0, so a sum's relative error is at
  most its depth times 2^-53: about 40 additions deep on the GPU (16 per thread, a block tree, the strided partials, a block
  tree) and about 30 in numpy's pairwise sum, 8e-15 in all.
- maps: 1e-4 degrees absolute against error_maps.  The kernel evaluates the same float64 formula and rounds once to float32;
  every finite error here stays below 360 degrees, where half a float32 ulp is 1.5e-5.
- losses: 1e-5 relative, the bar of the golden comparisons.  A pixel's term is a few float32 roundings (the cross-entropy's sum
  of C exponentials, its log and one subtraction; the regression's differences, squares and absolute values) that do not
  repeat from pixel to pixel, so the mean's relative error stays near 1e-7 (about 1e-6 for the confident logits, whose small
  loss is closer to the fp32 rounding of their sum of exponentials near 1.0).

Conventions of the *_ops files: every output is filled with a NaN whose payload no kernel produces (-7 for integers) and
followed by spare entries; the owned entries must all be overwritten, finite or NaN exactly where the oracle is, and the spare
entries must keep their bits.  The workspace is NaN-filled before every call, so a partial that no block wrote poisons the
result.  Every call runs twice and the two results must be bit-identical.  Rejected calls launch nothing.

Coverage is asserted, not assumed: the block counts are restated from the kernels' constants and the case lists must reach
field_stats with more than kFeSelThreads error blocks in one image, a regression pass and classification heads with more than
256 blocks (loss_finish's stride), heads with fewer, a ragged last block in every kernel, and class counts below, off and on
multiples of kCeUnroll."""
import ctypes
import math

import numpy as np
import pytest
import torch

import oracle_metrics as om
from perspectivefields_b200 import _native

pytestmark = pytest.mark.gpu

# csrc/metrics.cuh
MET_THREADS, REG_PIX, CE_PIX, CE_UNROLL, FE_TILE, FE_SEL_THREADS, FE_MAX_THR = 256, 16, 4, 8, 16 * 256, 1024, 8
PAD = 67                                                  # spare entries behind every output
POISON32 = 0x7FC0DEAD                                      # quiet NaNs with payloads no kernel writes
POISON64 = 0x7FF80000DEADBEEF
TOL_LOSS, TOL_MEAN, TOL_MAP = 1e-5, 1e-12, 1e-4


def L():
    return _native.lib()


def cdiv(a, b):
    return -(-a // b)


def launches():
    return L().pf_kernel_launch_count()


def stream():
    return torch.cuda.current_stream().cuda_stream


def dev():
    return torch.cuda.current_device()


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


_INT_VIEW = {torch.float32: torch.int32, torch.float64: torch.int64, torch.int64: torch.int64}


def bits(t):
    return t.view(_INT_VIEW[t.dtype])


def out_buf(numel, dtype):
    """numel owned entries filled with the poison (-7 for int64), then PAD spare entries (NaN / -7)"""
    if dtype == torch.int64:
        return torch.full((numel + PAD,), -7, dtype=dtype, device="cuda")
    b = torch.full((numel + PAD,), float("nan"), dtype=dtype, device="cuda")
    bits(b)[:numel] = POISON32 if dtype == torch.float32 else POISON64
    return b


def owned(buf, numel):
    """the owned entries, all overwritten; the spare entries keep their bits"""
    spare = bits(buf[numel:])
    if buf.dtype == torch.int64:
        assert bool((spare == -7).all()), "an entry behind the output was written"
        assert not bool((buf[:numel] == -7).any()), "an owned entry was not written"
    else:
        want = bits(torch.full_like(buf[numel:], float("nan")))
        assert torch.equal(spare, want), "an entry behind the output was written"
        poison = POISON32 if buf.dtype == torch.float32 else POISON64
        assert not bool((bits(buf[:numel]) == poison).any()), "an owned entry was not written"
    return buf[:numel]


def workspace(nbytes):
    assert nbytes > 0
    return torch.full((cdiv(nbytes, 4),), float("nan"), dtype=torch.float32, device="cuda")


def twice(run):
    """run() -> tuple of tensors, twice; the two results must be bit-identical.  Returns the first."""
    a, b = run(), run()
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(bits(x), bits(y)), "two identical calls differ"
    return a


def close(got, want, tol):
    """relative tol; NaN exactly where want is NaN; infinities equal"""
    if math.isnan(want) or math.isinf(want):
        return (math.isnan(got) and math.isnan(want)) or got == want
    return abs(got - want) <= tol * abs(want)


# ------------------------------------------------------------------------------------------------------------ head losses
def head_losses(n, H, W, gc, lc, pg, gg, pl, gl, ig, il, wg, wl):
    need = L().pf_head_losses_workspace(n, H, W, gc, lc)
    k = 4 if gc == 2 else 2

    def run():
        out = out_buf(k, torch.float32)
        ws = workspace(need)
        _native.check(L().pf_head_losses(dev(), n, H, W, gc, pg.data_ptr(), gg.data_ptr(), lc, pl.data_ptr(), gl.data_ptr(), ig, il,
                                         wg, wl, out.data_ptr(), ws.data_ptr(), need, stream()))
        return (owned(out, k),)
    return twice(run)[0].cpu().tolist()


def reg_blocks(n, H, W):
    return cdiv(n * H * W, MET_THREADS * REG_PIX)


def scale_has_pairs(H, W, s):
    """msgil_norm_loss at scale s compares pixels 2 * 2^s apart along a row or a column"""
    return H > 2 << s or W > 2 << s


# (n, H, W, targets): "mixed" unit vectors, tiny and zero vectors and ones with a zero component; "none" no valid gravity pixel
REG_CASES = [
    (1, 1, 1, "mixed"), (1, 2, 3, "mixed"), (1, 7, 9, "mixed"), (2, 5, 37, "mixed"), (1, 37, 53, "mixed"), (3, 24, 40, "mixed"), (2, 53, 37, "mixed"),
    (1, 300, 417, "mixed"), (2, 640, 832, "mixed"), (1, 19, 23, "none"),
]


def reg_inputs(n, H, W, targets, seed):
    g = gen(seed)
    shape = (n, H, W)
    ang = torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) * (2 * math.pi)
    # |t| well above 1e-5 (1, 2.5, 1e-3, 3e-5), well below (2e-6, 1e-7) and 0
    norms = torch.tensor([1.0, 1.0, 1.0, 1.0, 2.5, 1e-3, 3e-5, 2e-6, 1e-7, 0.0], dtype=torch.float64, device="cuda")
    r = norms[torch.randint(0, norms.numel(), shape, generator=g, device="cuda")]
    x, y = torch.cos(ang) * r, torch.sin(ang) * r
    sel = torch.rand(shape, generator=g, device="cuda")
    x = torch.where(sel < 0.05, torch.zeros_like(x), x)                         # a zero x component, |t| = |y| = r
    y = torch.where(sel < 0.05, torch.where(ang < math.pi, r, -r), y)
    y = torch.where((sel >= 0.05) & (sel < 0.1), torch.zeros_like(y), y)      # a zero y component
    x = torch.where((sel >= 0.05) & (sel < 0.1), torch.where(ang < math.pi, r, -r), x)
    tg = torch.stack([x, y], 1).float()
    if targets == "none":
        tg = tg * 1e-6                                                          # every |t| <= 2.5e-6
    pg = (tg + 0.3 * torch.randn((n, 2, H, W), generator=g, device="cuda")).contiguous()
    tl = torch.rand((n, 1, H, W), generator=g, device="cuda") * 2 - 1
    pl = (tl + 0.2 * torch.randn((n, 1, H, W), generator=g, device="cuda")).clamp(-1, 1)
    return pg, tg.contiguous(), pl.contiguous(), tl.contiguous()


def test_regression_cases_cover_the_partitions():
    blocks = [reg_blocks(n, H, W) for n, H, W, _ in REG_CASES]
    assert max(blocks) > MET_THREADS                                               # loss_finish strides over the partials
    assert any(n * H * W % (MET_THREADS * REG_PIX) for n, H, W, _ in REG_CASES)   # a ragged last block
    assert any(b > 1 and n * H * W % (MET_THREADS * REG_PIX) for b, (n, H, W, _) in zip(blocks, REG_CASES))
    assert any(H != W for _, H, W, _ in REG_CASES)
    assert any(not scale_has_pairs(H, W, 0) for _, H, W, _ in REG_CASES)          # no pair at any scale
    assert any(scale_has_pairs(H, W, 1) and not scale_has_pairs(H, W, 3) for _, H, W, _ in REG_CASES)
    assert any(t == "none" for *_, t in REG_CASES)


@pytest.mark.parametrize("n,H,W,targets", REG_CASES, ids=[f"n{n}-{h}x{w}-{t}" for n, h, w, t in REG_CASES])
def test_regression_losses(n, H, W, targets):
    pg, tg, pl, tl = reg_inputs(n, H, W, targets, seed=n * 1000 + H * 7 + W)
    wg, wl = 0.75, 2.5
    got = head_losses(n, H, W, 2, 1, pg, tg, pl, tl, 0, 0, wg, wl)
    want = om.losses(pg, pl, tg, tl, "regression", wg, wl)
    names = ["gravity-msg-normal-loss", "gravity-l2-loss", "latitude-msg-normal-loss", "latitude-l2-loss"]
    for k, name in enumerate(names):
        assert close(got[k], want[name], TOL_LOSS), (name, got[k], want[name])
    valid = float(tg.double().norm(dim=1).gt(1e-5).sum())
    assert math.isnan(got[1]) == (valid == 0)                                   # the gravity L2 mean over no pixel is NaN
    if targets == "none":
        assert valid == 0 and got[0] == 0.0
    if not scale_has_pairs(H, W, 0):
        assert got[0] == 0.0 and got[2] == 0.0                                  # 0 / (0 + 1e-8) at every scale


# (n, H, W, gravity C, latitude C, logits, gravity ignore, latitude ignore, labels)
CLS_CASES = [
    (1, 1, 4, 3, 2, "randn", 72, -1, "plain"),
    (2, 6, 10, 8, 5, "randn", 72, -1, "plain"),
    (3, 37, 12, 9, 16, "scale80", 72, -1, "plain"),
    (1, 64, 64, 73, 180, "randn", 72, -1, "plain"),
    (3, 320, 320, 73, 180, "randn", 72, -1, "plain"),
    (1, 516, 521, 8, 16, "scale80", 72, -1, "plain"),
    (2, 40, 64, 73, 180, "confident", 72, -1, "plain"),
    (1, 48, 48, 9, 16, "confident", 72, -1, "plain"),
    (2, 24, 36, 73, 180, "neginf", 72, -1, "plain"),
    (1, 8, 12, 3, 2, "neginf", 72, -1, "plain"),
    (1, 20, 20, 9, 5, "neginf", 72, -1, "plain"),
    (1, 16, 16, 8, 5, "nan", 72, -1, "plain"),
    (2, 12, 20, 8, 16, "randn", 1, 3, "plain"),
    (1, 12, 20, 73, 180, "randn", 72, -1, "all_ignored"),
    (1, 12, 20, 9, 5, "randn", 72, -1, "out_of_range"),
]
CONF_MAX = 301.3         # the confident pixels' largest logit (the target's)


def ce_blocks(n, H, W):
    return cdiv(n * H * W // CE_PIX, MET_THREADS)


def confident_row(C):
    """float32 [C]: CONF_MAX, then C - 1 logits about ln((C - 1) / (e^0.1 - 1)) below it, so the pixel's loss is about 0.1.
    (At a loss of 0.01 the fp32 sum of exponentials alone would miss the bar: its C - 1 roundings near 1.0 leave a bias of up to
    2e-5 of such a loss.)"""
    rng = np.random.default_rng(C)
    d = math.log((C - 1) / math.expm1(0.1)) + rng.uniform(-0.5, 0.5, C - 1)
    return np.concatenate([[CONF_MAX], CONF_MAX - d]).astype(np.float32)


def confident_loss(C):
    """(float64 loss of confident_row, the loss as (max + log(sum)) - target rounds it in float32)"""
    v = confident_row(C).astype(np.float64)
    lse = math.log(np.exp(v - v[0]).sum())
    m = np.float32(v[0])
    return lse, float(np.float32(m + np.float32(lse)) - m)


def cls_head(g, n, C, HW, kind, ignore, labels):
    shape = (n, C, HW)
    if kind in ("randn", "nan", "neginf"):
        x = 3 * torch.randn(shape, generator=g, device="cuda")
    elif kind == "scale80":
        x = 80 * torch.randn(shape, generator=g, device="cuda")
    if kind == "confident":
        # every pixel holds the same logits in its own order: the exact loss is the same at every pixel, so a rounding of it
        # repeats over the mean, while the order of the fp32 sum of exponentials changes from pixel to pixel
        perm = torch.rand(shape, generator=g, device="cuda").argsort(dim=1)
        x = torch.from_numpy(confident_row(C)).cuda()[perm]
        lab = (perm == 0).int().argmax(dim=1).long()
    else:
        lab = torch.randint(0, C, (n, HW), generator=g, device="cuda")
    if kind == "neginf":
        # -inf in channel 0 (10 % of the pixels) or in channels 0 .. k - 1 for k up to C - 1 (10 %); the target is finite
        u = torch.rand((n, HW), generator=g, device="cuda")
        kk = torch.where(u < 0.1, 1, 0)
        deep = torch.randint(1, C, (n, HW), generator=g, device="cuda")
        kk = torch.where((u >= 0.1) & (u < 0.2), deep, kk)
        x = x.masked_fill(torch.arange(C, device="cuda")[None, :, None] < kk[:, None, :], float("-inf"))
        lab = torch.minimum(kk + (torch.rand((n, HW), generator=g, device="cuda") * (C - kk)).long(), torch.full_like(kk, C - 1))
        assert bool((lab >= kk).all())
    if kind == "nan":
        x[0, C // 2, 3] = float("nan")
    lab = torch.where(torch.rand((n, HW), generator=g, device="cuda") < 0.05, torch.full_like(lab, ignore), lab)
    if kind == "nan":
        lab[0, 3] = 0 if ignore != 0 else 1                                     # the NaN pixel is counted
    if labels == "all_ignored":
        lab = torch.full_like(lab, ignore)
    if labels == "out_of_range":
        lab[0, 5] = C if ignore != C else -5
    return x.contiguous(), lab.contiguous()


def test_classification_cases_cover_the_partitions():
    blocks = [ce_blocks(n, H, W) for n, H, W, *_ in CLS_CASES]
    assert min(blocks) < MET_THREADS and max(blocks) > MET_THREADS
    assert any(b > MET_THREADS and n * H * W % (CE_PIX * MET_THREADS) for b, (n, H, W, *_) in zip(blocks, CLS_CASES))
    assert any(n * H * W % (CE_PIX * MET_THREADS) for n, H, W, *_ in CLS_CASES)
    assert all(H * W % CE_PIX == 0 for _, H, W, *_ in CLS_CASES)
    cs = {c for case in CLS_CASES for c in case[3:5]}
    assert {3, 8, 9, 73} | {2, 5, 16, 180} == cs
    assert any(c < CE_UNROLL for c in cs) and any(c > CE_UNROLL and c % CE_UNROLL for c in cs) and any(c % CE_UNROLL == 0 for c in cs)
    kinds = {case[5] for case in CLS_CASES}
    assert kinds == {"randn", "scale80", "confident", "neginf", "nan"}
    # the confident logits tell the two orders of the final subtraction apart: rounding max + log(sum) at the magnitude of the
    # max is off by more than 5x the bar, for every class count they run at
    for C in {c for case in CLS_CASES if case[5] == "confident" for c in case[3:5]}:
        lse, rounded = confident_loss(C)
        assert 0.05 < lse < 0.15 and abs(rounded - lse) > 5 * TOL_LOSS * lse, (C, lse, rounded)


@pytest.mark.parametrize("n,H,W,gc,lc,kind,ig,il,labels", CLS_CASES,
                         ids=[f"n{c[0]}-{c[1]}x{c[2]}-c{c[3]}-c{c[4]}-{c[5]}-{c[8]}" + (f"-ign{c[6]}" if c[6] != 72 else "") for c in CLS_CASES])
def test_classification_losses(n, H, W, gc, lc, kind, ig, il, labels):
    g = gen(n * 7919 + H * W + gc * 31 + lc)
    pg, gg = cls_head(g, n, gc, H * W, kind, ig, labels)
    pl, gl = cls_head(g, n, lc, H * W, kind, il, labels)
    wg, wl = 0.75, 2.5
    got = head_losses(n, H, W, gc, lc, pg, gg, pl, gl, ig, il, wg, wl)
    shp = lambda t: t.view(n, -1, H, W)
    want = om.losses(shp(pg), shp(pl), gg.view(n, H, W), gl.view(n, H, W), "classification", wg, wl, ig, il)
    for k, name in enumerate(("loss_gravity", "loss_latitude")):
        assert close(got[k], want[name], TOL_LOSS), (name, got[k], want[name])
    nan_expected = kind == "nan" or labels in ("all_ignored", "out_of_range")
    assert all(math.isnan(v) for v in want.values()) == nan_expected
    if kind == "confident":
        assert all(0.05 * w < v < 0.15 * w for v, w in zip(got, (wg, wl)))


def test_head_loss_rejections_launch_nothing():
    Lb = L()
    n, H, W = 1, 8, 8
    pg = torch.zeros(73 * H * W + 16, device="cuda")
    pl = torch.zeros(180 * H * W + 16, device="cuda")
    lab = torch.zeros(H * W, dtype=torch.int64, device="cuda")
    out = torch.zeros(8, device="cuda")
    ws = workspace(1 << 20)

    def call(n, H, W, gc, lc, pgp, plp):
        return Lb.pf_head_losses(dev(), n, H, W, gc, pgp, lab.data_ptr(), lc, plp, lab.data_ptr(), 72, -1, 1.0, 1.0, out.data_ptr(),
                                 ws.data_ptr(), ws.numel() * 4, stream())

    torch.cuda.synchronize()
    before = launches()
    assert call(1, 3, 5, 73, 180, pg.data_ptr(), pl.data_ptr()) < 0                  # H * W % 4 != 0
    assert call(1, 8, 8, 73, 180, pg.data_ptr() + 4, pl.data_ptr()) < 0              # logits not 16-byte aligned
    assert call(1, 8, 8, 73, 180, pg.data_ptr(), pl.data_ptr() + 8) < 0
    assert call(1, 8, 8, 73, 1, pg.data_ptr(), pl.data_ptr()) < 0                    # mixed head kinds
    assert call(1, 8, 8, 2, 180, pg.data_ptr(), pl.data_ptr()) < 0
    assert call(1, 8, 8, 2, 1, None, pl.data_ptr()) < 0
    assert Lb.pf_head_losses_workspace(1, 8, 8, 73, 1) < 0 and Lb.pf_head_losses_workspace(1, 8, 8, 2, 180) < 0
    assert Lb.pf_head_losses_workspace(1, 8, 8, 2, 2) < 0 and Lb.pf_head_losses_workspace(0, 8, 8, 2, 1) < 0
    # H * W >= 2^31 would wrap the pixel count of a plane; the logit-size check alone lets (50000 x 50000, 73 / 180) through
    assert Lb.pf_head_losses_workspace(1, 50000, 50000, 73, 180) < 0
    assert Lb.pf_head_losses_workspace(1, 46341, 46341, 2, 1) < 0
    assert call(1, 50000, 50000, 73, 180, pg.data_ptr(), pl.data_ptr()) < 0
    assert call(1, 46341, 46341, 2, 1, pg.data_ptr(), pl.data_ptr()) < 0
    torch.cuda.synchronize()
    assert launches() == before
    assert Lb.pf_head_losses_workspace(1, 46340, 46340, 2, 1) > 0                    # the largest square plane below 2^31
    assert Lb.pf_head_losses_workspace(2, 46340, 46340, 73, 180) > 0


# ------------------------------------------------------------------------------------------------------------ field errors
class Img:
    """One image of a pf_field_errors call: pu [2, H, W], pl [H, W] degrees, gu [H, W, 2], gl [H, W], mask bool [H, W] or
    None, all numpy float32; the predicted up field is stored [2, H, W] ("chw") or [H, W, 2] ("hwc"), and so is the true one."""

    def __init__(self, pu, pl, gu, gl, mask=None, pred="chw", gt="hwc"):
        self.pu, self.pl, self.gu, self.gl, self.mask, self.pred, self.gt = pu, pl, gu, gl, mask, pred, gt
        self.H, self.W = pl.shape

    @property
    def nblk(self):
        return cdiv(self.H * self.W, FE_TILE)


def random_img(rng, H, W, pred="chw", gt="hwc", mask=False, nonfinite=False):
    ang = rng.uniform(-math.pi, math.pi, (H, W))
    gu = np.stack([np.cos(ang), np.sin(ang)], -1)
    u = rng.random((H, W))
    gu[u < 0.03] = 0.0                                                       # invalid: |g| <= 1e-5
    gu[(u >= 0.03) & (u < 0.05)] = 1e-7
    pu = gu.transpose(2, 0, 1) + 0.2 * rng.standard_normal((2, H, W))
    v = rng.random((H, W))
    pu[:, v < 0.04] = 0.0                                                    # the decoder's "no direction": 180
    pu[:, (v >= 0.04) & (v < 0.06)] = gu.transpose(2, 0, 1)[:, (v >= 0.04) & (v < 0.06)]   # exact: +0
    gl = rng.uniform(-89.0, 89.0, (H, W))
    pl = gl + 3.0 * rng.standard_normal((H, W))
    w = rng.random((H, W))
    pl[w < 0.03] = gl[w < 0.03]
    gl[(w >= 0.03) & (w < 0.05)] = np.nan                                    # invalid latitude
    if nonfinite:
        gu[(u >= 0.05) & (u < 0.06)] = np.nan
        pu[0, v > 0.98] = np.nan                                             # 180
        pl[w > 0.98] = np.inf                                                # +inf
        pl[(w > 0.96) & (w <= 0.98)] = np.nan
    m = rng.random((H, W)) < 0.7 if mask else None
    f = np.float32
    return Img(pu.astype(f), pl.astype(f), gu.astype(f), gl.astype(f), m, pred, gt)


def lat_img(rng, errors, invalid=0, up="random", H=None):
    """An image whose latitude errors are exactly ``errors`` (true latitude 0, prediction the value; inf / nan predictions give
    +inf), followed by ``invalid`` pixels with a NaN true latitude; the up field is random, exact ("exact": error 0) or
    "none" (every prediction the zero vector: 180)."""
    vals = np.asarray(errors, np.float32).reshape(-1)
    k = vals.size + invalid
    H = H or 1
    W = k // H
    assert H * W == k
    gl = np.zeros(k, np.float32)
    gl[vals.size:] = np.nan
    pl = np.zeros(k, np.float32)
    pl[:vals.size] = vals
    img = random_img(rng, H, W)
    gu = img.gu.reshape(-1, 2)
    gu[:] = np.stack([np.cos(np.arange(k)), np.sin(np.arange(k))], -1)
    pu = img.pu.reshape(2, -1)
    if up == "exact":
        pu[:] = gu.T
    elif up == "none":
        pu[:] = 0.0
    return Img(img.pu, pl.reshape(H, W), img.gu, gl.reshape(H, W), None, img.pred, img.gt)


INF = float("inf")
ULP = (np.float32(1.0).view(np.uint32) + np.arange(601, dtype=np.uint32)).view(np.float32)   # 1.0f + k ulp, k = 0 .. 600


def constructed_imgs(rng):
    """(name, image) pairs whose latitude maps meet the radix select's edges"""
    c = [
        ("count0", lat_img(rng, [], invalid=12, H=3, up="none")),
        ("count1", lat_img(rng, [2.75])),
        ("count1of6", lat_img(rng, [-4.5], invalid=5, H=2)),
        ("count2", lat_img(rng, [7.0, 2.5])),
        ("equal", lat_img(rng, [3.25] * 50, H=5, up="none")),
        ("aab", lat_img(rng, [1.5, -1.5, 4.0])),                        # odd count: the middle is a
        ("aaab", lat_img(rng, [4.0, 1.5, 1.5, -1.5])),                  # lower middle a, not the last of its equals
        ("aabb", lat_img(rng, [4.0, 1.5, 4.0, 1.5])),                   # lower middle the last a: the next value is b
        ("aaabcc", lat_img(rng, [6.0, 1.5, 1.5, 4.0, 1.5, 6.0])),
        ("a_inf", lat_img(rng, [INF, 2.0])),                            # the next value is +inf
        ("aa_inf_nan", lat_img(rng, [2.0, INF, 2.0, float("nan")])),    # a NaN prediction also counts +inf
        ("inf_majority", lat_img(rng, [INF, 1.0, INF])),
        ("exact", lat_img(rng, [0.0] * 7 + [5.0], up="exact")),
        ("ulp601", lat_img(rng, rng.permutation(ULP))),
        ("ulp600", lat_img(rng, rng.permutation(ULP[:600]), invalid=2, H=2)),
        ("ulp256", lat_img(rng, rng.permutation(ULP[:256]), H=16)),     # one top three bytes: the last digit decides
        ("thresholds", lat_img(rng, [5.0] * 10 + [4.0] * 3 + [6.0] * 2 + [10.0] * 4 + [180.0, 45.0], invalid=3, H=4)),
    ]
    return c


THR8 = (-INF, 0.0, 1.0, 5.0, 10.0, 45.0, 180.0, INF)


def pack(imgs, lat_scale=1.0):
    """device blobs and descriptors of one call; the images lie one after the other with a 3-element gap"""
    n = len(imgs)
    descs = (_native.pf_field_image * n)()
    pu, pl, gu, gl, mk = [], [], [], [], []
    o = {"pu": 0, "pl": 0, "gu": 0, "gl": 0, "mk": 0}
    gap = np.full(3, 7.0, np.float32)

    def put(lst, key, a):
        off = o[key]
        lst.append(a.reshape(-1))
        lst.append(gap if key != "mk" else np.ones(3, np.uint8))
        o[key] += a.size + 3
        return off

    for d, im in zip(descs, imgs):
        H, W = im.H, im.W
        d.height, d.width = H, W
        if im.pred == "chw":
            d.pred_up_offset, d.pred_up_stride[:] = put(pu, "pu", im.pu), (W, 1, H * W)
        else:
            d.pred_up_offset, d.pred_up_stride[:] = put(pu, "pu", im.pu.transpose(1, 2, 0)), (2 * W, 2, 1)
        d.pred_lat_offset = put(pl, "pl", im.pl)
        if im.gt == "hwc":
            d.gt_up_offset, d.gt_up_stride[:] = put(gu, "gu", im.gu), (2 * W, 2, 1)
        else:
            d.gt_up_offset, d.gt_up_stride[:] = put(gu, "gu", im.gu.transpose(2, 0, 1)), (W, 1, H * W)
        d.gt_lat_offset = put(gl, "gl", (im.gl.astype(np.float64) * lat_scale).astype(np.float32))
        d.mask_offset = put(mk, "mk", im.mask.astype(np.uint8)) if im.mask is not None else -1
    cu = lambda lst, dt=np.float32: torch.from_numpy(np.concatenate(lst).astype(dt)).cuda()
    return descs, cu(pu), cu(pl), cu(gu), cu(gl), (cu(mk, np.uint8) if mk else None)


def field_errors(imgs, thresholds, lat_rad=0, with_maps=True):
    """One pf_field_errors call (twice).  Returns (count [2, n], mean, median [2, n], fraction [2, n, T] or None, maps [2, P]
    or None) on the CPU."""
    n, T = len(imgs), len(thresholds)
    descs, pu, pl, gu, gl, mk = pack(imgs, (math.pi / 180.0) if lat_rad else 1.0)
    P = sum(im.H * im.W for im in imgs)
    need = L().pf_field_errors_workspace(descs, n, int(with_maps))
    th = (ctypes.c_double * max(T, 1))(*thresholds)

    def run():
        maps = out_buf(2 * P, torch.float32) if with_maps else None
        count, mean, median = out_buf(2 * n, torch.int64), out_buf(2 * n, torch.float64), out_buf(2 * n, torch.float64)
        frac = out_buf(2 * n * T, torch.float64) if T else None
        ws = workspace(need)
        _native.check(L().pf_field_errors(dev(), descs, n, pu.data_ptr(), pl.data_ptr(), gu.data_ptr(), gl.data_ptr(),
                                          mk.data_ptr() if mk is not None else None, lat_rad, th if T else None, T,
                                          maps.data_ptr() if with_maps else None, maps[P:].data_ptr() if with_maps else None,
                                          count.data_ptr(), mean.data_ptr(), median.data_ptr(), frac.data_ptr() if T else None,
                                          ws.data_ptr(), need, stream()))
        return (owned(count, 2 * n).view(2, n), owned(mean, 2 * n).view(2, n), owned(median, 2 * n).view(2, n),
                owned(frac, 2 * n * T).view(2, n, T) if T else None, owned(maps, 2 * P).view(2, P) if with_maps else None)
    return tuple(None if t is None else t.cpu() for t in twice(run))


def check_field_errors(imgs, thresholds, res, lat_mode="deg"):
    count, mean, median, frac, maps = res
    T = len(thresholds)
    p = 0
    for i, im in enumerate(imgs):
        hw = im.H * im.W
        gl = im.gl.astype(np.float64) * (math.pi / 180.0) if lat_mode == "rad" else im.gl
        if lat_mode == "rad":
            gl = gl.astype(np.float32)
        want = om.error_maps(im.pu, im.pl, im.gu, gl, lat_mode, im.mask)
        for f in range(2):
            mp = maps[f, p:p + hw].double().numpy().reshape(im.H, im.W)
            o = want[f]
            assert np.array_equal(np.isnan(mp), np.isnan(o)), (i, f)
            assert np.array_equal(np.isinf(mp), np.isinf(o)) and np.array_equal(mp[np.isinf(o)], o[np.isinf(o)]), (i, f)
            fin = np.isfinite(o)
            assert np.all(np.abs(mp[fin] - o[fin]) <= TOL_MAP), (i, f, float(np.abs(mp[fin] - o[fin]).max()))
            c, mn, med, fr = om.stats(mp, thresholds)
            assert int(count[f, i]) == c, (i, f)
            got_mean, got_med = float(mean[f, i]), float(median[f, i])
            got_fr = frac[f, i].tolist() if T else []
            if c == 0:
                assert math.isnan(got_mean) and math.isnan(got_med) and all(math.isnan(x) for x in got_fr), (i, f)
                continue
            assert got_med == med, (i, f, got_med, med)
            assert got_fr == fr, (i, f, got_fr, fr)
            assert close(got_mean, mn, TOL_MEAN), (i, f, got_mean, mn)
        p += hw


@pytest.fixture(scope="module")
def many_images():
    """the images of one call: 1 x 1, exactly one tile, one tile and a row, a few hundred small images of mixed sizes (the
    block-to-image search), both up-field layouts on both sides, masks (one of them empty), non-finite predictions, the
    constructed latitude maps, and one 2048 x 2100 image (1050 error blocks)"""
    rng = np.random.default_rng(20261019)
    imgs, names = [], []

    def add(name, im):
        names.append(name)
        imgs.append(im)

    add("1x1", random_img(rng, 1, 1))
    add("64x64", random_img(rng, 64, 64, pred="hwc"))
    add("64x65", random_img(rng, 64, 65, gt="chw", mask=True))
    for k in range(300):
        H, W = int(rng.integers(1, 41)), int(rng.integers(1, 41))
        add(f"small{k}", random_img(rng, H, W, pred=("chw", "hwc")[k % 2], gt=("hwc", "chw")[(k // 2) % 2], mask=k % 3 == 0,
                                    nonfinite=k % 7 == 0))
    add("masked_out", random_img(rng, 30, 17, mask=True))
    imgs[-1].mask[:] = False
    add("97x131", random_img(rng, 97, 131, pred="hwc", mask=True, nonfinite=True))
    for name, im in constructed_imgs(rng):
        add(name, im)
    add("2048x2100", random_img(rng, 2048, 2100))
    add("5x3", random_img(rng, 5, 3))
    return names, imgs


def test_field_error_cases_cover_the_partitions(many_images):
    names, imgs = many_images
    nblk = [im.nblk for im in imgs]
    assert max(nblk) > FE_SEL_THREADS                                           # field_stats strides over an image's partials
    assert any(im.H * im.W == FE_TILE for im in imgs)
    assert any(b > 1 and im.H * im.W % FE_TILE for b, im in zip(nblk, imgs))    # a ragged last block after a full one
    assert sum(b == 1 and im.H * im.W < FE_TILE for b, im in zip(nblk, imgs)) >= 300
    assert {im.pred for im in imgs} == {"chw", "hwc"} and {im.gt for im in imgs} == {"chw", "hwc"}
    assert any(im.mask is not None for im in imgs) and any(im.mask is None for im in imgs)
    assert any(im.mask is not None and not im.mask.any() for im in imgs)
    counts = {int(np.isfinite(im.gl).sum()) for im in imgs if im.mask is None}
    assert {0, 1, 2} <= counts
    assert len(set((ULP[:256].view(np.uint32) >> 8).tolist())) == 1            # the ulp256 map shares its top three bytes
    assert len(set((ULP.view(np.uint32) >> 8).tolist())) == 3                  # the ulp601 map does not


def test_field_errors_many_images(many_images):
    _, imgs = many_images
    res = field_errors(imgs, THR8)
    check_field_errors(imgs, THR8, res)
    # without maps, the maps live in the workspace: the statistics keep their bits
    plain = field_errors(imgs, THR8, with_maps=False)
    for a, b in zip(res[:4], plain[:4]):
        assert torch.equal(bits(a), bits(b))
    assert plain[4] is None


def test_field_errors_constructed_medians(many_images):
    """the constructed maps' statistics, stated by hand (the oracle's np.median agrees, test_field_errors_many_images)"""
    names, imgs = many_images
    sel = [i for i, nm in enumerate(names) if not nm.startswith(("small", "2048", "97x", "64x", "1x1", "5x3", "masked"))]
    sub = [imgs[i] for i in sel]
    count, mean, median, frac, _ = field_errors(sub, THR8)
    got = {names[i]: (int(count[1, k]), float(mean[1, k]), float(median[1, k]), frac[1, k].tolist()) for k, i in enumerate(sel)}
    mid = lambda a, b: (float(a) + float(b)) * 0.5
    want_median = {"count1": 2.75, "count1of6": 4.5, "count2": mid(2.5, 7.0), "equal": 3.25, "aab": 1.5, "aaab": 1.5,
                   "aabb": mid(1.5, 4.0), "aaabcc": mid(1.5, 4.0), "a_inf": INF, "aa_inf_nan": INF, "inf_majority": INF,
                   "exact": 0.0, "ulp601": float(ULP[300]), "ulp600": mid(ULP[299], ULP[300]), "ulp256": mid(ULP[127], ULP[128]),
                   "thresholds": 5.0}
    for name, med in want_median.items():
        assert got[name][2] == med, (name, got[name][2], med)
    assert got["count0"][0] == 0 and math.isnan(got["count0"][1]) and math.isnan(got["count0"][2])
    assert all(math.isnan(x) for x in got["count0"][3])
    assert got["inf_majority"][1] == INF and got["a_inf"][1] == INF
    assert int(count[0, sel.index(names.index("equal"))]) == 50 and float(median[0, sel.index(names.index("equal"))]) == 180.0
    k = sel.index(names.index("exact"))
    assert float(median[0, k]) == 0.0 and float(mean[0, k]) == 0.0 and float(median[1, k]) == 0.0
    assert frac[0, k].tolist() == [0.0, 0.0] + [1.0] * 6                         # exact errors are +0: not below 0
    # strict comparisons: errors of exactly 5 are not below 5, nor 180 below 180, nor +inf below +inf; -inf counts nothing
    c, _, _, fr = got["thresholds"]
    assert c == 21 and fr == [0.0, 0.0, 0.0, 3 / 21, 15 / 21, 19 / 21, 20 / 21, 1.0]
    assert got["a_inf"][3] == [0.0, 0.0, 0.0, 1 / 2, 1 / 2, 1 / 2, 1 / 2, 1 / 2]


def test_field_errors_radians_and_masks(many_images):
    names, imgs = many_images
    sub = [im for nm, im in zip(names, imgs) if nm.startswith(("small", "64x", "masked"))]
    res = field_errors(sub, (), lat_rad=1)
    assert res[3] is None
    check_field_errors(sub, (), res, lat_mode="rad")
    res = field_errors(sub[:40], (2.0,), lat_rad=1)
    check_field_errors(sub[:40], (2.0,), res, lat_mode="rad")


def test_field_error_rejections_launch_nothing():
    Lb = L()
    rng = np.random.default_rng(3)
    imgs = [random_img(rng, 4, 5), random_img(rng, 3, 3)]
    descs, pu, pl, gu, gl, _ = pack(imgs)
    need = Lb.pf_field_errors_workspace(descs, 2, 1)
    ws = workspace(need)
    outs = torch.zeros(64, dtype=torch.float64, device="cuda")
    maps = torch.zeros(64, device="cuda")

    def call(thr, T, lat_rad=0, up_maps=maps.data_ptr(), lat_maps=maps[32:].data_ptr(), nbytes=need, d=descs):
        th = (ctypes.c_double * max(len(thr), 1))(*thr)
        return Lb.pf_field_errors(dev(), d, 2, pu.data_ptr(), pl.data_ptr(), gu.data_ptr(), gl.data_ptr(), None, lat_rad, th, T,
                                  up_maps, lat_maps, outs.data_ptr(), outs[4:].data_ptr(), outs[8:].data_ptr(), outs[12:].data_ptr(),
                                  ws.data_ptr(), nbytes, stream())

    torch.cuda.synchronize()
    before = launches()
    assert call((1.0,) * 9, 9) < 0                                              # more than 8 thresholds
    assert call((1.0, float("nan")), 2) < 0                                     # a NaN threshold
    assert call((1.0,), -1) < 0
    assert call((1.0,), 1, lat_rad=2) < 0
    assert call((1.0,), 1, lat_maps=None) < 0                                   # one map without the other
    assert call((1.0,), 1, nbytes=need - 1) < 0
    bad = (_native.pf_field_image * 2)(descs[0], descs[1])
    bad[1].height = 0
    assert call((1.0,), 1, d=bad) < 0
    assert Lb.pf_field_errors_workspace(bad, 2, 1) < 0
    bad[1].height, bad[1].width = 46341, 46341                                  # H * W >= 2^31
    assert Lb.pf_field_errors_workspace(bad, 2, 1) < 0
    torch.cuda.synchronize()
    assert launches() == before


# ------------------------------------------------------------------------------------------------------------ encoders
ENC_CASES = [("chw", 3, 2, 0), ("hwc", 3, 2, 1), ("chw", 8, 5, 1), ("hwc", 8, 5, 0), ("chw", 2, 1, 0), ("hwc", 2, 1, 1)]


@pytest.mark.parametrize("layout,gc,lc,lat_rad", ENC_CASES, ids=[f"{a}-c{b}-c{c}-rad{d}" for a, b, c, d in ENC_CASES])
def test_encode_fields(layout, gc, lc, lat_rad):
    n, H, W = 2, 5, 37                                                         # 370 pixels: a ragged second block
    assert n * H * W % MET_THREADS and n * H * W > MET_THREADS
    rng = np.random.default_rng(gc * 10 + lc)
    ang = rng.uniform(-math.pi, math.pi, (n, H, W))
    up = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)          # [n, H, W, 2]
    up[0, 0, :4] = [(0.0, 0.0), (1.0, 0.0), (-1.0, 0.0), (0.0, -1.0)]
    up[1, 2, 5:9] = 0.0
    deg = rng.uniform(-90.0, 90.0, (n, H, W)).astype(np.float32)
    bnd = om.latitude_boundaries(max(lc, 2))
    deg[0, 1, :bnd.size] = bnd[:W]                                             # on the class boundaries
    deg[1, 0, :4] = [0.0, -0.0, -90.0, 90.0]
    if lc > 1:
        deg[1, 4, 0] = np.nan                                                 # the last class, as in torch.bucketize
    lat = (deg.astype(np.float64) * (math.pi / 180)).astype(np.float32) if lat_rad else deg
    if layout == "chw":
        ub = torch.from_numpy(up.transpose(0, 3, 1, 2).copy()).cuda()
        us = (2 * H * W, W, 1, H * W)
    else:
        ub = torch.from_numpy(up.copy()).cuda()
        us = (2 * H * W, 2 * W, 2, 1)
    lb = torch.from_numpy(lat.copy()).cuda()
    i64x4 = ctypes.c_int64 * 4
    ng = n * 2 * H * W if gc == 2 else n * H * W
    nl = n * H * W
    gdt = torch.float32 if gc == 2 else torch.int64
    ldt = torch.float32 if lc == 1 else torch.int64

    def run():
        og, ol = out_buf(ng, gdt), out_buf(nl, ldt)
        _native.check(L().pf_encode_fields(dev(), n, H, W, ub.data_ptr(), i64x4(*us), lb.data_ptr(), i64x4(H * W, W, 1, 0), lat_rad,
                                           gc, lc, og.data_ptr(), ol.data_ptr(), stream()))
        return owned(og, ng), owned(ol, nl)
    gg, gl = (t.cpu() for t in twice(run))
    if gc == 2:
        assert torch.equal(bits(gg.view(n, 2, H, W)), bits(torch.from_numpy(up.transpose(0, 3, 1, 2).copy())))
    else:
        want = torch.stack([om.encode_bin(torch.from_numpy(u.transpose(2, 0, 1).copy()), gc) for u in up])
        q = ((np.degrees(np.arctan2(up[..., 1].astype(np.float64), up[..., 0])) + 180.0) % 360.0) / (360.0 / (gc - 1))
        near = np.abs(q % 1.0 - 0.5) < 1e-4
        off = (gg.view(n, H, W) != want).numpy()
        assert not (off & ~near).any()
        assert gg.min() >= 0 and gg.max() <= gc - 1
    if lc == 1:
        want = torch.sin(torch.from_numpy(deg).double() * (math.pi / 180) if not lat_rad else torch.from_numpy(lat).double()).float()
        assert float((gl.view(n, H, W) - want).abs().max()) <= 6e-8
    else:
        d = deg if not lat_rad else lat * np.float32(180 / math.pi)
        assert torch.equal(gl.view(n, H, W), torch.stack([om.encode_bin_latitude(x, lc) for x in d]))
