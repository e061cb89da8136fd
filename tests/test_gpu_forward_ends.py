"""GPU: the launches at the two ends of every pf_forward, as the graph runs them, against Pillow and float64 restatements.

The counterpart of ``test_gpu_forward_ops.py`` / ``test_gpu_forward_tc_ops.py`` for ``preprocess_kernel``,
``normalize_chw_kernel``, the three decode kernels, ``postprocess_kernel`` and ``conf_resample_kernel``.  Everything runs through
``pf_forward`` / ``pf_forward_confidence`` on the engine of a ``PerspectiveFields`` model, with this file's own input blob (image
offsets that are not multiples of 4 or 16) and NaN-filled output blobs with gaps between the images and after the last one.

A. Pre-process.  ``x0`` (debug tap ``"pre"``) is the uint8 resize of ``oracle/pillow_resize.py`` (Pillow's arithmetic, horizontal pass
   first) normalised in fp32, bit for bit.  (Pillow itself takes the vertical pass first for some of the very tall images here,
   which moves single pixels by one level.)  A block of 8 output
   rows stages the input rows it needs in shared memory; when they exceed the launch's row budget (``min(pre_rows_needed(tallest
   image), 200 KB / (3 NW))``: 1066 rows at NW = 64, 213 at 320, 106 at 640) it makes several passes.  ``passes()`` restates
   that split, and the batches reach 2, 3 and 8 passes per block, the tallest accepted image at each working size and mixed
   batches (tall among small, up- and down-sampled, 1 x 1 and 1 x N, wider than 4 NW).  One image taller is rejected before
   any launch.

B. Resize-table slab.  One launch reads all tables of its batch: a reset of the 8 MB slab happens before the first fetch and
   never inside the descriptor loop (``pf_resize_table_stats``); batches that cross the boundary come back Pillow-exact.

C. Head decode.  Logits are recomputed in float64 from the same forward's ``head.conv1`` tap; argmax, decode and max-softmax
   in float64.  Batch sizes put ``pred_argmax_decode_kernel``'s grid-stride loop (4224 blocks = 270,336 pixels per pass) at
   less than one, exactly one and 2.73 passes.

D. Post-process and confidence resample, restated in float64 on the engine's own working-size fields and confidence maps,
   with the sampling positions ``fma(y + 0.5, sch, -0.5)`` rounded to fp32 as the kernels compute them (one FFMA).

Bars (u = 2^-24, the fp32 unit roundoff; every bar is per pixel and derived from the operations involved):
  * up (post-process): each blended component takes 7 roundings (scale by W/SW, two products and a sum per axis, and the fp32
    1 - l weight), so |e_c| <= 7 u M_c, M_c the largest |tap| of that component after scaling.  Normalising adds rsqrtf's
    2^-22 relative and two products (2u): bar = 7 u (M_x + M_y) / |blend| + 2^-22 + 3u.  Pixels where this exceeds the
    existing 2e-5 (a blend near zero length) are not judged; at least 99% are.
  * latitude in degrees (classification): 7 u M (M = largest |tap|, <= 90): at most 3.8e-5 deg, against the 1e-3 deg bar.
  * latitude from sin (regression): the blend's 7 u M in the sine domain, fast_asinf's 1.7e-7 rad, the product by 180/pi (u):
    bar = (7 u M / sqrt(1 - s^2) + 1.7e-7) * 180/pi + u |deg| + ulp(90)/2 where |s| <= 0.99; nearer the poles, where asin
    amplifies, the comparison is in the sine domain: |sin(got) - s| <= 7 u M + 1.7e-7 + 6.7e-8 (got's own rounding).
    Taps at exactly +-1 give exactly +-90.
  * confidence resample: 7 u M.
  * decode: fp32 logits carry |e| <= 34 u S, S = sum |w x| + |b| of the 1x1 conv; pixels whose top-2 margin is below
    max(1e-4, 4 e) are not judged.  Argmax up: 2e-6 (fp32 angle, cos, sin); argmax latitude: exact (-90 + c + 1/2).  Sub-bin:
    delta = (a - b) / (2 (a + b)) moves by at most 2 e / (a + b) + 4u, times 5 deg (up) or 1 deg (latitude), plus the argmax bar
    and the roundings of p = c + delta and the sums after it (SUBBIN_ROUNDING: 7.3e-7 rad up, 1.5e-5 deg latitude).
    Confidence: relative 2e-5 (the fp32 online sum over up to 180 classes: 180 * 2u = 2.1e-5) plus 2 e.
"""
import collections
import ctypes
import functools
import gc
import math

import numpy as np
import pytest
import torch

import pf_test_util as U
from perspectivefields_b200 import _native
from oracle.pillow_resize import resize_bilinear_u8
from perspectivefields_b200.variants import PIXEL_MEAN, PIXEL_STD

pytestmark = pytest.mark.gpu

REG, CLS = "Paramnet-360Cities-edina-centered", "PersNet-360Cities"
MEAN, STD = np.array(PIXEL_MEAN, np.float32), np.array(PIXEL_STD, np.float32)
U32 = 2.0 ** -24
PRE_ROWS, SMEM = 8, 200 * 1024
SLAB = 8 << 20
EW_PIXELS = 132 * 32 * 256 // 4           # pixels per grid-stride pass of pred_argmax_decode_kernel (4 threads per pixel)
WORKING = [(64, 640), (640, 64), (320, 320), (320, 640), (640, 384)]

# ------------------------------------------------------------------------------------------------ restatements
def ksize(in_size, out_size):
    """make_resample_table's coefficients per output pixel"""
    return int(math.ceil(max(in_size / out_size, 1.0))) * 2 + 1


def table_bytes(in_size, out_size):
    """get_table's slab bytes: bounds and coefficients, each rounded up to 256 bytes"""
    r = lambda b: (b + 255) // 256 * 256
    return r(2 * out_size * 4) + r(out_size * ksize(in_size, out_size) * 4)


def max_rows(NW):
    return SMEM // (3 * NW)


def rows_needed(H, NH):
    s = H / NH
    return int(PRE_ROWS * s) + 2 * int(math.ceil(max(s, 1.0))) + 3


def tallest(NH, NW):
    """the tallest image the pre-process accepts at this working size: ksize + 1 <= max_rows"""
    c = (max_rows(NW) - 2) // 2
    return c * NH


def bounds(in_size, out_size):
    """Pillow's (xmin, xmax) per output pixel"""
    scale = in_size / out_size
    support = max(scale, 1.0)
    center = (np.arange(out_size) + 0.5) * scale
    lo = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    hi = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64)
    return lo, hi


@functools.lru_cache(maxsize=None)
def passes(H, NH, budget):
    """largest number of shared-memory passes any block of preprocess_kernel makes for an image of H rows"""
    lo, hi = bounds(H, NH)
    worst = 0
    for oy0 in range(0, NH, PRE_ROWS):
        r0, n = 0, 0
        while r0 < PRE_ROWS:
            first, rc = lo[oy0 + r0], 0
            while r0 + rc < PRE_ROWS:
                if hi[oy0 + r0 + rc] - first > budget and rc > 0:
                    break
                rc += 1
            r0 += rc
            n += 1
        worst = max(worst, n)
    return worst


def batch_budget(heights, NH, NW):
    return min(rows_needed(max(heights), NH), max_rows(NW))


def height_with_passes(NH, NW, want):
    """a height whose blocks need exactly `want` passes (at most) in a batch whose row budget is max_rows(NW)"""
    budget = max_rows(NW)
    for c in range(1, tallest(NH, NW) // NH + 1):
        for H in (c * NH - 7, c * NH + 3):
            if passes(H, NH, budget) == want:
                return H
    raise AssertionError((NH, NW, want))


def pillow_x0(img, NH, NW):
    r = resize_bilinear_u8(img, NH, NW)
    return (r.astype(np.float32) - MEAN) / STD


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def positions(out, src):
    """(i0, i1, l) of the bilinear sample of each of `out` output pixels from `src` source pixels: ATen's rule with the position
    fma(y + 0.5, (float)src / (float)out, -0.5) rounded once to fp32, as the kernels' FFMA computes it"""
    sc = np.float32(src) / np.float32(out)
    y = np.arange(out, dtype=np.float32) + np.float32(0.5)
    s = np.maximum(f32(y.astype(np.float64) * np.float64(sc) - 0.5), np.float32(0)).astype(np.float64)
    i0 = np.minimum(s.astype(np.int64), src - 1)
    return i0, i0 + (i0 < src - 1), s - i0


def resample64(v, H, W):
    """[C, SH, SW] float64 -> [C, H, W] bilinear blend (vertical then horizontal, as postprocess_kernel nests it), and the
    largest |tap| per pixel"""
    _, SH, SW = v.shape
    y0, y1, ly = positions(H, SH)
    x0, x1, lx = positions(W, SW)
    ly, lx = ly[None, :, None], lx[None, None, :]
    a, b = v[:, y0][:, :, x0], v[:, y0][:, :, x1]
    c, d = v[:, y1][:, :, x0], v[:, y1][:, :, x1]
    out = (1 - lx) * ((1 - ly) * a + ly * c) + lx * ((1 - ly) * b + ly * d)
    m = np.maximum(np.maximum(np.abs(a), np.abs(b)), np.maximum(np.abs(c), np.abs(d)))
    return out, m


# ------------------------------------------------------------------------------------------------ models and the forward
_models = {}


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """The cached models hold weights, workspaces and (in debug mode) every intermediate of their last forward, tens of GB in
    all: free them and their engines when this file's tests are done, so that later test modules get the device memory back."""
    yield
    _models.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def model(version, NH, NW, debug=True):
    key = (version, NH, NW)
    if key not in _models:
        _models[key] = U.make_model(version, seed=1, model_kwargs={"resize": (NH, NW)})[0]
        _models[key]._debug = None
    m = _models[key]
    if m._debug != debug:
        m.debug_taps(debug)
        m._debug = debug
    return m


def fresh_engine(NH, NW):
    """the cached model with a new engine handle: an empty resize-table slab"""
    m = model(REG, NH, NW)
    m._drop_engine()
    m.debug_taps(True)
    return m


def images(sizes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]


def pack(parts, pads):
    """concatenate uint8 images with pads[i] bytes before image i -> (device blob, offsets)"""
    offs, total = [], 0
    for p, im in zip(pads, parts):
        total += p
        offs.append(total)
        total += im.size
    blob = np.zeros(total + 7, np.uint8)
    for o, im in zip(offs, parts):
        blob[o:o + im.size] = im.reshape(-1)
    return torch.from_numpy(blob).cuda(), np.array(offs, np.int64)


def out_offsets(sizes, per_pixel, misalign=()):
    """offsets (floats) of each image's block in an output blob, with a gap before every image: the gap realigns the block to
    4 floats unless the image is listed in `misalign`, where it keeps the offset of a tightly packed predecessor + 4"""
    offs, end = [], 0
    for i, (h, w) in enumerate(sizes):
        start = end + 4 if i in misalign else end + 1 + (-(end + 1)) % 4
        offs.append(start)
        end = start + per_pixel * h * w
    return np.array(offs, np.int64), end + 5


def tap(m, name):
    eng = m._get_engine()
    L = eng.L
    n = L.pf_debug_numel(eng.handle, name.encode())
    assert n > 0, name
    t = torch.empty(n, dtype=torch.float32, device="cuda")
    _native.check(L.pf_debug_copy(eng.handle, name.encode(), t.data_ptr(), n, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return t


def table_stats(m):
    eng = m._get_engine()
    b, r = ctypes.c_int64(), ctypes.c_int64()
    _native.check(eng.L.pf_resize_table_stats(eng.handle, ctypes.byref(b), ctypes.byref(r)))
    return b.value, r.value


def forward(m, imgs, pads=None, conf=False, chw=None, misalign=()):
    """one pf_forward (pf_forward_confidence with conf) on this file's blobs -> dict of outputs and layout"""
    eng = m._get_engine()
    NH, NW = m.net_size()
    sizes = [im.shape[:2] for im in imgs]
    n = len(sizes)
    h = np.array([s[0] for s in sizes], np.int32)
    w = np.array([s[1] for s in sizes], np.int32)
    g_off, g_len = out_offsets(sizes, 2, misalign)
    l_off, l_len = out_offsets(sizes, 1, misalign)
    nanf = lambda *s: torch.full(s, float("nan"), device="cuda")
    gc, lc = (2, 1) if eng.decode_only else (eng.gravity_classes, eng.latitude_classes)
    out = {"pred_gravity": nanf(n, gc, NH, NW), "pred_latitude": nanf(n, lc, NH, NW), "gravity_original": nanf(g_len),
           "latitude_original": nanf(l_len), "params": nanf(n, 8), "g_off": g_off, "l_off": l_off, "sizes": sizes}
    bt = _native.pf_batch()
    bt.n = n
    i64p, i32p = ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int32)
    if chw is None:
        blob, offsets = pack(imgs, pads or [0] * n)
        out["blob"] = blob
        bt.images_u8, bt.image_offset = blob.data_ptr(), offsets.ctypes.data_as(i64p)
    else:
        bt.images_chw = chw.data_ptr()
    bt.height, bt.width = h.ctypes.data_as(i32p), w.ctypes.data_as(i32p)
    bt.pred_gravity, bt.pred_latitude = out["pred_gravity"].data_ptr(), out["pred_latitude"].data_ptr()
    bt.gravity_original, bt.gravity_original_offset = out["gravity_original"].data_ptr(), g_off.ctypes.data_as(i64p)
    bt.latitude_original, bt.latitude_original_offset = out["latitude_original"].data_ptr(), l_off.ctypes.data_as(i64p)
    bt.params = out["params"].data_ptr()
    cur = torch.cuda.current_stream()
    ws = eng._workspace(_native.check(eng.L.pf_workspace_bytes(eng.handle, n, int(h.max()))), cur)
    if conf:
        for k in ("gravity", "latitude"):
            out[k + "_confidence"] = nanf(n, NH, NW)
            out[k + "_confidence_original"] = nanf(l_len)
        cf = _native.pf_confidence(out["gravity_confidence"].data_ptr(), out["latitude_confidence"].data_ptr(),
                                   out["gravity_confidence_original"].data_ptr(), out["latitude_confidence_original"].data_ptr())
        _native.check(eng.L.pf_forward_confidence(eng.handle, ctypes.byref(bt), ctypes.byref(cf), ws.data_ptr(), ws.numel(), cur.cuda_stream))
    else:
        _native.check(eng.L.pf_forward(eng.handle, ctypes.byref(bt), ws.data_ptr(), ws.numel(), cur.cuda_stream))
    torch.cuda.synchronize()
    return out


def check_x0(m, imgs, label=""):
    NH, NW = m.net_size()
    x0 = tap(m, "pre").view(len(imgs), NH, NW, 4).cpu().numpy()
    for i, im in enumerate(imgs):
        assert np.array_equal(x0[i, ..., :3], pillow_x0(im, NH, NW)), (label, i, im.shape)
        assert (x0[i, ..., 3] == 0).all()
    return x0


def gaps_untouched(blob, offs, sizes, per_pixel):
    """every float outside the images' blocks still holds the fill's NaN bit pattern"""
    mask = torch.ones(blob.numel(), dtype=torch.bool, device=blob.device)
    for o, (h, w) in zip(offs, sizes):
        mask[int(o):int(o) + per_pixel * h * w] = False
    nan_bits = torch.full((1,), float("nan"), device=blob.device).view(torch.int32)
    assert mask.sum() > 0
    assert bool((blob.view(torch.int32)[mask] == nan_bits).all())


# ------------------------------------------------------------------------------------------------ A. pre-process
def pre_batches(NH, NW):
    """(label, sizes, pads) of the pre-process batches at one working size"""
    T = tallest(NH, NW)
    out = [
        ("split 2/3/8 passes + tallest", [(height_with_passes(NH, NW, 2), 5), (3, 7), (height_with_passes(NH, NW, 3), 3), (T, 2),
                                          (height_with_passes(NH, NW, 8), 1)], [0, 1, 3, 5, 2]),
        ("tall among small, up/down-sampled, 1x1, 1xN, wide", [(1, 1), (NH // 2 + 1, NW // 3 + 2), (T - 5, 3), (1, 37), (2 * NH + 9, 4 * NW + 3),
                                                              (37, 1), (NH, NW)], [3, 1, 6, 0, 13, 2, 17]),
    ]
    return out


@pytest.mark.parametrize("NH,NW", WORKING)
def test_preprocess_batches_are_pillow_exact(NH, NW):
    m = model(REG if (NH + NW) % 3 else CLS, NH, NW)
    for label, sizes, pads in pre_batches(NH, NW):
        imgs = images(sizes, NH * 7 + NW + len(label))
        forward(m, imgs, pads)
        x0 = check_x0(m, imgs, label)
        forward(m, imgs, pads)
        assert np.array_equal(tap(m, "pre").view(x0.shape).cpu().numpy().view(np.uint32), x0.view(np.uint32)), label   # run twice


@pytest.mark.parametrize("NH,NW", WORKING)
def test_next_taller_image_is_rejected_before_any_launch(NH, NW):
    m = model(REG if (NH + NW) % 3 else CLS, NH, NW)
    T = tallest(NH, NW)
    assert ksize(T, NH) + 1 <= max_rows(NW) < ksize(T + 1, NH) + 1
    if NW in (64, 640):
        assert ksize(T, NH) + 1 == max_rows(NW)       # the edge itself is reachable at these widths (ksize is odd)
    imgs = images([(8, 8), (T + 1, 2)], 3)
    before = _native.lib().pf_kernel_launch_count()
    with pytest.raises(_native.PfError, match="too tall"):
        forward(m, imgs)
    assert _native.lib().pf_kernel_launch_count() == before


@pytest.mark.parametrize("NH,NW", [(320, 320), (64, 640)])
def test_chw_input_is_normalised_bit_for_bit(NH, NW):
    m = model(CLS if (NH + NW) % 3 == 0 else REG, NH, NW)
    g = torch.Generator().manual_seed(NH + NW)
    chw = (torch.rand(3, 3, NH, NW, generator=g) * 255).round()
    chw[0, :, 0, :5] = torch.tensor([0.0, 255.0, 0.5, -3.0, 300.25])
    forward(m, [np.zeros((NH + 1, NW + 2, 3), np.uint8)] * 3, chw=chw.cuda().contiguous())
    x0 = tap(m, "pre").view(3, NH, NW, 4).cpu().numpy()
    want = (chw.permute(0, 2, 3, 1).numpy() - MEAN) / STD
    assert np.array_equal(x0[..., :3].view(np.uint32), want.astype(np.float32).view(np.uint32))
    assert (x0[..., 3] == 0).all()


# ------------------------------------------------------------------------------------------------ B. resize-table slab
SLAB_NH, SLAB_NW = 640, 64


def slab_heights(start, count, step=1):
    return [start + step * i for i in range(count)]


def first_reset(used, cached, sizes):
    """(image, axis) at which the descriptor loop's sequential fetches (W table, then H table, per image) would overflow a slab
    holding `used` bytes and the tables `cached`: where a reset inside the loop would have made the earlier tables stale"""
    cached, off = set(cached), used
    for i, (h, w) in enumerate(sizes):
        for axis, key in (("W", (w, SLAB_NW)), ("H", (h, SLAB_NH))):
            if key in cached:
                continue
            if off + table_bytes(*key) > SLAB:
                return i, axis
            cached.add(key)
            off += table_bytes(*key)
    return None


def keys(sizes):
    return {(w, SLAB_NW) for _, w in sizes} | {(h, SLAB_NH) for h, _ in sizes}


def test_table_slab_crosses_between_images():
    """The slab holds 4 H tables of a ~200,000-row image (1.6 MB each) from a first batch; the second batch's three new heights
    fit the rest only up to its image k = 1: the reset comes once, before the batch's first fetch."""
    m = fresh_engine(SLAB_NH, SLAB_NW)
    b0, r0 = table_stats(m)
    assert (b0, r0) == (0, 0)
    first = [(h, 2) for h in slab_heights(200_000, 4)]
    forward(m, images(first, 1))
    used = table_bytes(2, SLAB_NW) + sum(table_bytes(h, SLAB_NH) for h, _ in first)
    assert table_stats(m) == (used, 0)
    second = [(h, 2) for h in slab_heights(200_100, 3)]
    assert first_reset(used, keys(first), second) == (1, "H")      # image 1, whose W table is cached
    imgs = images(second, 2)
    forward(m, imgs)
    want = table_bytes(2, SLAB_NW) + sum(table_bytes(h, SLAB_NH) for h, _ in second)
    assert table_stats(m) == (want, 1)                # one reset, and every table of the batch was fetched after it
    check_x0(m, imgs, "after reset")
    forward(m, imgs)                                   # the same batch again: all tables cached, still exact
    assert table_stats(m) == (want, 1)
    check_x0(m, imgs, "cached")


def test_table_slab_crosses_between_w_and_h_tables():
    """The boundary falls between one image's W table and its H table."""
    m = fresh_engine(SLAB_NH, SLAB_NW)
    second = [(9, 5), (5_000, 7)]
    # four ~1.5 MB H tables and a filler height chosen so that image 1's W table fits the rest of the slab and its H table does not
    big = [(h, 3) for h in slab_heights(190_000, 4)]
    first = next(big + [(hf, 3)] for hf in range(640, tallest(SLAB_NH, SLAB_NW), 640) if first_reset(sum(table_bytes(*k) for k in keys(big + [(hf, 3)])),
                                                                                 keys(big + [(hf, 3)]), second) == (1, "H"))
    forward(m, images(first, 3))
    used = sum(table_bytes(*k) for k in keys(first))
    assert table_stats(m) == (used, 0)
    imgs = images(second, 4)
    forward(m, imgs, pads=[1, 3])
    want = sum(table_bytes(*k) for k in keys(second))
    assert table_stats(m) == (want, 1)
    check_x0(m, imgs, "W/H boundary")


def test_batch_larger_than_the_slab_is_rejected():
    m = fresh_engine(SLAB_NH, SLAB_NW)
    sizes = [(h, 2) for h in slab_heights(200_000, 6)]
    assert sum(table_bytes(h, SLAB_NH) for h, _ in sizes) > SLAB
    before = _native.lib().pf_kernel_launch_count()
    with pytest.raises(_native.PfError, match="split the batch"):
        forward(m, images(sizes, 5))
    assert _native.lib().pf_kernel_launch_count() == before
    assert table_stats(m) == (0, 0)
    ok = images(sizes[:5], 6)                          # five of them fit
    forward(m, ok)
    check_x0(m, ok, "five")


# ------------------------------------------------------------------------------------------------ C. head decode
DECODE_CASES = [(320, 320, 1), (192, 352, 4), (640, 384, 3)]      # < 1, exactly 1 and 2.73 passes of the fused decode


# fp32 roundings the sub-bin decode adds to the argmax decode's: p = c + delta (half an ulp of the largest bin index), and for the
# latitude the two sums -90 + p w + w / 2 (half an ulp of 90 each); for the up head p * 5 (360 u deg), in radians
SUBBIN_ROUNDING = {True: (np.spacing(np.float32(72)) / 2 * 5 + 360 * U32) * math.pi / 180,
                   False: np.spacing(np.float32(179)) / 2 + np.spacing(np.float32(90))}


def decode_passes(NH, NW, n):
    return n * NH * NW / EW_PIXELS


def decode64(logits, is_gravity, refine):
    """float64 argmax (+ sub-bin) decode of [n, NC, P] logits -> field [n, C, P], (a + b) per pixel (inf where not refined)"""
    NC = logits.shape[1]
    c = logits.argmax(1)
    take = lambda i: logits.gather(1, i.unsqueeze(1)).squeeze(1)
    if is_gravity:
        refined = c < NC - 1
        lo, hi = torch.where(refined, (c - 1) % (NC - 1), c), torch.where(refined, (c + 1) % (NC - 1), c)
    else:
        refined = (c > 0) & (c < NC - 1)
        lo, hi = (c - 1).clamp_min(0), (c + 1).clamp_max(NC - 1)
    a, b = take(c) - take(lo), take(c) - take(hi)
    s = torch.where(refined, a + b, torch.full_like(a, math.inf))
    d = torch.where(refined & (s > 0) & torch.isfinite(s), (a - b) / (2 * s), torch.zeros_like(a)) if refine else torch.zeros_like(a)
    p = c.double() + d
    if is_gravity:
        ang = (p * (360.0 / (NC - 1)) - 180.0) / 180.0 * math.pi
        f = torch.stack([torch.cos(ang), torch.sin(ang)], 1)
        f = torch.where((c == NC - 1).unsqueeze(1), torch.zeros_like(f), f)
    else:
        f = (-90.0 + p * (180.0 / NC) + 90.0 / NC).unsqueeze(1)
    return f, s


@pytest.mark.parametrize("NH,NW,n", DECODE_CASES)
def test_head_decode_as_the_graph_launches_it(NH, NW, n):
    m = model(CLS, NH, NW)
    eng = m._get_engine()
    imgs = images([(NH + 13 * i, NW - 7 * i) for i in range(n)], n + NH)
    P = NH * NW
    sd = {k: eng.tensors[k].double() for k in ("head.pred_g.w", "head.pred_g.b", "head.pred_l.w", "head.pred_l.b")}
    worst = collections.defaultdict(float)
    fields = {}
    for decode_only in (0, 1):
        for refine in (0, 1):
            for conf in (False, True):
                m.set_option("decode_only", decode_only)
                m.set_option("subbin", refine)
                out = forward(m, imgs, conf=conf)
                feat = tap(m, "head.conv1").view(n, P, 64).double()
                for head, k, coff, is_g in (("gravity", "g", 0, True), ("latitude", "l", 32, False)):
                    x = feat[:, :, coff:coff + 32]
                    w, b = sd[f"head.pred_{k}.w"], sd[f"head.pred_{k}.b"]
                    logits = (x @ w.t() + b).permute(0, 2, 1)                       # [n, NC, P]
                    err = 34 * U32 * ((x.abs() @ w.abs().t()) + b.abs()).permute(0, 2, 1).amax(1)    # fp32 logit error bound
                    top2 = logits.topk(2, dim=1).values
                    stable = (top2[:, 0] - top2[:, 1]) > torch.clamp(4 * err, min=1e-4)
                    want, s = decode64(logits, is_g, refine)
                    if not decode_only:        # the returned fp32 logits (pred_tail_kernel) within their bound
                        el = (out["pred_" + head].view(n, -1, P).double() - logits).abs()
                        assert bool((el <= err.unsqueeze(1)).all()), (head, el.max().item())
                    else:
                        got = out["pred_" + head].view(n, -1, P).double()
                        base = (2e-6 if is_g else 0.0) + (SUBBIN_ROUNDING[is_g] if refine else 0.0)
                        bar = base + (((2 * err / s) + 4 * U32) * (5.0 * math.pi / 180 if is_g else 1.0) if refine else 0 * err)
                        e = (got - want).abs().amax(1)
                        assert stable.float().mean() > 0.99
                        assert bool((e[stable] <= bar[stable]).all()), (head, decode_only, refine, conf, e[stable].max().item())
                        worst[f"{head} field"] = max(worst[f"{head} field"], e[stable].max().item())
                    fields[(head, decode_only, refine, conf)] = (out["pred_" + head] if decode_only else out[f"{head}_original"]).clone()
                    if conf:
                        cw = 1.0 / torch.exp(logits - logits.amax(1, keepdim=True)).sum(1)
                        gc = out[f"{head}_confidence"].view(n, P).double()
                        rel = (gc / cw - 1).abs()
                        cbar = 2e-5 + 2 * err
                        assert bool((rel <= cbar).all()), (head, rel.max().item())
                        worst[f"{head} conf"] = max(worst[f"{head} conf"], rel.max().item())
                        fields[(head + "_conf", decode_only, refine)] = out[f"{head}_confidence"].clone()
                fields[("orig", decode_only, refine, conf)] = (out["gravity_original"].clone(), out["latitude_original"].clone())
    m.set_option("decode_only", 0)
    m.set_option("subbin", 0)
    # the decode_only and logits paths: bit-identical resampled fields and confidence on the same features
    for refine in (0, 1):
        for conf in (False, True):
            for a, b in zip(fields[("orig", 0, refine, conf)], fields[("orig", 1, refine, conf)]):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (refine, conf)
        for head in ("gravity", "latitude"):
            assert torch.equal(fields[(head + "_conf", 0, refine)].view(torch.int32), fields[(head + "_conf", 1, refine)].view(torch.int32))
    print(f"decode {NH}x{NW} n={n} ({decode_passes(NH, NW, n):.3f} passes): max errors {dict(worst)}")


# ------------------------------------------------------------------------------------------------ D. post-process
def post_sizes(NH, NW):
    """(sizes, indices of images whose blocks are misaligned by an earlier odd-area image)"""
    sizes = [(3, 7),                         # odd area: the next image's blocks start misaligned
             (37, 3076),                     # W % 4 == 0, no table (Wp > 3072), misaligned -> scalar stores
             (5, 3072), (19, 3073),          # table / no table
             (33, 1020), (16, 1024), (21, 1028),    # W4 = 255, 256, 257
             (1, 1021),                      # H = 1, W % 4 != 0
             (NH // 16, NW // 16), (NH * 16, 9), (17, NW * 16),      # 16x smaller / larger targets
             (50, 64)]
    return sizes, {1}


def post_edges(sizes, misalign):
    """the postprocess_kernel paths the batch reaches (restated from the kernel)"""
    edges = set()
    for i, (h, w) in enumerate(sizes):
        W4 = (w + 3) // 4
        edges.add("table" if W4 * 4 <= 3072 else "no table")
        edges.add("W4<256" if W4 < 256 else "W4=256" if W4 == 256 else "W4>256")
        edges |= {"W%4" if w % 4 else "vec" if i not in misalign else "W%4=0 misaligned"}
        if h % 16:
            edges.add("ragged band")
        if h % 4:
            edges.add("ragged group")
        if h == 1:
            edges.add("H=1")
    return edges


def check_post(NH, NW, out, imgs, fields, lat_is_sin, conf=None):
    """compare gravity / latitude originals (and confidence originals) with the float64 restatement; returns worst errors"""
    worst = collections.defaultdict(float)
    judged = [0, 0]
    for i, im in enumerate(imgs):
        H, W = im.shape[:2]
        vec = fields[0][i].double().cpu().numpy()
        lat = fields[1][i].double().cpu().numpy()
        sc = np.array([np.float32(W / NW), np.float32(H / NH)], np.float64).reshape(2, 1, 1)
        blend, M = resample64(vec * sc, H, W)
        nrm = np.sqrt((blend ** 2).sum(0))
        want = blend / np.maximum(nrm, 1e-12)
        g = out["gravity_original"][int(out["g_off"][i]):int(out["g_off"][i]) + 2 * H * W].view(2, H, W).double().cpu().numpy()
        bar = 7 * U32 * M.sum(0) / np.maximum(nrm, 1e-300) + 2.0 ** -22 + 3 * U32
        ok = bar <= 2e-5
        judged[0] += int(ok.sum()); judged[1] += ok.size
        e = np.abs(g - want).max(0)
        assert (e[ok] <= bar[ok]).all(), (i, H, W, e[ok].max())
        worst["up"] = max(worst["up"], float(e[ok].max(initial=0)))
        lb, lm = resample64(lat[None], H, W)
        lb, lm = lb[0], lm[0]
        l = out["latitude_original"][int(out["l_off"][i]):int(out["l_off"][i]) + H * W].view(H, W).double().cpu().numpy()
        if lat_is_sin:
            s = np.clip(lb, -1, 1)
            pole = np.abs(s) > 0.99
            deg = np.degrees(np.arcsin(s))
            dbar = (7 * U32 * lm / np.sqrt(np.maximum(1 - s * s, 1e-300)) + 1.7e-7) * 180 / math.pi + U32 * np.abs(deg) + 3.9e-6
            el = np.abs(l - deg)
            assert (el[~pole] <= dbar[~pole]).all(), (i, el[~pole].max())
            es = np.abs(np.sin(np.radians(l)) - lb)
            sbar = 7 * U32 * lm + 1.7e-7 + 6.7e-8
            assert (es[pole] <= sbar[pole]).all(), (i, es[pole].max())
            worst["lat deg"] = max(worst["lat deg"], float(el[~pole].max(initial=0)))
            worst["lat sin (poles)"] = max(worst["lat sin (poles)"], float(es[pole].max(initial=0)))
            y0, y1, _ = positions(H, NH)
            x0, x1, _ = positions(W, NW)
            taps = np.stack([lat[y0][:, x0], lat[y0][:, x1], lat[y1][:, x0], lat[y1][:, x1]])
            for sgn in (1, -1):
                at = (taps == sgn).all(0)
                assert (l[at] == 90.0 * sgn).all(), (i, sgn)
                worst[f"taps {sgn:+d}"] += int(at.sum())
        else:
            el = np.abs(l - lb)
            assert (el <= 7 * U32 * lm).all(), (i, el.max())
            worst["lat deg"] = max(worst["lat deg"], float(el.max()))
        if conf is not None:
            for k, src in zip(("gravity", "latitude"), conf):
                cb, cm = resample64(src[i].double().cpu().numpy()[None], H, W)
                o = out[k + "_confidence_original"][int(out["l_off"][i]):int(out["l_off"][i]) + H * W].view(H, W).double().cpu().numpy()
                ec = np.abs(o - cb[0])
                assert (ec <= 7 * U32 * cm[0]).all(), (k, i, ec.max())
                worst["conf"] = max(worst["conf"], float(ec.max()))
    assert judged[0] >= 0.99 * judged[1], judged
    gaps_untouched(out["gravity_original"], out["g_off"], [im.shape[:2] for im in imgs], 2)
    gaps_untouched(out["latitude_original"], out["l_off"], [im.shape[:2] for im in imgs], 1)
    for k in ("gravity", "latitude"):
        if k + "_confidence_original" in out:
            gaps_untouched(out[k + "_confidence_original"], out["l_off"], [im.shape[:2] for im in imgs], 1)
    return worst


@pytest.mark.parametrize("variant", [REG, CLS])
@pytest.mark.parametrize("NH,NW", [(320, 320), (320, 640)])
def test_postprocess_as_the_graph_launches_it(variant, NH, NW):
    m = model(variant, NH, NW, debug=False)
    sizes, mis = post_sizes(NH, NW)
    imgs = images(sizes, NH + NW)
    pads = [(5 * i + 3) % 17 for i in range(len(sizes))]
    if variant == CLS:
        m.set_option("decode_only", 1)
    try:
        out = forward(m, imgs, pads, conf=variant == CLS, misalign=mis)
    finally:
        m.set_option("decode_only", 0) if variant == CLS else None
    assert int(out["g_off"][1]) % 4 and int(out["l_off"][1]) % 4          # image 1 (W % 4 == 0) starts misaligned
    conf = (out["gravity_confidence"], out["latitude_confidence"]) if variant == CLS else None
    worst = check_post(NH, NW, out, imgs, (out["pred_gravity"], out["pred_latitude"][:, 0]), variant == REG, conf)
    print(f"post-process {variant} {NH}x{NW}: max errors {dict(worst)}")


def test_postprocess_at_the_poles():
    """lat_is_sin with taps at exactly +-1 and values next to them, through the same host helper (pf_op_postprocess_sized)."""
    NH, NW = 64, 640
    sizes, mis = post_sizes(NH, NW)
    g = torch.Generator().manual_seed(9)
    n = len(sizes)
    vec = torch.nn.functional.normalize(torch.randn(n, 2, 5, 7, generator=g) + torch.tensor([0.5, -1.0]).view(1, 2, 1, 1), dim=1)
    vec = torch.nn.functional.interpolate(vec, size=(NH, NW), mode="bicubic", align_corners=False).contiguous()
    lat = torch.sign(torch.randn(n, 1, NH, NW, generator=g)) * (1 - (torch.rand(n, 1, NH, NW, generator=g) < 0.3).float() * 1e-3)
    lat[:, :, :, : NW // 2] = 1.0
    lat[:, :, NH // 2:, NW // 2:] = -1.0
    lat[:, :, 3:7] = torch.rand(n, 1, 4, NW, generator=g) * 2 - 1
    imgs = [np.zeros((h, w, 1), np.uint8) for h, w in sizes]
    h = np.array([s[0] for s in sizes], np.int32)
    w = np.array([s[1] for s in sizes], np.int32)
    g_off, g_len = out_offsets(sizes, 2, mis)
    l_off, l_len = out_offsets(sizes, 1, mis)
    out = {"gravity_original": torch.full((g_len,), float("nan"), device="cuda"), "latitude_original": torch.full((l_len,), float("nan"), device="cuda"),
           "g_off": g_off, "l_off": l_off}
    i32p, i64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    vd, ld = vec.cuda(), lat.cuda().contiguous()
    _native.check(_native.lib().pf_op_postprocess_sized(vd.data_ptr(), ld.data_ptr(), n, NH, NW, h.ctypes.data_as(i32p), w.ctypes.data_as(i32p),
                                                        out["gravity_original"].data_ptr(), g_off.ctypes.data_as(i64p), out["latitude_original"].data_ptr(),
                                                        l_off.ctypes.data_as(i64p), 1, U.stream_ptr()))
    torch.cuda.synchronize()
    worst = check_post(NH, NW, out, imgs, (vd, ld[:, 0]), True)
    assert worst["taps +1"] > 0 and worst["taps -1"] > 0
    print(f"post-process at the poles: max errors {dict(worst)}")


# ------------------------------------------------------------------------------------------------ E. the restatement is the graph
def restated_launches(variant, u8, decode_only, conf):
    c = collections.Counter({"preprocess_kernel" if u8 else "normalize_chw_kernel": 1, "postprocess_kernel": 1})
    if variant == CLS:
        if decode_only:
            c["kern"] += 2                                            # pred_argmax_decode_kernel<conf, subbin>, one per head
        else:
            c["pred_tail_kernel"] += 2
            c["dec_conf" if conf else "dec"] += 2                     # argmax_{conf_,}decode_kernel<subbin>
        if conf:
            c["conf_resample_kernel"] += 1
    return c


END_KERNELS = {"preprocess_kernel", "normalize_chw_kernel", "postprocess_kernel", "conf_resample_kernel", "pred_tail_kernel", "dec", "dec_conf", "kern"}


def profiled(m, run):
    eng = m._get_engine()
    _native.check(eng.L.pf_profile_kernels_enable(eng.handle, 4096))
    try:
        run()
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(1 << 16)
        _native.check(eng.L.pf_profile_kernels_read(eng.handle, buf, len(buf)))
    finally:
        eng.L.pf_profile_kernels_enable(eng.handle, 0)
    rows = [r.rsplit(",", 2) for r in buf.value.decode().strip().splitlines()[1:]]       # (template names hold commas)
    return collections.Counter({k: int(v) for k, v, _ in rows if k in END_KERNELS})


CONFIGS = [(REG, NH, NW, 0, 0, False) for NH, NW in WORKING] + [(CLS, NH, NW, d, s, c) for NH, NW, _ in DECODE_CASES + [(320, 640, 1)]
                                                                  for d in (0, 1) for s in (0, 1) for c in (False, True)]


def test_restatement_matches_the_graph():
    """For every configuration the file runs, the pre, decode and post launches of one forward equal the restated ones; and the
    file's cases reach every edge named in its docstring."""
    for variant, NH, NW, d, s, c in CONFIGS:
        m = model(variant, NH, NW, debug=False)
        if variant == CLS:
            m.set_option("decode_only", d)
            m.set_option("subbin", s)
        imgs = images([(NH + 3, NW - 5), (41, 77)], 1)
        try:
            got = profiled(m, lambda: forward(m, imgs, conf=c))
            assert got == restated_launches(variant, True, d, c), (variant, NH, NW, d, s, c, got)
            if not d and not c and not s:
                chw = torch.zeros(2, 3, NH, NW, device="cuda")
                assert profiled(m, lambda: forward(m, imgs, chw=chw)) == restated_launches(variant, False, d, c)
        finally:
            if variant == CLS:
                m.set_option("decode_only", 0)
                m.set_option("subbin", 0)
    # edges of A
    seen = set()
    for NH, NW in WORKING:
        for _, sizes, pads in pre_batches(NH, NW):
            budget = batch_budget([h for h, _ in sizes], NH, NW)
            seen |= {f"{passes(h, NH, budget)} passes" for h, _ in sizes}
            seen |= {"up" for h, w in sizes if h < NH or w < NW} | {"down" for h, w in sizes if h > NH and w > NW}
            seen |= {"1x1" for h, w in sizes if h == w == 1} | {"1xN" for h, w in sizes if h == 1 and w > 1}
            seen |= {"wide" for h, w in sizes if w > 4 * NW} | {"tallest" for h, w in sizes if h == tallest(NH, NW)}
            offs = np.cumsum([0] + [p + h * w * 3 for p, (h, w) in zip(pads, sizes)])[:-1] + np.array(pads)
            seen |= {"offset%4" for o in offs if o % 4} | {"offset%16" for o in offs if o % 16 and o % 4 == 0}
    assert {"2 passes", "3 passes", "8 passes", "1 passes", "up", "down", "1x1", "1xN", "wide", "tallest", "offset%4", "offset%16"} <= seen, seen
    assert {ksize(tallest(NH, NW), NH) + 1 == max_rows(NW) for NH, NW in WORKING} == {True, False}
    # edges of C
    p = sorted(decode_passes(*c) for c in DECODE_CASES)
    assert p[0] < 1 and p[1] == 1 and p[2] > 2 and p[2] % 1
    # edges of D
    sizes, mis = post_sizes(320, 320)
    want = {"table", "no table", "W4<256", "W4=256", "W4>256", "W%4", "vec", "W%4=0 misaligned", "ragged band", "ragged group", "H=1"}
    assert post_edges(sizes, mis) == want
    assert (320 * 16, 9) in sizes and (320 // 16, 320 // 16) in sizes
