"""How the feature calls (panorama crops, drawing, scoring, camera fit, upright warp) describe a batch of differently sized
device tensors to one library call: the CUDA device the call runs on, descriptors that address tensors as base pointer +
element offset, packed output blobs, one pinned upload of host arrays, the library's workspace and the checks their
arguments share."""
import math

import numpy as np
import torch

from . import _native


def device(module, tensors=(), device=None):
    """The CUDA device a call of ``module`` runs on: the device of the first CUDA tensor among ``tensors``, else ``device``, else
    the current one, always with an index."""
    for t in tensors:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            return t.device
    if not torch.cuda.is_available():
        raise RuntimeError(f"{module} needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda") if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"{module} needs a CUDA device (there is no CPU path)")
    return torch.device("cuda", torch.cuda.current_device()) if dev.index is None else dev


def base(tensors):
    """Common base address of a list of device tensors (None entries allowed): descriptors address each by its element offset
    from it (``offset``), so one library call reads them in place."""
    ptrs = [t.data_ptr() for t in tensors if t is not None]
    return min(ptrs) if ptrs else 0


def offset(t, base):
    """``t``'s offset from ``base`` in its own elements; -1 (absent) for None."""
    return -1 if t is None else (t.data_ptr() - base) // t.element_size()


def up_view(up, h, w):
    """An up field given as ``[2, H, W]`` or ``[H, W, 2]`` -> its ``[H, W, 2]`` view, whose strides are the (row, column,
    component) strides the library reads; None for any other shape."""
    shape = tuple(up.shape)
    if shape == (2, h, w):
        return up.permute(1, 2, 0)
    return up if shape == (h, w, 2) else None


def layout(sizes, align=1):
    """Items of ``sizes`` elements packed back to back, each starting at a multiple of ``align`` -> (offsets, total)."""
    offsets, total = [], 0
    for s in sizes:
        offsets.append(total)
        total += (s + align - 1) // align * align
    return offsets, total


def views(blob, offsets, shapes):
    """Per-item views of the given shapes into a packed blob."""
    return [blob[o:o + math.prod(s)].view(s) for o, s in zip(offsets, shapes)]


def upload(arrays, dtype, dev):
    """Host arrays -> one pinned buffer of ``dtype``, one non-blocking copy to ``dev`` -> per-array device views."""
    arrays = [np.asarray(a) for a in arrays]
    offsets, total = layout([a.size for a in arrays])
    host = torch.empty(total, dtype=dtype, pin_memory=True)
    flat = host.numpy()
    for a, o in zip(arrays, offsets):
        flat[o:o + a.size] = a.reshape(-1)
    return views(host.to(dev, non_blocking=True), offsets, [a.shape for a in arrays])


def workspace(need, dev):
    """A library call's workspace of ``need`` bytes (the result of its ``*_workspace`` query, checked) on ``dev``."""
    return torch.empty(_native.check(need), dtype=torch.uint8, device=dev)


def cuda_f32(t, what, device=None):
    """A float32 CUDA tensor (on ``device`` when given), else TypeError / ValueError: there is no CPU path."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch tensor, got {type(t).__name__}")
    if t.dtype != torch.float32:
        raise TypeError(f"{what} must be float32, got {t.dtype}")
    if not t.is_cuda:
        raise ValueError(f"{what} is on {t.device}: perspectivefields_b200 scores on a CUDA device only (there is no CPU path)")
    if device is not None and t.device != device:
        raise ValueError(f"{what} is on {t.device}, expected {device}")
    return t


def prediction_fields(results, mask, min_size):
    """``results[i]["pred_gravity_original"]`` ([2, H, W]) and ``["pred_latitude_original"]`` ([H, W]) float32 CUDA tensors of one
    device, at least ``min_size`` x ``min_size``, and ``mask`` (None or a list of bool [H, W] tensors, None entries allowed) ->
    (up fields as [H, W, 2] views, contiguous latitude maps, masks as uint8 or None, device)."""
    n = len(results)
    pu = [cuda_f32(r["pred_gravity_original"], f"results[{i}]['pred_gravity_original']") for i, r in enumerate(results)]
    dev = pu[0].device
    pl = [cuda_f32(r["pred_latitude_original"], f"results[{i}]['pred_latitude_original']", dev) for i, r in enumerate(results)]
    ms = [None] * n if mask is None else list(mask)
    for i in range(n):
        if pu[i].dim() != 3 or pu[i].shape[0] != 2:
            raise ValueError(f"results[{i}]['pred_gravity_original'] must be [2, H, W], got {list(pu[i].shape)}")
        h, w = int(pu[i].shape[1]), int(pu[i].shape[2])
        if h < min_size or w < min_size:
            raise ValueError(f"image {i} has size {h}x{w} ({min_size}x{min_size} at least)")
        if tuple(pl[i].shape) != (h, w):
            raise ValueError(f"results[{i}]['pred_latitude_original'] must be [{h}, {w}], got {list(pl[i].shape)}")
        if ms[i] is not None:
            m = ms[i]
            if not isinstance(m, torch.Tensor) or m.dtype != torch.bool or tuple(m.shape) != (h, w) or m.device != dev:
                raise ValueError(f"mask[{i}] must be a bool [{h}, {w}] tensor on {dev}")
            ms[i] = m.contiguous().view(torch.uint8)
        pu[i], pl[i] = pu[i].permute(1, 2, 0), pl[i].contiguous()
    return pu, pl, ms, dev


CONFIDENCE_KEYS = ("pred_gravity_confidence_original", "pred_latitude_confidence_original")


def fit_weights(weights, results, pu, dev):
    """``fit_camera``'s ``weights`` for the fields ``prediction_fields`` returned (``pu``: the [H, W, 2] up views): None, "confidence"
    (the two ``CONFIDENCE_KEYS`` maps of each result) or a list of n entries, each None or a pair (up weight, latitude weight) of
    float32 [H, W] tensors on ``dev``, either of them None -> per image (up weight, latitude weight), contiguous or None.
    ValueError for anything else, before any GPU work of the library."""
    n = len(results)
    if weights is None:
        return [(None, None)] * n
    if isinstance(weights, str):
        if weights != "confidence":
            raise ValueError(f"weights must be None, 'confidence' or a list of (up, latitude) weight pairs, got {weights!r}")
        for i, r in enumerate(results):
            for k in CONFIDENCE_KEYS:
                if k not in r:
                    raise ValueError(f"weights='confidence': results[{i}] has no {k!r} (run a model built with confidence=True)")
        entries = [(r[CONFIDENCE_KEYS[0]], r[CONFIDENCE_KEYS[1]]) for r in results]
        what = ["results[{i}]['" + k + "']" for k in CONFIDENCE_KEYS]
    else:
        if isinstance(weights, torch.Tensor) or not isinstance(weights, (list, tuple)):
            raise ValueError(f"weights must be None, 'confidence' or a list of {n} entries, got {type(weights).__name__}")
        entries = list(weights)
        if len(entries) != n:
            raise ValueError(f"{n} results but {len(entries)} weight entries")
        what = ["weights[{i}][0]", "weights[{i}][1]"]
    out = []
    for i, e in enumerate(entries):
        if e is None:
            out.append((None, None))
            continue
        if not isinstance(e, (tuple, list)) or len(e) != 2:
            raise ValueError(f"weights[{i}] must be None or a pair (up weight, latitude weight), got {type(e).__name__}")
        h, w = int(pu[i].shape[0]), int(pu[i].shape[1])
        for j, t in enumerate(e):
            if t is not None and (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != (h, w) or t.device != dev):
                raise ValueError(f"{what[j].format(i=i)} must be None or a float32 [{h}, {w}] tensor on {dev}")
        out.append(e)
    return [tuple(None if t is None else t.contiguous() for t in e) for e in out]


def _number(x, kinds):
    return isinstance(x, kinds) and not isinstance(x, (bool, np.bool_))


def real(x, name):
    """A finite real number as a float, else ValueError."""
    if not _number(x, (int, float, np.integer, np.floating)) or not math.isfinite(float(x)):
        raise ValueError(f"{name} must be a finite real number, got {x!r}")
    return float(x)


def positive_int(x, name):
    """A positive integer as an int, else ValueError."""
    if not _number(x, (int, np.integer)) or int(x) < 1:
        raise ValueError(f"{name} must be a positive integer, got {x!r}")
    return int(x)


def unit(x, name):
    """A number in [0, 1] as a float, else ValueError."""
    if not _number(x, (int, float, np.integer, np.floating)) or not 0.0 <= float(x) <= 1.0:
        raise ValueError(f"{name} must be a number in [0, 1], got {x!r}")
    return float(x)
