"""Scoring of predictions against ground-truth Perspective Fields on the GPU (hand-written sm_90a kernels, csrc/metrics.cuh).

- ``encode_bin`` / ``encode_bin_latitude``: the reference's bin encoders (utils/utils.py:94-146), for one field or a batch.
- ``field_errors``: per-image errors of ``pred_gravity_original`` / ``pred_latitude_original`` against ground-truth fields at
  each image's own size (this project's rule, DESIGN.md section 1), with mixed sizes in one call.
- ``param_errors``: absolute differences of the ParamNet's camera parameters.
- ``param_targets`` / ``param_net_losses``: the targets and the loss rule of ParamNet's training branch.

The heads' training losses are ``PerspectiveFields.losses`` and their targets ``PerspectiveFields.targets_from_fields``, and
ParamNet's are ``PerspectiveFields.param_losses``, which use the helpers here.  Nothing here synchronises with the device.
"""
import ctypes

import numpy as np
import torch
import torch.nn.functional as F

from . import _batch, _native

MAX_THRESHOLDS = 8
_LAT_MODES = {"deg": 0, "rad": 1}


def _lat_rad(lat_mode):
    if lat_mode not in _LAT_MODES:
        raise ValueError(f"lat_mode must be 'deg' or 'rad', got {lat_mode!r}")
    return _LAT_MODES[lat_mode]


def batch_view(ts):
    """A list of equally shaped tensors -> one [n, ...] tensor: a view of their common storage when they are rows of one buffer
    at a constant spacing (e.g. the results of one ``inference_batch`` call or the fields of one crop call), else one stack."""
    t0 = ts[0]
    n = len(ts)
    same = all(t.shape == t0.shape and t.stride() == t0.stride() and t.dtype == t0.dtype and t.device == t0.device for t in ts)
    if same and n > 1 and all(t.untyped_storage().data_ptr() == t0.untyped_storage().data_ptr() for t in ts):
        step = ts[1].storage_offset() - t0.storage_offset()
        if step > 0 and all(t.storage_offset() - t0.storage_offset() == i * step for i, t in enumerate(ts)):
            return t0.as_strided((n,) + tuple(t0.shape), (step,) + tuple(t0.stride()), t0.storage_offset())
    if same and n == 1:
        return t0.unsqueeze(0)
    return torch.stack(ts)


def encode_fields(up, lat, gravity_classes, latitude_classes, lat_rad=0):
    """One ``pf_encode_fields`` launch.  up: float32 CUDA [n, H, W, 2]-indexed view given as (tensor, strides (img, row, col,
    comp)) or None; lat: (tensor [n, H, W], strides) or None.  Returns (gt_gravity, gt_latitude), each None when its input is."""
    ref = up[0] if up is not None else lat[0]
    n, h, w = int(ref.shape[0]), int(up[2] if up is not None else lat[2]), int(up[3] if up is not None else lat[3])
    dev = ref.device
    with torch.cuda.device(dev):
        gg = gl = None
        if up is not None:
            gg = torch.empty((n, 2, h, w) if gravity_classes == 2 else (n, h, w), dtype=torch.float32 if gravity_classes == 2 else torch.int64, device=dev)
        if lat is not None:
            gl = torch.empty((n, 1, h, w) if latitude_classes == 1 else (n, h, w), dtype=torch.float32 if latitude_classes == 1 else torch.int64, device=dev)
        i64x4 = ctypes.c_int64 * 4
        us = i64x4(*up[1]) if up is not None else None
        ls = i64x4(*lat[1], 0) if lat is not None else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(_native.lib().pf_encode_fields(
            dev.index, n, h, w, up[0].data_ptr() if up is not None else None, us, lat[0].data_ptr() if lat is not None else None, ls,
            lat_rad, gravity_classes, latitude_classes, gg.data_ptr() if gg is not None else None, gl.data_ptr() if gl is not None else None,
            stream))
    return gg, gl


def encode_bin(vector_field, num_bin):
    """utils/utils.py:94-111 on the GPU: up field(s) ``[2, H, W]`` or ``[n, 2, H, W]`` (float32 CUDA, channels (x, y)) -> int64
    bin labels ``[H, W]`` / ``[n, H, W]`` on the input's device (the reference returns them on the CPU)."""
    v = _batch.cuda_f32(vector_field, "vector_field")
    if v.dim() not in (3, 4) or v.shape[-3] != 2:
        raise ValueError(f"vector_field must be [2, H, W] or [n, 2, H, W], got {list(v.shape)}")
    if _batch.positive_int(num_bin, "num_bin") < 3:
        raise ValueError(f"num_bin must be an integer >= 3, got {num_bin!r}")
    b = v if v.dim() == 4 else v.unsqueeze(0)
    if b.numel() == 0:
        return torch.empty(tuple(b.shape[:1]) + tuple(b.shape[2:]) if v.dim() == 4 else tuple(v.shape[1:]), dtype=torch.int64, device=v.device)
    s = b.stride()
    gg, _ = encode_fields((b, (s[0], s[2], s[3], s[1]), b.shape[2], b.shape[3]), None, int(num_bin), 1)
    return gg if v.dim() == 4 else gg[0]


def encode_bin_latitude(latimap, num_classes):
    """utils/utils.py:133-146 on the GPU: latitude map(s) in degrees ``[H, W]`` or ``[n, H, W]`` (float32 CUDA) -> int64 class
    labels of the same shape on the input's device (the reference returns them on the CPU)."""
    v = _batch.cuda_f32(latimap, "latimap")
    if v.dim() not in (2, 3):
        raise ValueError(f"latimap must be [H, W] or [n, H, W], got {list(v.shape)}")
    if _batch.positive_int(num_classes, "num_classes") < 2:
        raise ValueError(f"num_classes must be an integer >= 2, got {num_classes!r}")
    b = v if v.dim() == 3 else v.unsqueeze(0)
    if b.numel() == 0:
        return torch.empty(v.shape, dtype=torch.int64, device=v.device)
    _, gl = encode_fields(None, (b, b.stride(), b.shape[1], b.shape[2]), 2, int(num_classes))
    return gl if v.dim() == 3 else gl[0]


def field_errors(results, up, lat, lat_mode="deg", mask=None, thresholds=(1.0, 5.0, 10.0), return_maps=False):
    """Per-image errors of ``results[i]["pred_gravity_original"]`` ([2, H, W]) and ``["pred_latitude_original"]`` ([H, W],
    degrees) against ground truth ``up[i]`` ([H, W, 2]) and ``lat[i]`` ([H, W], ``lat_mode`` "deg" or "rad") at each image's
    own size, in one pass (sizes may differ).  ``mask``: None or a list of bool [H, W] tensors (None entries allowed) that
    restricts both fields.  The rule (DESIGN.md section 1):

    - up: the angle in degrees between the predicted and the true vector, atan2(|p x g|, p . g), at pixels where g is finite and
      |g| > 1e-5; a prediction of length <= 1e-5 (the classification decoder's "no direction" bin) or not finite counts as 180.
    - latitude: |pred - gt| in degrees where gt is finite; a non-finite prediction counts as +inf.

    Returns ``{"up": stats, "latitude": stats}`` with ``stats = {"count": int64 [n], "mean": float64 [n], "median": float64
    [n], "fraction": float64 [n, T]}`` on the device: the valid pixels, their mean and median (``np.median``: the mean of the
    two middle values; NaN for count 0) and the fraction of them with an error below each threshold.  With ``return_maps``
    each stats dict also holds ``"map"``, the list of float32 [H, W] error maps (NaN at invalid pixels)."""
    lat_rad = _lat_rad(lat_mode)
    thr = [float(t) for t in thresholds]
    if len(thr) > MAX_THRESHOLDS:
        raise ValueError(f"at most {MAX_THRESHOLDS} thresholds, got {len(thr)}")
    if any(t != t for t in thr):
        raise ValueError("a threshold is NaN")
    n = len(results)
    if len(up) != n or len(lat) != n or (mask is not None and len(mask) != n):
        raise ValueError(f"{n} results but {len(up)} up fields, {len(lat)} latitude maps" + ("" if mask is None else f", {len(mask)} masks"))
    T = len(thr)
    if n == 0:
        dev = _batch.device(__name__)
        empty = lambda: {"count": torch.empty(0, dtype=torch.int64, device=dev), "mean": torch.empty(0, dtype=torch.float64, device=dev),
                         "median": torch.empty(0, dtype=torch.float64, device=dev), "fraction": torch.empty((0, T), dtype=torch.float64, device=dev)}
        out = {"up": empty(), "latitude": empty()}
        if return_maps:
            out["up"]["map"], out["latitude"]["map"] = [], []
        return out
    pu, pl, ms, dev = _batch.prediction_fields(results, mask, 1)
    gu = [_batch.cuda_f32(u, f"up[{i}]", dev) for i, u in enumerate(up)]
    gl = [_batch.cuda_f32(v, f"lat[{i}]", dev) for i, v in enumerate(lat)]
    for i in range(n):
        h, w = int(pu[i].shape[0]), int(pu[i].shape[1])
        if tuple(gu[i].shape) != (h, w, 2):
            raise ValueError(f"up[{i}] must be [{h}, {w}, 2], got {list(gu[i].shape)}")
        if tuple(gl[i].shape) != (h, w):
            raise ValueError(f"lat[{i}] must be [{h}, {w}], got {list(gl[i].shape)}")
        gl[i] = gl[i].contiguous()
    L = _native.lib()
    bpu, bpl, bgu, bgl, bm = _batch.base(pu), _batch.base(pl), _batch.base(gu), _batch.base(gl), _batch.base(ms)
    descs = (_native.pf_field_image * n)()
    for i in range(n):
        d = descs[i]
        d.height, d.width = int(pu[i].shape[0]), int(pu[i].shape[1])
        d.pred_up_offset, d.pred_up_stride[:] = _batch.offset(pu[i], bpu), pu[i].stride()
        d.pred_lat_offset = _batch.offset(pl[i], bpl)
        d.gt_up_offset, d.gt_up_stride[:] = _batch.offset(gu[i], bgu), gu[i].stride()
        d.gt_lat_offset = _batch.offset(gl[i], bgl)
        d.mask_offset = _batch.offset(ms[i], bm)
    with torch.cuda.device(dev):
        ws = _batch.workspace(L.pf_field_errors_workspace(descs, n, int(bool(return_maps))), dev)
        total = sum(d.height * d.width for d in descs)
        maps = torch.empty((2, total), dtype=torch.float32, device=dev) if return_maps else None
        count = torch.empty((2, n), dtype=torch.int64, device=dev)
        mean = torch.empty((2, n), dtype=torch.float64, device=dev)
        median = torch.empty((2, n), dtype=torch.float64, device=dev)
        frac = torch.empty((2, n, T), dtype=torch.float64, device=dev)
        th = (ctypes.c_double * max(T, 1))(*thr)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_field_errors(dev.index, descs, n, bpu, bpl, bgu, bgl, bm or None, lat_rad, th, T,
                                        maps[0].data_ptr() if return_maps else None, maps[1].data_ptr() if return_maps else None,
                                        count.data_ptr(), mean.data_ptr(), median.data_ptr(), frac.data_ptr() if T else None,
                                        ws.data_ptr(), ws.numel(), stream))
    out = {}
    for f, key in enumerate(("up", "latitude")):
        out[key] = {"count": count[f], "mean": mean[f], "median": median[f], "fraction": frac[f]}
        if return_maps:
            sizes = [d.height * d.width for d in descs]
            out[key]["map"] = [m.view(d.height, d.width) for m, d in zip(maps[f].split(sizes), descs)]
    return out


_PARAMS_CENTERED = ("roll", "pitch", "vfov")
_PARAMS_UNCENTERED = ("roll", "pitch", "general_vfov", "rel_cx", "rel_cy")


def param_errors(results, gt):
    """|prediction - ground truth| of the camera parameters the variant's ParamNet predicts: roll, pitch and vfov (centred
    variants) or roll, pitch, general_vfov, rel_cx and rel_cy (uncentred variants), in the units of the results.  ``gt``: dict
    from some of those names to [n] tensors or sequences.  Returns a dict of float64 [n] tensors on the results' device."""
    if not results:
        raise ValueError("no results")
    r0 = results[0]
    if "pred_roll" not in r0:
        raise ValueError("the results carry no camera parameters: this variant has no ParamNet")
    keys = _PARAMS_CENTERED if "pred_vfov" in r0 else _PARAMS_UNCENTERED
    out = {}
    for k, v in gt.items():
        if k not in keys:
            raise ValueError(f"{k!r} is not predicted by this variant (it predicts {keys})")
        pred = torch.stack([r["pred_" + k] for r in results]).double()
        g = torch.as_tensor(v, dtype=torch.float64, device=pred.device)
        if tuple(g.shape) != (len(results),):
            raise ValueError(f"gt[{k!r}] must have shape [{len(results)}], got {list(g.shape)}")
        out[k] = (pred - g).abs()
    return out


# ParamNetConvNextRegress.factors (param_network.py:183-191)
_PARAM_FACTORS = {"roll": 90.0, "pitch": 90.0, "vfov": 90.0, "rel_focal": 1.0, "rel_cx": 1.0, "rel_cy": 1.0, "general_vfov": 90.0}


def param_targets(batched_inputs, n, param_net, predict_params):
    """Host float32 targets of ParamNet's training branch (param_network.py:72-98, :223-229) from ``batched_inputs[i][key]``
    (host numbers, degrees): ``ParamNet`` [n, 5] = (roll / 90, pitch / 90, vfov / 90, 0, 0); ``ParamNetConvNextRegress``
    [n, len(predict_params)] = value / factor per key.  Each quotient is taken in float64 and then rounded to float32."""
    if len(batched_inputs) != n:
        raise ValueError(f"{n} pairs of fields but {len(batched_inputs)} batched_inputs")
    keys = _PARAMS_CENTERED if param_net == "ParamNet" else tuple(predict_params)
    gt = np.zeros((n, 5 if param_net == "ParamNet" else len(keys)), np.float64)
    for i, x in enumerate(batched_inputs):
        for j, k in enumerate(keys):
            if k not in x:
                raise KeyError(f"batched_inputs[{i}] has no {k!r} (the targets need {keys})")
            v = x[k]
            if isinstance(v, torch.Tensor) or not isinstance(v, (int, float, np.integer, np.floating)) or isinstance(v, (bool, np.bool_)):
                raise TypeError(f"batched_inputs[{i}][{k!r}] must be a host number, got {type(v).__name__}")
            gt[i, j] = float(v) / _PARAM_FACTORS[k]
    return gt.astype(np.float32)


def param_net_losses(raw, gt, param_net, predict_params, loss_weight):
    """ParamNet's losses (param_network.py:102-128 ``ParamNet.losses`` with RECOVER_RPF and without RECOVER_PP, :233-241
    ``ParamNetConvNextRegress.losses``) from its raw head outputs ``raw`` float32 [n, 5] and ``param_targets``' ``gt`` on the
    same device, in float32 and in the reference's order of operations:

    - ``ParamNet``: ``{"param-l1-loss": mean(|raw - gt| * [1, 1, 1, 0, 0]) * loss_weight}``, the mean over all 5n entries;
    - ``ParamNetConvNextRegress``: ``{"param/<key>-loss": mean_i((raw - gt)^2 * loss_weight)}`` per key of ``predict_params``.

    Device-agnostic torch operations; returns 0-dim float32 tensors on ``raw``'s device."""
    if param_net == "ParamNet":
        mask = torch.ones_like(raw)
        mask[:, 3:] = 0.0
        return {"param-l1-loss": (F.l1_loss(raw, gt, reduction="none") * mask).mean() * loss_weight}
    itemized = F.mse_loss(raw, gt, reduction="none") * loss_weight
    return {f"param/{k}-loss": itemized[:, j].mean() for j, k in enumerate(predict_params)}
