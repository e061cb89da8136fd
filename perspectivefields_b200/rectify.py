"""Straightened images from camera parameters on the GPU (hand-written sm_90a kernels, csrc/rectify.cuh).

``upright`` warps each image to a camera with a level horizon (roll 0) and, by default, pitch 0, so vertical lines stay
vertical: this project's rule, DESIGN.md section 1 "Upright warp".  It takes the camera parameters every ParamNet variant's
``inference_batch`` results carry, or ``calibrate.fit_camera``'s output, straight from the device without synchronising, and
returns images that ``PerspectiveFields.inference_batch`` accepts, with the output camera in a centred ParamNet variant's keys.
"""
import ctypes
import math
import numbers

import numpy as np
import torch

from . import _batch, _native

CAMERA_KEYS = ("pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy")
OUTPUT_KEYS = ("pred_roll", "pred_pitch", "pred_vfov", "pred_rel_focal", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy")
MODES = {"bilinear": _native.PF_RECTIFY_BILINEAR, "nearest": _native.PF_RECTIFY_NEAREST}
OUTPUTS = ("mask", "map")
_REAL_DTYPES = (torch.float64, torch.float32, torch.float16, torch.bfloat16, torch.int32, torch.int64)


def _real_number(x):
    return isinstance(x, (numbers.Real, np.floating, np.integer)) and not isinstance(x, (bool, np.bool_))


def _check_images(images):
    """-> (list of uint8 images, channels, device or None for host images); no GPU work."""
    if isinstance(images, (torch.Tensor, np.ndarray)):
        raise TypeError("images must be a list of [H, W, 3] or [H, W] uint8 images, not one array")
    images = list(images)
    if not images:
        raise ValueError("no images")
    on_dev = [isinstance(im, torch.Tensor) and im.is_cuda for im in images]
    if any(on_dev) and not all(on_dev):
        raise TypeError("the list mixes CUDA tensors and host images; pass one kind per call")
    out, chans = [], set()
    for i, im in enumerate(images):
        if not on_dev[i]:
            if isinstance(im, torch.Tensor):
                raise TypeError(f"images[{i}] is a CPU tensor: pass a numpy array or a CUDA tensor")
            im = np.asarray(im)
        if im.dtype not in (np.uint8, torch.uint8):
            raise TypeError(f"images[{i}] must be uint8, got {im.dtype}")
        if im.ndim not in (2, 3) or (im.ndim == 3 and im.shape[2] != 3):
            raise TypeError(f"images[{i}] must be [H, W, 3] or [H, W], got {list(im.shape)}")
        if im.shape[0] < 1 or im.shape[1] < 1 or im.shape[0] * im.shape[1] >= 1 << 31:
            raise ValueError(f"images[{i}] has size {im.shape[0]} x {im.shape[1]}")
        chans.add(1 if im.ndim == 2 else 3)
        out.append(im)
    if len(chans) != 1:
        raise TypeError("the images mix [H, W] and [H, W, 3]; pass one channel count per call")
    dev = None
    if on_dev[0]:
        dev = out[0].device
        if any(im.device != dev for im in out):
            raise ValueError("the images are on more than one CUDA device")
    return out, chans.pop(), dev


def _check_cameras(cameras, n, dev):
    """-> per key, a list of n entries: a 0-dim CUDA tensor on dev (None: any device) or a float."""
    if isinstance(cameras, dict):
        raise TypeError("cameras must be a list of dicts, one per image")
    cameras = list(cameras)
    if len(cameras) != n:
        raise ValueError(f"{n} images but {len(cameras)} cameras")
    cols = {k: [] for k in CAMERA_KEYS}
    for i, c in enumerate(cameras):
        if not isinstance(c, dict):
            raise TypeError(f"cameras[{i}] must be a dict, got {type(c).__name__}")
        missing = [k for k in CAMERA_KEYS if k not in c]
        if missing:
            raise ValueError(f"cameras[{i}] lacks {missing} (a variant without ParamNet: use calibrate.fit_camera's output)")
        for k in CAMERA_KEYS:
            v = c[k]
            if isinstance(v, torch.Tensor):
                if v.dim() != 0 and v.numel() != 1 or v.dtype not in _REAL_DTYPES:
                    raise ValueError(f"cameras[{i}][{k!r}] must be one real number, got {v.dtype} {list(v.shape)}")
                if v.is_cuda:
                    if dev is not None and v.device != dev:
                        raise ValueError(f"cameras[{i}][{k!r}] is on {v.device}, the images on {dev}")
                    cols[k].append(v if v.dim() == 0 else v.reshape(()))
                    continue
                v = v.item()
            if not _real_number(v):
                raise TypeError(f"cameras[{i}][{k!r}] must be a real number or a 0-dim tensor, got {type(v).__name__}")
            cols[k].append(float(v))
    return cols


def _check_size(size, images):
    if size is None:
        return [(int(im.shape[0]), int(im.shape[1])) for im in images]
    sizes = list(size)
    if len(sizes) == 2 and all(isinstance(s, (int, np.integer)) and not isinstance(s, bool) for s in sizes):
        sizes = [tuple(sizes)] * len(images)
    if len(sizes) != len(images):
        raise ValueError(f"size must be (H, W) or one (H, W) per image, got {size!r}")
    out = []
    for i, s in enumerate(sizes):
        if s is None:
            out.append((int(images[i].shape[0]), int(images[i].shape[1])))
            continue
        s = tuple(s)
        if len(s) != 2:
            raise ValueError(f"size[{i}] must be two positive integers, got {s!r}")
        h, w = _batch.positive_int(s[0], f"size[{i}][0]"), _batch.positive_int(s[1], f"size[{i}][1]")
        if h * w >= 1 << 31:
            raise ValueError(f"size[{i}] is {h} x {w}: too large")
        out.append((h, w))
    return out


def _params(cols, n, dev):
    """float64 [n, 5] on dev: CUDA values stacked on the device, numbers uploaded once from pinned memory (no synchronisation)."""
    host = np.full((n, 5), math.nan)
    any_host = False
    for j, k in enumerate(CAMERA_KEYS):
        for i, v in enumerate(cols[k]):
            if not isinstance(v, torch.Tensor):
                host[i, j] = v
                any_host = True
    up = _batch.upload([host], torch.float64, dev)[0] if any_host else None
    out = []
    for j, k in enumerate(CAMERA_KEYS):
        col = cols[k]
        if all(isinstance(v, torch.Tensor) for v in col):
            out.append(torch.stack([v.to(torch.float64) for v in col]) if len(set(v.dtype for v in col)) > 1 else torch.stack(col).to(torch.float64))
        elif not any(isinstance(v, torch.Tensor) for v in col):
            out.append(up[:, j])
        else:
            out.append(torch.stack([v.to(torch.float64) if isinstance(v, torch.Tensor) else up[i, j] for i, v in enumerate(col)]))
    return torch.stack(out, dim=1).contiguous()


def upright(images, cameras, keep_pitch=False, focal="same", size=None, mode="bilinear", fill=0, outputs=("mask",)):
    """Straighten ``images[i]`` (uint8 [H, W, 3] or [H, W]; CUDA tensors read in place, or numpy arrays uploaded once; sizes may
    differ) with the camera ``cameras[i]``: a dict with ``pred_roll``, ``pred_pitch``, ``pred_general_vfov`` (degrees),
    ``pred_rel_cx`` and ``pred_rel_cy`` (0-dim CUDA tensors or numbers), as every ParamNet variant's ``inference_batch`` results
    and ``calibrate.fit_camera``'s output carry them.  f_rel comes from the general vfov and principal point.

    - ``keep_pitch``: False (roll 0 and pitch 0: vertical lines stay vertical) or True (roll 0 only: an in-plane rotation about
      the principal point that levels the horizon).
    - ``focal``: "same" (f_rel of the input times the output height), a vertical field of view in degrees, or "fill" (the
      smallest zoom at or above "same" that leaves no fill in the canvas; "same" and status 1 where no zoom can).
    - ``size``: None (each input's size), one (H, W) for all, or one per image.
    - ``mode``: "bilinear" (rounded to nearest) or "nearest" (for masks and label images).  No antialiasing: a focal length that
      shrinks an image strongly aliases.
    - ``fill``: the value (0 .. 255, or one per channel) of output pixels whose ray misses the input.
    - ``outputs``: any of "mask" (bool [H_o, W_o], True where sampled) and "map" (float32 [H_o, W_o, 2], the input pixel-centre
      position (x, y) each output pixel samples, pixel (i, j) centred at (j + 0.5, i + 0.5); NaN where not sampled).

    Returns a dict: ``im`` (list of CUDA views into one 16-byte-aligned blob; the [H, W, 3] ones are valid
    ``PerspectiveFields.inference_batch`` input), ``mask`` / ``map`` (lists) if asked for, ``camera`` (one dict per image of 0-dim
    float64 CUDA tensors with a centred ParamNet variant's keys, for ``panocam.fields_from_predictions`` and
    ``viz.draw_from_r_p_f_cx_cy``) and ``status`` (int32 CUDA [n]: 0 ok, 1 "fill" impossible, 2 unusable parameters -- non-finite,
    a general vfov outside (0, 180) or f_rel <= 0 --: the image is all fill, the mask False, the map and camera NaN).  Nothing
    synchronises with the device; invalid arguments raise before any GPU work."""
    if not isinstance(keep_pitch, bool):
        raise TypeError(f"keep_pitch must be a bool, got {keep_pitch!r}")
    vfov = 0.0
    if isinstance(focal, str):
        if focal not in ("same", "fill"):
            raise ValueError(f"focal must be 'same', 'fill' or a vfov in degrees, got {focal!r}")
        focal_mode = _native.PF_RECTIFY_SAME if focal == "same" else _native.PF_RECTIFY_FILL
    else:
        if not _real_number(focal) or not 0.0 < float(focal) < 180.0:
            raise ValueError(f"focal must be 'same', 'fill' or a vfov in (0, 180) degrees, got {focal!r}")
        focal_mode, vfov = _native.PF_RECTIFY_VFOV, float(focal)
    if mode not in MODES:
        raise ValueError(f"mode must be one of {tuple(MODES)}, got {mode!r}")
    outputs = (outputs,) if isinstance(outputs, str) else tuple(outputs)
    bad = [o for o in outputs if o not in OUTPUTS]
    if bad:
        raise ValueError(f"unknown outputs {bad}; choose from {OUTPUTS}")
    imgs, channels, dev = _check_images(images)
    n = len(imgs)
    if n > 65535:
        raise ValueError(f"{n} images: at most 65535 per call")
    fills = [fill] * channels if _real_number(fill) else list(fill)
    if len(fills) != channels or any(not _real_number(v) or int(v) != v or not 0 <= v <= 255 for v in fills):
        raise ValueError(f"fill must be an integer in 0 .. 255 or one per channel ({channels}), got {fill!r}")
    sizes = _check_size(size, imgs)
    cols = _check_cameras(cameras, n, dev)
    cam_tensors = [v for k in CAMERA_KEYS for v in cols[k] if isinstance(v, torch.Tensor)]
    if dev is None and len({v.device for v in cam_tensors}) > 1:
        raise ValueError("the cameras are on more than one CUDA device")
    dev = _batch.device(__name__, imgs[:1] + cam_tensors[:1])
    L = _native.lib()
    out_offs, out_total = _batch.layout([channels * ho * wo for ho, wo in sizes], 16)
    mask_offs, mask_total = _batch.layout([ho * wo for ho, wo in sizes], 16) if "mask" in outputs else ([-1] * n, 0)
    map_offs, map_total = _batch.layout([2 * ho * wo for ho, wo in sizes], 4) if "map" in outputs else ([-1] * n, 0)
    descs = (_native.pf_rectify_image * n)()
    for i, (im, (ho, wo)) in enumerate(zip(imgs, sizes)):
        descs[i] = _native.pf_rectify_image(int(im.shape[0]), int(im.shape[1]), ho, wo, 0, out_offs[i], mask_offs[i], map_offs[i])
    with torch.cuda.device(dev):
        src = [im.contiguous() for im in imgs] if isinstance(imgs[0], torch.Tensor) else _batch.upload(imgs, torch.uint8, dev)
        base = _batch.base(src)
        for d, t in zip(descs, src):
            d.in_offset = t.data_ptr() - base
        params = _params(cols, n, dev)
        ws = _batch.workspace(L.pf_rectify_workspace(descs, n), dev)
        blob = torch.empty(out_total, dtype=torch.uint8, device=dev)
        mblob = torch.empty(mask_total, dtype=torch.uint8, device=dev) if "mask" in outputs else None
        xblob = torch.empty(map_total, dtype=torch.float32, device=dev) if "map" in outputs else None
        cam = torch.empty((n, 5), dtype=torch.float64, device=dev)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        fv = (ctypes.c_int32 * 3)(*[int(v) for v in fills] + [0] * (3 - channels))
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_rectify_views(dev.index, descs, n, base, blob.data_ptr(), mblob.data_ptr() if mblob is not None else None,
                                         xblob.data_ptr() if xblob is not None else None, channels, params.data_ptr(), int(keep_pitch),
                                         focal_mode, vfov, MODES[mode], fv, cam.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(),
                                         stream))
        roll, pitch, gv, cx, cy = cam.t()
        f = 0.5 / torch.tan(torch.deg2rad(gv) / 2.0)
        cols_out = torch.stack([roll, pitch, gv, f, gv, cx, cy]).t().unbind(0)
    res = {"im": _batch.views(blob, out_offs, [(ho, wo, 3) if channels == 3 else (ho, wo) for ho, wo in sizes])}
    if mblob is not None:
        res["mask"] = _batch.views(mblob.view(torch.bool), mask_offs, sizes)
    if xblob is not None:
        res["map"] = _batch.views(xblob, map_offs, [(ho, wo, 2) for ho, wo in sizes])
    res["camera"] = [dict(zip(OUTPUT_KEYS, c.unbind(0))) for c in cols_out]
    res["status"] = status
    return res
