"""Straightened images from camera parameters on the GPU (hand-written sm_90a kernels, csrc/rectify.cuh).

``upright`` warps each image to a camera with a level horizon (roll 0) and, by default, pitch 0, so vertical lines stay
vertical: this project's rule, DESIGN.md section 1 "Upright warp".  It takes the camera parameters every ParamNet variant's
``inference_batch`` results carry, or ``calibrate.fit_camera``'s output, straight from the device without synchronising, and
returns images that ``PerspectiveFields.inference_batch`` accepts, with the output camera in a centred ParamNet variant's keys.
``rotate_panoramas`` rotates equirectangular panoramas, and ``level_panoramas`` levels tilted ones from a model's predictions
on their crops (DESIGN.md section 1, "Panorama levelling").
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
    - ``focal``: "same" (f_rel of the input times the output height), a vertical field of view in degrees, "fill" (the
      smallest zoom at or above "same" that leaves no fill in the canvas; "same" and status 1 where no zoom can), or
      "fill_common" (one zoom for the whole call, e.g. the frames of a clip: the largest "fill" f_rel of the images with usable
      parameters, times each output height; every status-0 canvas is filled, and status 1 marks images whose own "fill" was
      impossible).  Read from the device cameras without synchronising.
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
        modes = {"same": _native.PF_RECTIFY_SAME, "fill": _native.PF_RECTIFY_FILL, "fill_common": _native.PF_RECTIFY_FILL_COMMON}
        if focal not in modes:
            raise ValueError(f"focal must be 'same', 'fill', 'fill_common' or a vfov in degrees, got {focal!r}")
        focal_mode = modes[focal]
    else:
        if not _real_number(focal) or not 0.0 < float(focal) < 180.0:
            raise ValueError(f"focal must be 'same', 'fill', 'fill_common' or a vfov in (0, 180) degrees, got {focal!r}")
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


PANO_MODES = {"bilinear": _native.PF_EQUI_BILINEAR, "nearest": _native.PF_EQUI_NEAREST}
_PANO_DTYPES = {torch.uint8: _native.PF_EQUI_U8, torch.float32: _native.PF_EQUI_F32}
ORTHONORMAL_TOL = 1e-9
DEFAULT_LEVEL_VIEWS = tuple((70.0, 320, 320, float(az), 0.0, 0.0, 1.0) for az in range(0, 360, 45))


def _check_panoramas(panos):
    """-> (list of panoramas, torch dtype, channels, device or None for host arrays); no GPU work."""
    if isinstance(panos, (torch.Tensor, np.ndarray)):
        raise TypeError("panos must be a list of [Hp, Wp, 3] or [Hp, Wp] panoramas, not one array")
    panos = list(panos)
    if not panos:
        raise ValueError("no panoramas")
    on_dev = [isinstance(p, torch.Tensor) and p.is_cuda for p in panos]
    if any(on_dev) and not all(on_dev):
        raise TypeError("the list mixes CUDA tensors and host panoramas; pass one kind per call")
    out, kinds = [], set()
    for i, p in enumerate(panos):
        if not on_dev[i]:
            if isinstance(p, torch.Tensor):
                raise TypeError(f"panos[{i}] is a CPU tensor: pass a numpy array or a CUDA tensor")
            p = torch.from_numpy(np.ascontiguousarray(p))
        if p.dtype not in _PANO_DTYPES:
            raise TypeError(f"panos[{i}] must be uint8 or float32, got {p.dtype}")
        if p.dim() not in (2, 3) or (p.dim() == 3 and p.shape[2] != 3):
            raise TypeError(f"panos[{i}] must be [Hp, Wp, 3] or [Hp, Wp], got {list(p.shape)}")
        if p.shape[0] < 2 or p.shape[1] < 2 or p.shape[0] * p.shape[1] >= 1 << 31:
            raise ValueError(f"panos[{i}] has size {p.shape[0]} x {p.shape[1]} (2 x 2 at least)")
        kinds.add((p.dtype, 1 if p.dim() == 2 else 3))
        out.append(p)
    if len(kinds) != 1:
        raise TypeError("the panoramas mix dtypes or channel counts; pass one kind per call")
    dev = out[0].device if on_dev[0] else None
    if dev is not None and any(p.device != dev for p in out):
        raise ValueError("the panoramas are on more than one CUDA device")
    dtype, channels = kinds.pop()
    return out, dtype, channels, dev


def _rotations(rotations, n, dev):
    """-> (CUDA float64 [n, 3, 3] tensors to stack or host arrays, device or None).  CUDA tensors are read as they are (no check, no
    synchronisation); host rotations must be orthonormal with determinant +1 to ORTHONORMAL_TOL."""
    if isinstance(rotations, torch.Tensor) and rotations.is_cuda:
        if rotations.dtype != torch.float64 or tuple(rotations.shape) != (n, 3, 3):
            raise ValueError(f"rotations as one CUDA tensor must be float64 [{n}, 3, 3], got {rotations.dtype} {list(rotations.shape)}")
        return list(rotations.unbind(0)), rotations.device
    rots = list(rotations)
    if len(rots) != n:
        raise ValueError(f"{n} panoramas but {len(rots)} rotations")
    out, devs = [], set()
    for i, r in enumerate(rots):
        if isinstance(r, torch.Tensor) and r.is_cuda:
            if r.dtype != torch.float64 or tuple(r.shape) != (3, 3):
                raise ValueError(f"rotations[{i}] must be a float64 [3, 3] tensor, got {r.dtype} {list(r.shape)}")
            devs.add(r.device)
            out.append(r)
            continue
        m = np.asarray(r.numpy() if isinstance(r, torch.Tensor) else r, dtype=np.float64)
        if m.shape != (3, 3) or not np.all(np.isfinite(m)):
            raise ValueError(f"rotations[{i}] must be a finite 3 x 3 matrix, got shape {m.shape}")
        if np.max(np.abs(m @ m.T - np.eye(3))) > ORTHONORMAL_TOL or abs(np.linalg.det(m) - 1.0) > ORTHONORMAL_TOL:
            raise ValueError(f"rotations[{i}] is not a rotation (orthonormal with determinant 1 to {ORTHONORMAL_TOL})")
        out.append(m)
    if len(devs) > 1 or (dev is not None and devs and devs != {dev}):
        raise ValueError("the rotations are on another CUDA device than the panoramas")
    return out, (devs.pop() if devs else None)


def rotate_panoramas(panos, rotations, mode="bilinear", outputs=()):
    """Rotate equirectangular panoramas on the GPU: ``out(d) = P(R d)`` for every direction d (DESIGN.md section 1, "Panorama
    levelling"), so ``rotate_panoramas(P, [fit["rotation"]])`` with ``calibrate.fit_panorama``'s output levels P.  One launch for
    the whole list; sizes may differ.

    - ``panos``: a list of uint8 or float32 [Hp, Wp, 3] or [Hp, Wp] panoramas (one dtype and channel count per call), CUDA
      tensors read in place or numpy arrays uploaded once.  Pixel (i, j) is the direction at longitude 2 pi j / Wp - pi and
      latitude pi/2 - pi i / Hp (x right, y down, z at longitude 0), so row 0 is the pole and only rows 1 .. Hp - 1 of a
      panorama survive the identity unchanged.
    - ``rotations``: one 3 x 3 matrix per panorama, as a CUDA float64 [n, 3, 3] tensor or a list of CUDA float64 [3, 3] tensors
      (read on the device: not checked, no synchronisation) or of host arrays (checked to be rotations to 1e-9).
    - ``mode``: "bilinear" (columns wrap, rows clamp, float64 weights; uint8 rounded to nearest) or "nearest".
    - ``outputs``: () or ("map",): also a float32 [Hp, Wp, 2] map of the input position (u, v) each output pixel samples.

    Returns a dict: ``im`` (list of CUDA views into one 16-byte-aligned blob, in the input dtype) and ``map`` if asked for.
    Nothing synchronises with the device; invalid arguments raise before any GPU work."""
    if mode not in PANO_MODES:
        raise ValueError(f"mode must be one of {tuple(PANO_MODES)}, got {mode!r}")
    outputs = (outputs,) if isinstance(outputs, str) else tuple(outputs)
    bad = [o for o in outputs if o != "map"]
    if bad:
        raise ValueError(f"unknown outputs {bad}; choose from ('map',)")
    src, dtype, channels, dev = _check_panoramas(panos)
    n = len(src)
    if n > 65535:
        raise ValueError(f"{n} panoramas: at most 65535 per call")
    rots, rdev = _rotations(rotations, n, dev)
    dev = _batch.device(__name__, src[:1] + [r for r in rots if isinstance(r, torch.Tensor)][:1])
    if rdev is not None and rdev != dev:
        raise ValueError(f"the rotations are on {rdev}, the panoramas on {dev}")
    L = _native.lib()
    esize = 4 if dtype == torch.float32 else 1
    shapes = [tuple(p.shape) for p in src]
    out_offs, out_total = _batch.layout([math.prod(s) for s in shapes], 16 // esize)
    map_offs, map_total = _batch.layout([2 * s[0] * s[1] for s in shapes], 4) if "map" in outputs else ([-1] * n, 0)
    descs = (_native.pf_rotate_pano * n)()
    with torch.cuda.device(dev):
        if src[0].is_cuda:
            src = [p.contiguous() for p in src]
        else:
            src = _batch.upload([p.numpy() for p in src], dtype, dev)
        base = _batch.base(src)
        for i, p in enumerate(src):
            descs[i] = _native.pf_rotate_pano(shapes[i][0], shapes[i][1], _batch.offset(p, base), out_offs[i], map_offs[i])
        host = [r for r in rots if not isinstance(r, torch.Tensor)]
        up = iter(_batch.upload(host, torch.float64, dev)) if host else iter(())
        R = torch.stack([r if isinstance(r, torch.Tensor) else next(up) for r in rots]).contiguous()
        ws = _batch.workspace(L.pf_rotate_panoramas_workspace(descs, n), dev)
        blob = torch.empty(out_total, dtype=dtype, device=dev)
        xblob = torch.empty(map_total, dtype=torch.float32, device=dev) if "map" in outputs else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_rotate_panoramas(dev.index, descs, n, channels, _PANO_DTYPES[dtype], PANO_MODES[mode], base, blob.data_ptr(),
                                            xblob.data_ptr() if xblob is not None else None, R.data_ptr(), ws.data_ptr(), ws.numel(),
                                            stream))
    res = {"im": _batch.views(blob, out_offs, shapes)}
    if xblob is not None:
        res["map"] = _batch.views(xblob, map_offs, [(s[0], s[1], 2) for s in shapes])
    return res


def level_panoramas(model, panos, views=None, mode="bilinear", weights=None, huber=None):
    """Level tilted 360-degree panoramas with a Perspective Fields model, on the GPU from end to end: for each panorama,
    ``panocam.crop_equi_views`` crops ``views``, ``model.inference_batch`` predicts their fields (one batch for all panoramas),
    ``calibrate.fit_panorama`` fits each panorama's tilt to them, and ``rotate_panoramas`` rotates each panorama upright.

    - ``panos``: a list of uint8 [Hp, Wp, 3] panoramas (CUDA tensors or numpy arrays) in the channel order the model's
      ``inference_batch`` takes; the crops keep it.
    - ``views``: the crops of every panorama, ``crop_equi_views``' ``(vfov, im_w, im_h, azimuth, elevation, roll, ar)`` tuples or
      dicts; by default ``DEFAULT_LEVEL_VIEWS``, 8 crops of 320 x 320 at azimuth 0, 45, ..., 315 degrees, elevation 0, roll 0,
      vfov 70 degrees, ar 1.  Which view set levels real panoramas best has not been measured, nor has the accuracy of the
      levelling on real tilted panoramas.
    - ``mode``: the sampler of the rotation; ``weights`` ("confidence" needs a model built with ``confidence=True``) and
      ``huber``: as in ``calibrate.fit_panorama``.  A model built with ``decode="subbin"`` works unchanged: the fit reads its
      refined fields.

    Returns a dict: ``im`` (the levelled panoramas, ``rotate_panoramas``' output) and ``fits`` (``fit_panorama``'s dicts).
    The fields the model predicts for a crop are its own: no ground truth is used."""
    views = list(DEFAULT_LEVEL_VIEWS if views is None else views)
    if not views:
        raise ValueError("no views")
    src, dtype, channels, dev = _check_panoramas(panos)
    if dtype != torch.uint8 or channels != 3:
        raise TypeError("level_panoramas needs uint8 [Hp, Wp, 3] panoramas (the model's input)")
    from . import calibrate, panocam
    if dev is None:   # host panoramas: uploaded once, for the crops and the rotation
        dev = _batch.device(__name__)
        src = [p.to(dev) for p in src]
    crops = [c for p in src for c in panocam.crop_equi_views(p, views, outputs=())["im"]]
    results = model.inference_batch(crops)
    nv = len(views)
    fits = calibrate.fit_panorama(results, views * len(src), [P for P in range(len(src)) for _ in range(nv)], weights=weights, huber=huber)
    levelled = rotate_panoramas(src, [f["rotation"] for f in fits], mode)
    return {"im": levelled["im"], "fits": fits}
