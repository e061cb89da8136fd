"""Camera parameters from Perspective Fields on the GPU (hand-written sm_90a kernels, csrc/calib.cuh).

``fit_camera`` fits roll, pitch, focal length and optionally the principal point to the up and latitude fields of each image
by Levenberg-Marquardt (this project's rule, DESIGN.md section 1 "Camera fit").  It gives every field-only variant
(``PersNet-360Cities``) the camera parameters its ParamNet-less model lacks, and gives ParamNet variants a geometric check or
refinement of theirs.  With ``groups`` it fits images taken with one camera together (the frames of a video, a burst, one
phone's photos): each image keeps its own roll and pitch, and each group gets one focal length (and principal point), which one
image alone constrains least (DESIGN.md section 1, "Shared intrinsics").  Its output has the keys of a ParamNet variant's
results, so ``metrics.param_errors``, ``panocam.fields_from_predictions`` and ``viz.draw_from_r_p_f_cx_cy`` take it unchanged.
``fit_panorama`` fits one tilt per equirectangular panorama to the fields of views cropped from it (DESIGN.md section 1,
"Panorama levelling").
"""
import ctypes
import math
import numbers

import numpy as np
import torch

from . import _batch, _native
from .panocam import _check_equi_view, general_vfov, general_vfov_to_focal

MAX_ITERATIONS = 1000
_NAN_INIT = (math.nan,) * 5


def _init_from_results(results):
    """The ParamNet parameters the results carry as fit starts (roll, pitch in radians, f_rel, cx_rel, cy_rel).  f_rel is
    recomputed from the general vfov and principal point, as ``fields_from_predictions`` draws them.  Reads them on the host."""
    keys = ("pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy")
    for i, r in enumerate(results):
        if any(k not in r for k in keys):
            raise ValueError(f"init='results': results[{i}] carries no camera parameters (a variant without ParamNet); use init='fields'")
    v = torch.stack([torch.stack([torch.as_tensor(r[k]).reshape(()).to("cpu", torch.float64) for k in keys]) for r in results]).numpy()
    f = general_vfov_to_focal(v[:, 3], v[:, 4], 1, v[:, 2], True)
    out = []
    for i in range(len(results)):
        t = (math.radians(v[i, 0]), math.radians(v[i, 1]), float(f[i]), float(v[i, 3]), float(v[i, 4]))
        if not all(math.isfinite(x) for x in t) or not t[2] > 0:
            raise ValueError(f"init='results': results[{i}] has camera parameters that give no valid start: {t}")
        out.append(t)
    return out


def _group_ids(groups, n):
    """Labels compacted in order of first appearance: (int32 group of each image, number of groups)."""
    try:
        labels = list(groups)
    except TypeError:
        raise ValueError(f"groups must be None or a sequence of {n} integers, got {groups!r}") from None
    if len(labels) != n:
        raise ValueError(f"{n} results but {len(labels)} group labels")
    ids = {}
    for i, v in enumerate(labels):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Integral):
            raise ValueError(f"groups[{i}] must be an integer, got {v!r}")
        ids.setdefault(int(v), len(ids))
    return (ctypes.c_int32 * n)(*(ids[int(v)] for v in labels)), len(ids)


def _smoothness(smoothness, groups):
    """None, or the prior's (sigma_roll, sigma_pitch) in degrees, each finite and > 0."""
    if smoothness is None:
        return None
    if groups is None:
        raise ValueError("smoothness needs groups: each group is one sequence of frames")
    pair = tuple(smoothness) if isinstance(smoothness, (tuple, list)) else (smoothness,) * 2
    if len(pair) != 2 or any(isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Real) or not math.isfinite(v) or v <= 0 for v in pair):
        raise ValueError(f"smoothness must be None, a finite number > 0 or a pair of them (degrees), got {smoothness!r}")
    return float(pair[0]), float(pair[1])


def fit_camera(results, principal_point=False, init="fields", mask=None, huber=None, max_iterations=50, groups=None, weights=None,
               smoothness=None):
    """Fit one camera per image to ``results[i]["pred_gravity_original"]`` ([2, H, W] up vectors) and
    ``["pred_latitude_original"]`` ([H, W], degrees), read in place; sizes may differ within one call.  A dict of ground-truth
    fields works too, e.g. ``{"pred_gravity_original": up.permute(2, 0, 1), "pred_latitude_original": lat}``.

    - ``principal_point``: also fit cx_rel and cy_rel (else both are 0).
    - ``init``: "fields" (a closed-form start from the centre of the fields) or "results" (the ParamNet parameters the results
      carry; this reads them on the host, the one case that synchronises).
    - ``mask``: None or a list of bool [H, W] tensors (None entries allowed) that restricts both fields.
    - ``huber``: None (least squares) or the Huber scale delta in radians (``least_squares(loss="huber", f_scale=delta)``).
    - ``max_iterations``: the most cost evaluations per image (1 .. 1000), per group with ``groups``.
    - ``groups``: None (one camera per image) or a sequence of n integers (numpy integers too, not bools): images with equal
      labels were taken with one camera.  They are fitted together, with their own roll and pitch and one shared f_rel (and,
      with ``principal_point``, one cx_rel, cy_rel), relative to each image's own size: a group may mix resolutions only if
      they are scaled copies of one camera (this is not checked).  The shared values are bit-identical across the group;
      ``fit_cost`` is each image's own cost at the group's final point, and ``fit_iterations`` and ``fit_status`` are the
      group's, except that an image with too few valid residuals is dropped from its group with status 2.  The start of the
      shared values is the mean of the members' starts.
    - ``weights``: None, "confidence" (each result's ``pred_gravity_confidence_original`` / ``pred_latitude_confidence_original``,
      what a model built with ``confidence=True`` returns) or a list of n entries, each None or a pair ``(w_up, w_lat)`` of float32
      [H, W] tensors on the results' device (either may be None): per-pixel weights of the up and latitude residuals.  A residual
      counts only where its weight is finite and > 0 (others are dropped as ``mask`` drops them); it adds ``w`` times its
      cost term and has ``w`` times its IRLS weight, and the closed-form start uses only pixels with a usable weight (DESIGN.md
      section 1, "Camera fit").  All-ones weights give the unweighted fit and 0 / 1 weights the fit
      under the matching ``mask``, bit for bit.  Checked on the host, no synchronisation.

    - ``smoothness``: None, or with ``groups`` the prior of a camera track (DESIGN.md section 1, "Camera tracks"): each group is
      one sequence of evenly spaced video frames, its members in index order.  Intrinsics stay shared; roll and pitch are fitted
      jointly along the sequence, each frame's cost divided by its number of residuals, plus a random-walk prior that makes a
      change of sigma degrees between neighbouring frames cost as much as a frame whose fields disagree with its camera by 1
      degree on average.  sigma is one number for both angles or a pair (sigma_roll, sigma_pitch), each finite and > 0.  A
      frame without usable residuals is kept: its angles come from its neighbours, and its ``fit_cost`` is 0.  The roll starts
      are unwrapped along the sequence.  Status 2 applies to the whole sequence (too few residuals, or a shared parameter no
      residual constrains).

    The fields of a model built with ``decode="subbin"`` (continuous, DESIGN.md section 1 "Sub-bin decode") are read as they are:
    nothing here changes for them.

    Returns one dict per image, as 0-dim float64 CUDA tensors in degrees: the keys of a centred (``principal_point=False``:
    ``pred_roll, pred_pitch, pred_vfov, pred_rel_focal, pred_general_vfov, pred_rel_cx, pred_rel_cy``) or uncentred ParamNet
    variant (``pred_roll, pred_pitch, pred_general_vfov, pred_rel_cx, pred_rel_cy, pred_rel_focal``), plus ``fit_cost`` (the
    final cost, radians^2), ``fit_iterations`` (cost evaluations) and ``fit_status`` (0 converged, 1 stopped at
    max_iterations, 2 fewer valid residuals than parameters: NaN parameters), both int32.  Nothing synchronises with the
    device (except ``init="results"``)."""
    if init not in ("fields", "results"):
        raise ValueError(f"init must be 'fields' or 'results', got {init!r}")
    if not isinstance(principal_point, bool):
        raise ValueError(f"principal_point must be a bool, got {principal_point!r}")
    if huber is not None:
        if isinstance(huber, bool) or not isinstance(huber, (int, float)) or not math.isfinite(huber) or huber <= 0:
            raise ValueError(f"huber must be None or a finite number > 0, got {huber!r}")
    if isinstance(max_iterations, bool) or not isinstance(max_iterations, int) or not 1 <= max_iterations <= MAX_ITERATIONS:
        raise ValueError(f"max_iterations must be an integer in 1 .. {MAX_ITERATIONS}, got {max_iterations!r}")
    n = len(results)
    if mask is not None and len(mask) != n:
        raise ValueError(f"{n} results but {len(mask)} masks")
    sigma = _smoothness(smoothness, groups)
    group_of = None if groups is None else _group_ids(groups, n)
    if n == 0:
        return []
    pu, pl, ms, dev = _batch.prediction_fields(results, mask, 3)
    wts = _batch.fit_weights(weights, results, pu, dev)
    starts = _init_from_results(results) if init == "results" else [_NAN_INIT] * n
    L = _native.lib()
    bu, bl, bm = _batch.base(pu), _batch.base(pl), _batch.base(ms)
    flat = [t for e in wts for t in e]
    bw = _batch.base(flat)
    uw = (ctypes.c_int64 * n)(*(_batch.offset(e[0], bw) for e in wts))
    lw = (ctypes.c_int64 * n)(*(_batch.offset(e[1], bw) for e in wts))
    descs = (_native.pf_fit_image * n)()
    for i in range(n):
        d = descs[i]
        d.height, d.width = int(pu[i].shape[0]), int(pu[i].shape[1])
        d.up_offset, d.up_stride[:] = _batch.offset(pu[i], bu), pu[i].stride()
        d.lat_offset = _batch.offset(pl[i], bl)
        d.mask_offset = _batch.offset(ms[i], bm)
        d.init[:] = starts[i]
    with torch.cuda.device(dev):
        if group_of is None:
            ws = _batch.workspace(L.pf_fit_camera_workspace(descs, n), dev)
        elif sigma is not None:
            ws = _batch.workspace(L.pf_fit_camera_sequences_workspace(descs, n, group_of[0], group_of[1]), dev)
        else:
            ws = _batch.workspace(L.pf_fit_camera_groups_workspace(descs, n, group_of[0], group_of[1]), dev)
        params = torch.empty((n, 5), dtype=torch.float64, device=dev)
        cost = torch.empty(n, dtype=torch.float64, device=dev)
        its = torch.empty(n, dtype=torch.int32, device=dev)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        fields = (bu, bl, bm or None, bw or None, uw, lw, int(principal_point), float(huber or 0.0), max_iterations, params.data_ptr(),
                  cost.data_ptr(), its.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(), stream)
        if group_of is None:
            _native.check(L.pf_fit_camera_weighted(dev.index, descs, n, *fields))
        elif sigma is not None:
            _native.check(L.pf_fit_camera_sequences(dev.index, descs, n, group_of[0], group_of[1], *fields[:9], *sigma, *fields[9:]))
        else:
            _native.check(L.pf_fit_camera_groups_weighted(dev.index, descs, n, group_of[0], group_of[1], *fields))
        roll, pitch, f, cx, cy = params.t()
        gv = general_vfov(cx, cy, 1, f, True)
        if principal_point:
            names = ("pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy", "pred_rel_focal")
            cols = torch.stack([roll, pitch, gv, cx, cy, f])
        else:
            vfov = torch.rad2deg(2.0 * torch.atan(0.5 / f))
            names = ("pred_roll", "pred_pitch", "pred_vfov", "pred_rel_focal", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy")
            cols = torch.stack([roll, pitch, vfov, f, gv, cx, cy])
    cols, cost, its, status = cols.unbind(1), cost.unbind(0), its.unbind(0), status.unbind(0)
    out = []
    for i in range(n):
        d = dict(zip(names, cols[i].unbind(0)))
        d.update({"fit_cost": cost[i], "fit_iterations": its[i], "fit_status": status[i]})
        out.append(d)
    return out


def _panorama_ids(panorama_of, n):
    """n integers 0 .. npano - 1, each used -> (int32 ctypes array, npano)."""
    try:
        labels = list(panorama_of)
    except TypeError:
        raise ValueError(f"panorama_of must be a sequence of {n} integers, got {panorama_of!r}") from None
    if len(labels) != n:
        raise ValueError(f"{n} results but {len(labels)} panorama_of entries")
    for i, v in enumerate(labels):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Integral) or int(v) < 0:
            raise ValueError(f"panorama_of[{i}] must be an integer >= 0, got {v!r}")
    npano = max(int(v) for v in labels) + 1
    missing = sorted(set(range(npano)) - {int(v) for v in labels})
    if missing:
        raise ValueError(f"panorama_of names panoramas 0 .. {npano - 1} but none of the views belongs to {missing}")
    return (ctypes.c_int32 * n)(*(int(v) for v in labels)), npano


def fit_panorama(results, views, panorama_of, mask=None, weights=None, huber=None, max_iterations=50, init=None):
    """Fit the tilt of equirectangular panoramas to the fields predicted on views cropped from them (DESIGN.md section 1,
    "Panorama levelling").  View i is ``results[i]`` (fields as ``fit_camera`` reads them, in place), cropped by
    ``panocam.crop_equi_views`` with ``views[i]`` (its ``(vfov, im_w, im_h, azimuth, elevation, roll, ar)`` tuple or dict, whose
    size must be the fields'), from panorama ``panorama_of[i]`` (integers 0 .. npano - 1, each used).  All views of a panorama
    share one unknown, its tilt T = Z(psi) X(phi) (pano roll psi, pano pitch phi; yaw is not observable): a panorama P with tilt
    T shows P(d) = P_level(T d).

    - ``mask``, ``weights`` (including ``"confidence"``), ``huber``, ``max_iterations``: as in ``fit_camera``, per view;
      ``max_iterations`` counts cost evaluations of each panorama.
    - ``init``: None (psi = phi = 0) or one ``(psi, phi)`` pair in degrees per panorama.

    Returns one dict per panorama of CUDA tensors: ``pano_roll`` and ``pano_pitch`` (0-dim float64, degrees, |roll| <= 90 and
    pitch in (-180, 180]), ``pano_up`` ([3], the panorama's up direction g = T^T (0, -1, 0) in its own pixel frame: x right, y
    down, z at azimuth 0), ``rotation`` ([3, 3], the smallest rotation R with R (0, -1, 0) = g: ``rectify.rotate_panoramas``
    with it levels the panorama), ``fit_cost``, ``fit_iterations`` and ``fit_status`` (as ``fit_camera``'s; status 2: NaN
    outputs).  Nothing synchronises with the device; invalid arguments raise before any GPU work."""
    if huber is not None:
        if isinstance(huber, bool) or not isinstance(huber, (int, float)) or not math.isfinite(huber) or huber <= 0:
            raise ValueError(f"huber must be None or a finite number > 0, got {huber!r}")
    if isinstance(max_iterations, bool) or not isinstance(max_iterations, int) or not 1 <= max_iterations <= MAX_ITERATIONS:
        raise ValueError(f"max_iterations must be an integer in 1 .. {MAX_ITERATIONS}, got {max_iterations!r}")
    n = len(results)
    if n == 0:
        raise ValueError("no views")
    vs = [_check_equi_view(v, i) for i, v in enumerate(views)]
    if len(vs) != n:
        raise ValueError(f"{n} results but {len(vs)} views")
    if mask is not None and len(mask) != n:
        raise ValueError(f"{n} results but {len(mask)} masks")
    pano_of, npano = _panorama_ids(panorama_of, n)
    starts = None
    if init is not None:
        starts = [tuple(p) if isinstance(p, (tuple, list, np.ndarray)) else p for p in init]
        if len(starts) != npano or any(not isinstance(p, tuple) or len(p) != 2 for p in starts):
            raise ValueError(f"init must be None or {npano} (pano_roll, pano_pitch) pairs in degrees")
        starts = (ctypes.c_double * (2 * npano))(*(_batch.real(v, "init") for p in starts for v in p))
    pu, pl, ms, dev = _batch.prediction_fields(results, mask, 3)
    for i, v in enumerate(vs):
        if (v[2], v[1]) != (int(pu[i].shape[0]), int(pu[i].shape[1])):
            raise ValueError(f"views[{i}] is {v[2]} x {v[1]} but results[{i}] has fields of {pu[i].shape[0]} x {pu[i].shape[1]}")
    wts = _batch.fit_weights(weights, results, pu, dev)
    L = _native.lib()
    bu, bl, bm = _batch.base(pu), _batch.base(pl), _batch.base(ms)
    bw = _batch.base([t for e in wts for t in e])
    uw = (ctypes.c_int64 * n)(*(_batch.offset(e[0], bw) for e in wts))
    lw = (ctypes.c_int64 * n)(*(_batch.offset(e[1], bw) for e in wts))
    descs = (_native.pf_fit_image * n)()
    crops = (_native.pf_pano_crop * n)()
    for i in range(n):
        d = descs[i]
        d.height, d.width = int(pu[i].shape[0]), int(pu[i].shape[1])
        d.up_offset, d.up_stride[:] = _batch.offset(pu[i], bu), pu[i].stride()
        d.lat_offset = _batch.offset(pl[i], bl)
        d.mask_offset = _batch.offset(ms[i], bm)
        d.init[:] = _NAN_INIT
        vfov, _, _, az, el, roll, ar = vs[i]
        crops[i] = _native.pf_pano_crop(vfov, az, el, roll, ar)
    with torch.cuda.device(dev):
        ws = _batch.workspace(L.pf_fit_panorama_workspace(descs, n, pano_of, npano), dev)
        ang = torch.empty((npano, 2), dtype=torch.float64, device=dev)
        up = torch.empty((npano, 3), dtype=torch.float64, device=dev)
        rot = torch.empty((npano, 3, 3), dtype=torch.float64, device=dev)
        cost = torch.empty(npano, dtype=torch.float64, device=dev)
        its = torch.empty(npano, dtype=torch.int32, device=dev)
        status = torch.empty(npano, dtype=torch.int32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_fit_panorama(dev.index, descs, crops, n, pano_of, npano, bu, bl, bm or None, bw or None, uw, lw, starts,
                                        float(huber or 0.0), max_iterations, ang.data_ptr(), up.data_ptr(), rot.data_ptr(), cost.data_ptr(),
                                        its.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(), stream))
    ang, cost, its, status = ang.unbind(0), cost.unbind(0), its.unbind(0), status.unbind(0)
    return [{"pano_roll": ang[P][0], "pano_pitch": ang[P][1], "pano_up": up[P], "rotation": rot[P], "fit_cost": cost[P],
             "fit_iterations": its[P], "fit_status": status[P]} for P in range(npano)]
