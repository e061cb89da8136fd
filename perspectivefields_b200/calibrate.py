"""Camera parameters from Perspective Fields on the GPU (hand-written sm_90a kernels, csrc/calib.cuh).

``fit_camera`` fits roll, pitch, focal length and optionally the principal point to the up and latitude fields of each image
by Levenberg-Marquardt (this project's rule, DESIGN.md section 1 "Camera fit").  It gives every field-only variant
(``PersNet-360Cities``) the camera parameters its ParamNet-less model lacks, and gives ParamNet variants a geometric check or
refinement of theirs.  Its output has the keys of a ParamNet variant's results, so ``metrics.param_errors``,
``panocam.fields_from_predictions`` and ``viz.draw_from_r_p_f_cx_cy`` take it unchanged.
"""
import math

import torch

from . import _batch, _native
from .panocam import general_vfov, general_vfov_to_focal

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


def fit_camera(results, principal_point=False, init="fields", mask=None, huber=None, max_iterations=50):
    """Fit one camera per image to ``results[i]["pred_gravity_original"]`` ([2, H, W] up vectors) and
    ``["pred_latitude_original"]`` ([H, W], degrees), read in place; sizes may differ within one call.  A dict of ground-truth
    fields works too, e.g. ``{"pred_gravity_original": up.permute(2, 0, 1), "pred_latitude_original": lat}``.

    - ``principal_point``: also fit cx_rel and cy_rel (else both are 0).
    - ``init``: "fields" (a closed-form start from the centre of the fields) or "results" (the ParamNet parameters the results
      carry; this reads them on the host, the one case that synchronises).
    - ``mask``: None or a list of bool [H, W] tensors (None entries allowed) that restricts both fields.
    - ``huber``: None (least squares) or the Huber scale delta in radians (``least_squares(loss="huber", f_scale=delta)``).
    - ``max_iterations``: the most cost evaluations per image (1 .. 1000).

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
    if n == 0:
        return []
    pu, pl, ms, dev = _batch.prediction_fields(results, mask, 3)
    starts = _init_from_results(results) if init == "results" else [_NAN_INIT] * n
    L = _native.lib()
    bu, bl, bm = _batch.base(pu), _batch.base(pl), _batch.base(ms)
    descs = (_native.pf_fit_image * n)()
    for i in range(n):
        d = descs[i]
        d.height, d.width = int(pu[i].shape[0]), int(pu[i].shape[1])
        d.up_offset, d.up_stride[:] = _batch.offset(pu[i], bu), pu[i].stride()
        d.lat_offset = _batch.offset(pl[i], bl)
        d.mask_offset = _batch.offset(ms[i], bm)
        d.init[:] = starts[i]
    with torch.cuda.device(dev):
        ws = _batch.workspace(L.pf_fit_camera_workspace(descs, n), dev)
        params = torch.empty((n, 5), dtype=torch.float64, device=dev)
        cost = torch.empty(n, dtype=torch.float64, device=dev)
        its = torch.empty(n, dtype=torch.int32, device=dev)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_fit_camera(dev.index, descs, n, bu, bl, bm or None, int(principal_point), float(huber or 0.0), max_iterations,
                                      params.data_ptr(), cost.data_ptr(), its.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(),
                                      stream))
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
