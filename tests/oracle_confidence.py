"""CPU restatement (float64 numpy) of the head confidence and of the weighted camera fit (DESIGN.md section 1, "Head confidence"
and "Camera fit"), built on tests/oracle_calib.py's model, Jacobians, start and solver; the weighted fit with shared intrinsics
is tests/oracle_calib_shared.py's joint solver on these weighted evaluations (fit_groups).

Weights: wu / wl float [H, W] maps of the up / latitude residuals or None (weight 1).  A residual counts where it is valid
unweighted and its weight is finite and > 0; it adds w delta^2 rho((r / delta)^2) to 2 C and has the IRLS weight w rho'.
"""
import math

import numpy as np

import oracle_calib as oc


def confidence(logits, axis=0):
    """max_c softmax(logits)_c = 1 / sum_c exp(l_c - l_max) over ``axis``, in float64."""
    l = np.asarray(logits, np.float64)
    return 1.0 / np.exp(l - l.max(axis=axis, keepdims=True)).sum(axis=axis)


def usable(w, shape):
    """The pixels whose weight keeps their residual (all of them for None) and the weights there (1 for None)."""
    if w is None:
        return np.ones(shape, bool), np.ones(shape)
    w = np.asarray(w, np.float64)
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(w) & (w > 0)
    return ok, np.where(ok, w, 0.0)


def residuals(theta, up, lat_deg, mask, P, wu=None, wl=None):
    """oracle_calib.residuals plus the weights: (r_u, J_u, v_u, r_l, J_l, v_l) over the residuals that count."""
    H, W = lat_deg.shape
    m = np.ones((H, W), bool) if mask is None else mask.astype(bool)
    mu, vu = usable(wu, (H, W))
    ml, vl = usable(wl, (H, W))
    u, l = oc.model(theta, H, W)
    du, dl = oc.jacobians(theta, H, W, P)
    p = up.astype(np.float64)
    px, py = p[..., 0], p[..., 1]
    with np.errstate(invalid="ignore", over="ignore"):
        u2 = u[..., 0] ** 2 + u[..., 1] ** 2
        su = m & mu & np.isfinite(px) & np.isfinite(py) & (np.sqrt(px * px + py * py) > oc.UP_MIN) & (u2 > 0)
        lp = lat_deg.astype(np.float64)
        sl = m & ml & np.isfinite(lp)
    ux, uy = u[..., 0][su], u[..., 1][su]
    qx, qy = px[su], py[su]
    ru = np.arctan2(ux * qy - uy * qx, ux * qx + uy * qy)
    Ju = -(ux[:, None] * du[..., 1, :][su] - uy[:, None] * du[..., 0, :][su]) / u2[su][:, None]
    rl = lp[sl] * (math.pi / 180.0) - l[sl]
    Jl = -dl[sl]
    return ru, Ju, vu[su], rl, Jl, vl[sl]


def evaluate(theta, up, lat_deg, mask, P, huber, wu=None, wl=None):
    """(C, A, g, count) of the weighted cost: C = 1/2 sum v delta^2 rho, A = sum v rho' J^T J, g = sum v rho' J^T r."""
    ru, Ju, vu, rl, Jl, vl = residuals(theta, up, lat_deg, mask, P, wu, wl)
    r = np.concatenate([ru, rl])
    J = np.concatenate([Ju, Jl])
    v = np.concatenate([vu, vl])
    c, w = oc.rho(r, huber)
    c, w = v * c, v * w
    return 0.5 * c.sum(), (J * w[:, None]).T @ J, (J * w[:, None]).T @ r, r.size


def cost(theta, up, lat_deg, mask, P, huber, wu=None, wl=None):
    return evaluate(np.asarray(theta, np.float64)[:P], up, lat_deg, mask, P, huber, wu, wl)[0]


def start(up, lat_deg, mask, wu=None, wl=None):
    """The closed-form start on the pixels with usable weights: the up weight for the roll term, the latitude weight for the pitch
    and gradient terms (the gradient's four neighbours included)."""
    H, W = lat_deg.shape
    m = np.ones((H, W), bool) if mask is None else mask.astype(bool)
    roll = oc.start(up, lat_deg, m & usable(wu, (H, W))[0])[0]
    _, pitch, s = oc.start(up, lat_deg, m & usable(wl, (H, W))[0])
    return roll, pitch, s


def fit(up, lat_deg, mask=None, principal_point=False, huber=None, max_iterations=50, init=None, wu=None, wl=None):
    """oracle_calib.fit with weights: the same Levenberg-Marquardt loop on the weighted cost; the same result dict."""
    P = 5 if principal_point else 3
    if init is None:
        th = list(start(up, lat_deg, mask, wu, wl)) + [0.0, 0.0]
    else:
        th = [init[0], init[1], math.log(init[2]), init[3] if principal_point else 0.0, init[4] if principal_point else 0.0]
    theta = np.array(th[:P], np.float64)
    st = theta.copy()
    C, A, g, count = evaluate(theta, up, lat_deg, mask, P, huber, wu, wl)
    evals = 1
    if count < P or np.any(np.diag(A) == 0):
        return {"theta": [math.nan] * 5, "params": [math.nan] * 5, "cost": math.nan, "iterations": evals, "status": 2, "start": st}
    lam = oc.LAMBDA0
    status = None
    while status is None:
        delta = None
        while lam <= oc.LAMBDA_MAX:
            delta = oc.cholesky_solve(A + lam * np.diag(np.diag(A)), -g)
            if delta is not None:
                break
            lam *= 10.0
        if delta is None or np.all(np.abs(delta) <= oc.STEP_RTOL * (1.0 + np.abs(theta))):
            status = 0
            break
        if evals >= max_iterations:
            status = 1
            break
        cand = theta + delta
        Cc, Ac, gc, _ = evaluate(cand, up, lat_deg, mask, P, huber, wu, wl)
        evals += 1
        if Cc < C:
            done = C - Cc <= oc.COST_RTOL * C
            theta, C, A, g = cand, Cc, Ac, gc
            lam /= 10.0
            if done:
                status = 0
        else:
            lam *= 10.0
            if lam > oc.LAMBDA_MAX:
                status = 0
    full = oc.normalise(list(theta) + [0.0] * (5 - P))
    params = [math.degrees(full[0]), math.degrees(full[1]), math.exp(full[2]), full[3], full[4]]
    return {"theta": full, "params": params, "cost": C, "iterations": evals, "status": status, "start": st}


class _WeightedCalib:
    """oracle_calib's interface as oracle_calib_shared calls it, with (mask, wu, wl) in the mask slot: its evaluations and starts
    become the weighted ones above."""

    def __getattr__(self, name):
        return getattr(oc, name)

    @staticmethod
    def evaluate(theta, up, lat_deg, packed, P, huber):
        mask, wu, wl = packed
        return evaluate(theta, up, lat_deg, mask, P, huber, wu, wl)

    @staticmethod
    def start(up, lat_deg, packed):
        mask, wu, wl = packed
        return start(up, lat_deg, mask, wu, wl)


def fit_groups(ups, lats, masks, weights, groups, principal_point=False, huber=None, max_iterations=50):
    """oracle_calib_shared.fit_groups with weights[i] = (wu, wl) (either None) per image: the grouped fit of the weighted cost."""
    import oracle_calib_shared as ocs

    packed = [(None if masks is None else masks[i], w[0], w[1]) for i, w in enumerate(weights)]
    saved = ocs.oc
    ocs.oc = _WeightedCalib()
    try:
        return ocs.fit_groups(ups, lats, packed, groups, principal_point, huber, max_iterations)
    finally:
        ocs.oc = saved
