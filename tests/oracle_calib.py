"""CPU restatement (float64 numpy) of the camera fit (DESIGN.md section 1, "Camera fit"): the forward model, its analytic
Jacobian, the closed-form start and the Levenberg-Marquardt loop, step for step as csrc/calib.cuh runs them.

Parameters theta = (roll, pitch, s = ln f_rel, cx_rel, cy_rel), angles in radians; with principal_point=False only the first
three are fitted and cx_rel = cy_rel = 0.  Fields: up [H, W, 2] (x, y), latitude [H, W] in degrees, mask bool [H, W] or None.
"""
import math

import numpy as np

LAMBDA0 = 1e-3
COST_RTOL = 1e-12
STEP_RTOL = 1e-12
LAMBDA_MAX = 1e16
UP_MIN = 1e-5
WINDOW = 4          # start window: rows H // 2 - 4 .. H // 2 + 3, the same around W // 2
F_DEFAULT = 1.0 / (2.0 * math.tan(math.radians(60.0) / 2.0))


def lat_grid(n, c):
    """get_lat_general's sample positions linspace(-c, n - c, n) as the kernel evaluates them: x0 + k * step with
    x0 = (-n/2) - (c - n/2), x1 = (n/2) - (c - n/2), step = (x1 - x0) / (n - 1), the last sample exactly x1."""
    x0, x1 = (-n / 2.0) - (c - n / 2.0), (n / 2.0) - (c - n / 2.0)
    step = (x1 - x0) / (n - 1)
    g = np.arange(n, dtype=np.float64) * step + x0
    g[-1] = x1
    return g


def _unpack(theta, H, W):
    r, e, s, cxr, cyr = (list(theta) + [0.0, 0.0])[:5]
    F = math.exp(s) * H
    return r, e, F, (cxr + 0.5) * W, (cyr + 0.5) * H


def model(theta, H, W):
    """(u [H, W, 2] unnormalised up vectors at the pixel centres, latitude [H, W] in radians)."""
    r, e, F, cx, cy = _unpack(theta, H, W)
    sr, cr, se, ce = math.sin(r), math.cos(r), math.sin(e), math.cos(e)
    px = np.arange(W, dtype=np.float64)[None, :] + 0.5
    py = np.arange(H, dtype=np.float64)[:, None] + 0.5
    ux = np.broadcast_to(-sr * ce * F + se * (cx - px), (H, W))
    uy = np.broadcast_to(-cr * ce * F + se * (cy - py), (H, W))
    x = (lat_grid(W, cx) / F)[None, :]
    y = (lat_grid(H, cy) / F)[:, None]
    xw = x * cr - y * sr
    yw = x * (ce * sr) + y * (ce * cr) - se
    zw = x * (se * sr) + y * (se * cr) + ce
    lat = -np.arctan2(yw, np.sqrt(xw * xw + zw * zw))
    return np.stack([ux, uy], axis=2), lat


def jacobians(theta, H, W, P):
    """d(model)/d(theta) analytic: (du [H, W, 2, P], dl [H, W, P]) with the latitude in radians."""
    r, e, F, cx, cy = _unpack(theta, H, W)
    sr, cr, se, ce = math.sin(r), math.cos(r), math.sin(e), math.cos(e)
    px = np.arange(W, dtype=np.float64)[None, :] + 0.5
    py = np.arange(H, dtype=np.float64)[:, None] + 0.5
    sh = (H, W)
    dux = [np.full(sh, -cr * ce * F), np.broadcast_to(sr * se * F + ce * (cx - px), sh), np.full(sh, -sr * ce * F)]
    duy = [np.full(sh, sr * ce * F), np.broadcast_to(cr * se * F + ce * (cy - py), sh), np.full(sh, -cr * ce * F)]
    if P == 5:
        dux += [np.full(sh, se * W), np.zeros(sh)]
        duy += [np.zeros(sh), np.full(sh, se * H)]
    x = np.broadcast_to((lat_grid(W, cx) / F)[None, :], sh)
    y = np.broadcast_to((lat_grid(H, cy) / F)[:, None], sh)
    xw = x * cr - y * sr
    yw = x * (ce * sr) + y * (ce * cr) - se
    zw = x * (se * sr) + y * (se * cr) + ce
    h = np.sqrt(xw * xw + zw * zw)
    n2 = 1.0 + x * x + y * y
    # l = -atan2(yw, h), |ray|^2 = n2:  dl = -(dyw - yw (x dx + y dy) / n2) / h
    dyw = [x * (ce * cr) - y * (ce * sr), -x * (se * sr) - y * (se * cr) - ce, -(yw + se)]
    dxy = [np.zeros(sh), np.zeros(sh), -(x * x + y * y)]
    if P == 5:
        dyw += [-(W / F) * (ce * sr) * np.ones(sh), -(H / F) * (ce * cr) * np.ones(sh)]
        dxy += [-x * (W / F), -y * (H / F)]
    dl = np.stack([-(a - yw * b / n2) / h for a, b in zip(dyw, dxy)], axis=2)
    return np.stack([np.stack(dux, axis=2), np.stack(duy, axis=2)], axis=2), dl


def residuals(theta, up, lat_deg, mask, P):
    """(r_u, J_u, r_l, J_l) over the valid pixels: r_u = atan2(u x p, u . p) (model to prediction), r_l = rad(lat) - l."""
    H, W = lat_deg.shape
    u, l = model(theta, H, W)
    du, dl = jacobians(theta, H, W, P)
    m = np.ones((H, W), bool) if mask is None else mask.astype(bool)
    p = up.astype(np.float64)
    px, py = p[..., 0], p[..., 1]
    with np.errstate(invalid="ignore", over="ignore"):
        u2 = u[..., 0] ** 2 + u[..., 1] ** 2
        vu = m & np.isfinite(px) & np.isfinite(py) & (np.sqrt(px * px + py * py) > UP_MIN) & (u2 > 0)
        lp = lat_deg.astype(np.float64)
        vl = m & np.isfinite(lp)
    ux, uy = u[..., 0][vu], u[..., 1][vu]
    qx, qy = px[vu], py[vu]
    ru = np.arctan2(ux * qy - uy * qx, ux * qx + uy * qy)
    # r_u = angle(p) - angle(u):  dr_u = -(ux duy - uy dux) / |u|^2
    Ju = -(ux[:, None] * du[..., 1, :][vu] - uy[:, None] * du[..., 0, :][vu]) / u2[vu][:, None]
    rl = lp[vl] * (math.pi / 180.0) - l[vl]
    Jl = -dl[vl]
    return ru, Ju, rl, Jl


def rho(r, huber):
    """delta^2 rho((r / delta)^2) and the IRLS weight rho'((r / delta)^2)."""
    a = np.abs(r)
    if huber is None:
        return r * r, np.ones_like(r)
    lin = a > huber
    return np.where(lin, 2.0 * huber * a - huber * huber, r * r), np.where(lin, huber / np.where(lin, a, 1.0), 1.0)


def evaluate(theta, up, lat_deg, mask, P, huber):
    """(C, A [P, P], g [P], count): C = 1/2 sum delta^2 rho((r/delta)^2), A = sum w J^T J, g = sum w J^T r."""
    ru, Ju, rl, Jl = residuals(theta, up, lat_deg, mask, P)
    r = np.concatenate([ru, rl])
    J = np.concatenate([Ju, Jl])
    c, w = rho(r, huber)
    return 0.5 * c.sum(), (J * w[:, None]).T @ J, (J * w[:, None]).T @ r, r.size


def start(up, lat_deg, mask):
    """Closed-form start (roll, pitch, ln f_rel) from the window of 8 x 8 pixels around (H // 2, W // 2)."""
    H, W = lat_deg.shape
    i0, j0 = max(H // 2 - WINDOW, 0), max(W // 2 - WINDOW, 0)
    i1, j1 = min(H // 2 + WINDOW, H), min(W // 2 + WINDOW, W)
    m = np.ones((H, W), bool) if mask is None else mask.astype(bool)
    p = up.astype(np.float64)
    lp = lat_deg.astype(np.float64) * (math.pi / 180.0)
    sx = sy = 0.0
    nu = nl = ng = 0
    sl = sg = 0.0
    for i in range(i0, i1):
        for j in range(j0, j1):
            if not m[i, j]:
                continue
            x, y = p[i, j]
            if math.isfinite(x) and math.isfinite(y) and math.sqrt(x * x + y * y) > UP_MIN:
                nn = math.sqrt(x * x + y * y)
                sx += x / nn
                sy += y / nn
                nu += 1
            if math.isfinite(lp[i, j]):
                sl += lp[i, j]
                nl += 1
                if 0 < i < H - 1 and 0 < j < W - 1:
                    a, b, c, d = lp[i, j + 1], lp[i, j - 1], lp[i + 1, j], lp[i - 1, j]
                    if m[i, j + 1] and m[i, j - 1] and m[i + 1, j] and m[i - 1, j] and all(math.isfinite(v) for v in (a, b, c, d)):
                        gx, gy = 0.5 * (a - b), 0.5 * (c - d)
                        sg += math.sqrt(gx * gx + gy * gy)
                        ng += 1
    roll = math.atan2(-sx, -sy) if nu else 0.0
    pitch = sl / nl if nl else 0.0
    f = 1.0 / (H * (sg / ng)) if ng and sg > 0 else F_DEFAULT
    return roll, pitch, math.log(f)


def cholesky_solve(M, b):
    """(M) x = b by Cholesky in float64; None when M is not positive definite."""
    P = M.shape[0]
    L = np.zeros_like(M)
    for i in range(P):
        for j in range(i + 1):
            s = M[i, j] - sum(L[i, k] * L[j, k] for k in range(j))
            if i == j:
                if not s > 0:
                    return None
                L[i, i] = math.sqrt(s)
            else:
                L[i, j] = s / L[j, j]
    y = np.zeros(P)
    for i in range(P):
        y[i] = (b[i] - sum(L[i, k] * y[k] for k in range(i))) / L[i, i]
    x = np.zeros(P)
    for i in reversed(range(P)):
        x[i] = (y[i] - sum(L[k, i] * x[k] for k in range(i + 1, P))) / L[i, i]
    return x


def normalise(theta):
    """(r, e) and (r + pi, pi - e) give identical fields: the one with |pitch| <= pi/2, roll in (-pi, pi]."""
    r, e = theta[0], theta[1]
    wrap = lambda a: a - 2.0 * math.pi * math.ceil((a - math.pi) / (2.0 * math.pi))   # (-pi, pi]
    e = wrap(e)
    if abs(e) > math.pi / 2:
        e = wrap(math.pi - e)
        r = r + math.pi
    return [wrap(r), e] + list(theta[2:])


def fit(up, lat_deg, mask=None, principal_point=False, huber=None, max_iterations=50, init=None):
    """Returns dict(theta (normalised, 5 entries, ln f_rel third), params (roll deg, pitch deg, f_rel, cx_rel, cy_rel), cost,
    iterations (cost evaluations), status, start (the unnormalised start theta, P entries))."""
    P = 5 if principal_point else 3
    if init is None:
        th = list(start(up, lat_deg, mask)) + [0.0, 0.0]
    else:
        th = [init[0], init[1], math.log(init[2]), init[3] if principal_point else 0.0, init[4] if principal_point else 0.0]
    theta = np.array(th[:P], np.float64)
    st = theta.copy()
    C, A, g, count = evaluate(theta, up, lat_deg, mask, P, huber)
    evals = 1
    if count < P or np.any(np.diag(A) == 0):
        return {"theta": [math.nan] * 5, "params": [math.nan] * 5, "cost": math.nan, "iterations": evals, "status": 2, "start": st}
    lam = LAMBDA0
    status = None
    while status is None:
        delta = None
        while lam <= LAMBDA_MAX:
            M = A + lam * np.diag(np.diag(A))
            delta = cholesky_solve(M, -g)
            if delta is not None:
                break
            lam *= 10.0
        if delta is None:
            status = 0
            break
        if np.all(np.abs(delta) <= STEP_RTOL * (1.0 + np.abs(theta))):
            status = 0
            break
        if evals >= max_iterations:
            status = 1
            break
        cand = theta + delta
        Cc, Ac, gc, _ = evaluate(cand, up, lat_deg, mask, P, huber)
        evals += 1
        if Cc < C:
            done = C - Cc <= COST_RTOL * C
            theta, C, A, g = cand, Cc, Ac, gc
            lam /= 10.0
            if done:
                status = 0
        else:
            lam *= 10.0
            if lam > LAMBDA_MAX:
                status = 0
    full = normalise(list(theta) + [0.0] * (5 - P))
    params = [math.degrees(full[0]), math.degrees(full[1]), math.exp(full[2]), full[3], full[4]]
    return {"theta": full, "params": params, "cost": C, "iterations": evals, "status": status, "start": st}


def cost_at(theta, up, lat_deg, mask=None, principal_point=False, huber=None):
    """C at theta = (roll, pitch, ln f_rel[, cx_rel, cy_rel])."""
    P = 5 if principal_point else 3
    return evaluate(np.asarray(theta, np.float64)[:P], up, lat_deg, mask, P, huber)[0]


def params_to_theta(roll_deg, pitch_deg, f_rel, cx_rel=0.0, cy_rel=0.0):
    return [math.radians(roll_deg), math.radians(pitch_deg), math.log(f_rel), cx_rel, cy_rel]


def noisy_fields(rng, theta, H, W, up_noise_deg=2.0, lat_noise_deg=1.0, outliers=0.02, holes=True):
    """Exact model fields with angular noise, a fraction of gross outliers, NaN holes and zero-length predictions.
    Returns (up [H, W, 2] float32, latitude [H, W] float32 degrees)."""
    u, l = model(theta, H, W)
    ang = np.arctan2(u[..., 1], u[..., 0]) + np.radians(up_noise_deg) * rng.standard_normal((H, W))
    lat = np.degrees(l) + lat_noise_deg * rng.standard_normal((H, W))
    out = rng.random((H, W)) < outliers
    ang[out] = rng.uniform(-math.pi, math.pi, out.sum())
    out = rng.random((H, W)) < outliers
    lat[out] = rng.uniform(-90, 90, out.sum())
    up = np.stack([np.cos(ang), np.sin(ang)], axis=2)
    if holes:
        up[: H // 9, : W // 6] = 0.0                    # the classification decoder's "no direction" bin
        up[H // 3, :] = np.nan
        lat[-3:, : W // 4] = np.nan
    return up.astype(np.float32), lat.astype(np.float32)
