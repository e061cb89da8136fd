"""CPU restatement (float64 numpy) of panorama levelling (DESIGN.md section 1, "Panorama levelling"): the camera-fit model
written in terms of the world up direction v, the tilt fit over the views of one panorama (Levenberg-Marquardt on (psi, phi),
step for step as csrc/calib.cuh runs it), the output normalisation and rotation, and the rotation warp of csrc/equi.cuh.

Built on tests/oracle_calib.py (grid, residual rules, Huber, Cholesky, stop rules) and tests/oracle_equi.py (the crop rule's
sampler).  Angles in radians unless a name says degrees.
"""
import math

import numpy as np

import oracle_calib as oc
import oracle_equi as oe

N = np.array([0.0, -1.0, 0.0])      # world up: y points down


def Rz(r):
    c, s = math.cos(r), math.sin(r)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def Rx(e):
    c, s = math.cos(e), math.sin(e)
    return np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])


def Ry(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])


def crop_rotation(azimuth, elevation, roll):
    """A = Y(a) X(e) Z(r) of a crop_equi_views view, angles in degrees (the crop rule's deg / 180 * pi)."""
    rad = lambda d: d / 180 * math.pi
    return Ry(rad(azimuth)) @ Rx(rad(elevation)) @ Rz(rad(roll))


def decompose(M):
    """M = Y(a) X(e) Z(r) -> (a, e, r) in degrees."""
    e = math.asin(max(-1.0, min(1.0, -M[1, 2])))
    return math.degrees(math.atan2(M[0, 2], M[2, 2])), math.degrees(e), math.degrees(math.atan2(M[1, 0], M[1, 1]))


def tilt(psi, phi):
    """T = Z(psi) X(phi): P(d) = P_level(T d)."""
    return Rz(psi) @ Rx(phi)


def gravity(theta):
    """g = T^T n and dg / dtheta ([3, 2])."""
    sp, cp, sf, cf = math.sin(theta[0]), math.cos(theta[0]), math.sin(theta[1]), math.cos(theta[1])
    g = np.array([-sp, -cp * cf, cp * sf])
    dg = np.array([[-cp, 0.0], [sp * cf, cp * sf], [-sp * sf, cp * cf]])
    return g, dg


def crop_focal(vfov, im_w, ar):
    """The crop's focal length in pixels, pf_equi_views' expressions."""
    fov_x = 2 * math.atan(math.tan(vfov * math.pi / 180.0 / 2) * ar) * 180 / math.pi
    return im_w / (2 * math.tan(fov_x * math.pi / 180 / 2))


def level_up(elevation, roll):
    """v of a level camera at (pitch e, roll r): (-sin r cos e, -cos r cos e, sin e)."""
    return np.array([-math.sin(roll) * math.cos(elevation), -math.cos(roll) * math.cos(elevation), math.sin(elevation)])


def model(v, H, W, F):
    """(u [H, W, 2] at the pixel centres, latitude [H, W] radians) for world up v, focal F (pixels), centred principal point."""
    cx, cy = W / 2.0, H / 2.0
    px = np.arange(W, dtype=np.float64)[None, :] + 0.5
    py = np.arange(H, dtype=np.float64)[:, None] + 0.5
    ux = np.broadcast_to(F * v[0] + v[2] * (cx - px), (H, W))
    uy = np.broadcast_to(F * v[1] + v[2] * (cy - py), (H, W))
    x = np.broadcast_to((oc.lat_grid(W, cx) / F)[None, :], (H, W))
    y = np.broadcast_to((oc.lat_grid(H, cy) / F)[:, None], (H, W))
    s = v[0] * x + v[1] * y + v[2]
    q = np.stack([v[1] - v[2] * y, v[2] * x - v[0], v[0] * y - v[1] * x])
    h = np.sqrt((q * q).sum(0))
    return np.stack([ux, uy], axis=2), np.arctan2(s, h), (x, y, h)


def residuals(v, F, up, lat_deg, mask, weights=(None, None)):
    """(r, J [., 3], w) over the used residuals of one view: r_u then r_l as oracle_calib defines them, J with respect to v,
    w the residual weights (1 without weight maps)."""
    H, W = lat_deg.shape
    u, l, (x, y, h) = model(v, H, W, F)
    cx, cy = W / 2.0, H / 2.0
    ex = np.broadcast_to(cx - (np.arange(W)[None, :] + 0.5), (H, W))
    ey = np.broadcast_to(cy - (np.arange(H)[:, None] + 0.5), (H, W))
    m = np.ones((H, W), bool) if mask is None else mask.astype(bool)
    p = up.astype(np.float64)
    wu = np.ones((H, W)) if weights[0] is None else weights[0].astype(np.float64)
    wl = np.ones((H, W)) if weights[1] is None else weights[1].astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        u2 = u[..., 0] ** 2 + u[..., 1] ** 2
        vu = m & np.isfinite(p[..., 0]) & np.isfinite(p[..., 1]) & (np.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2) > oc.UP_MIN) & (u2 > 0)
        vu &= np.isfinite(wu) & (wu > 0)
        lp = lat_deg.astype(np.float64)
        vl = m & np.isfinite(lp) & np.isfinite(wl) & (wl > 0)
    ux, uy, qx, qy = u[..., 0][vu], u[..., 1][vu], p[..., 0][vu], p[..., 1][vu]
    ru = np.arctan2(ux * qy - uy * qx, ux * qx + uy * qy)
    # dux / dv = (F, 0, ex), duy / dv = (0, F, ey); dr_u = -(ux duy - uy dux) / |u|^2
    Ju = np.stack([uy * F, -ux * F, uy * ex[vu] - ux * ey[vu]], axis=1) / u2[vu][:, None]
    rl = lp[vl] * (math.pi / 180.0) - l[vl]
    Jl = -np.stack([x[vl], y[vl], np.ones(vl.sum())], axis=1) / h[vl][:, None]
    return np.concatenate([ru, rl]), np.concatenate([Ju, Jl]), np.concatenate([wu[vu], wl[vl]])


def evaluate(theta, views, huber):
    """(C, A [2, 2], g [2], count) of one panorama at theta: views = list of dicts (A: crop rotation, F, up, lat, mask,
    weights).  Per view the sums with respect to v, chained through D = A^T dg / dtheta."""
    g, dg = gravity(theta)
    C, A, gg, count = 0.0, np.zeros((2, 2)), np.zeros(2), 0
    for vw in views:
        v = vw["A"].T @ g
        r, J, w = residuals(v, vw["F"], vw["up"], vw["lat"], vw.get("mask"), vw.get("weights", (None, None)))
        c, wi = oc.rho(r, huber)
        D = vw["A"].T @ dg
        Av, gv = (J * (w * wi)[:, None]).T @ J, (J * (w * wi)[:, None]).T @ r
        C += 0.5 * (w * c).sum()
        A += D.T @ Av @ D
        gg += D.T @ gv
        count += r.size
    return C, A, gg, count


def normalise(theta):
    """(psi, phi) and (pi - psi, phi + pi) give the same g: the pair with |psi| <= pi/2 and phi in (-pi, pi]."""
    wrap = lambda a: a - 2.0 * math.pi * math.ceil((a - math.pi) / (2.0 * math.pi))
    psi, phi = wrap(theta[0]), theta[1]
    if abs(psi) > math.pi / 2:
        psi, phi = wrap(math.pi - psi), phi + math.pi
    return psi, wrap(phi)


def rotation_to(g):
    """The smallest rotation R with R n = g: Rodrigues about n x g by the angle between them (180 degrees about x for g = -n)."""
    w = np.cross(N, g)
    s, c = np.linalg.norm(w), float(N @ g)
    if s == 0.0:
        return np.eye(3) if c > 0 else np.diag([1.0, -1.0, -1.0])
    k = w / s
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    a = math.atan2(s, c)
    return np.eye(3) + math.sin(a) * K + (1.0 - math.cos(a)) * K @ K


def fit(views, huber=None, max_iterations=50, init=(0.0, 0.0)):
    """One panorama's fit -> dict(theta (normalised, radians), angles (degrees), up, rotation, cost, iterations, status)."""
    theta = np.array(init, np.float64)
    C, A, g, count = evaluate(theta, views, huber)
    evals = 1
    nan = {"theta": [math.nan] * 2, "angles": [math.nan] * 2, "up": [math.nan] * 3, "rotation": np.full((3, 3), math.nan),
           "cost": math.nan, "iterations": evals, "status": 2}
    if count < 2 or np.any(np.diag(A) == 0):
        return nan
    lam, status = oc.LAMBDA0, None
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
        Cc, Ac, gc, _ = evaluate(cand, views, huber)
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
    th = normalise(theta)
    up = gravity(th)[0]
    return {"theta": list(th), "angles": [math.degrees(th[0]), math.degrees(th[1])], "up": up, "rotation": rotation_to(up), "cost": C,
            "iterations": evals, "status": status}


def panorama_map(Hp, Wp, R):
    """The warp's input position (u, v) of every output pixel, float64 [Hp, Wp] each: out(d) = P(R d)."""
    j = np.arange(Wp, dtype=np.float64)[None, :]
    i = np.arange(Hp, dtype=np.float64)[:, None]
    theta = 2 * np.pi * j / Wp - np.pi
    phi = np.pi / 2 - np.pi * i / Hp
    d = np.stack(np.broadcast_arrays(np.cos(phi) * np.sin(theta), -np.sin(phi), np.cos(phi) * np.cos(theta)))
    x, y, z = np.einsum("rc,chw->rhw", np.asarray(R, np.float64), d)
    n = np.sqrt(x * x + y * y + z * z)
    return (np.arctan2(x, z) + np.pi) * (Wp / (2 * np.pi)), (np.pi / 2 + np.arcsin(y / n)) * (Hp / np.pi)


def rotate(pano, R, mode="bilinear"):
    """(the rotated panorama in the input dtype, float64 sample [Hp, Wp, C], u, v): uint8 rounded to nearest and clamped."""
    pano = np.asarray(pano)
    chw = pano.transpose(2, 0, 1) if pano.ndim == 3 else pano[None]
    u, v = panorama_map(chw.shape[1], chw.shape[2], R)
    s = oe.sample(chw, u, v, mode)
    out = np.clip(np.rint(s), 0, 255).astype(np.uint8) if pano.dtype == np.uint8 else s.astype(pano.dtype)
    out = out.transpose(1, 2, 0)
    return (out[:, :, 0] if pano.ndim == 2 else out), s.transpose(1, 2, 0), u, v
