"""CPU restatement (float64 numpy) of the upright warp (DESIGN.md section 1, "Upright warp"), in the order of operations of
csrc/rectify.cuh: the input and output cameras, the "fill" focal length, the map, both samplers and the status.
TEST INFRASTRUCTURE (oracle).

Cameras are (roll, pitch, general vfov) in degrees plus (cx_rel, cy_rel), as ``upright`` reads them from ParamNet results.
"""
import math

import numpy as np

from perspectivefields_b200.panocam import general_vfov_to_focal

D2R, R2D = math.pi / 180.0, 180.0 / math.pi


def rz(r):
    """R_z(r)(x, y, z) = (x cos r - y sin r, x sin r + y cos r, z)."""
    c, s = math.cos(r), math.sin(r)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def rx(e):
    """R_x(e)(x, y, z) = (x, y cos e - z sin e, y sin e + z cos e)."""
    c, s = math.cos(e), math.sin(e)
    return np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])


def input_camera(params, H, W):
    """(r, e radians, f_rel, F, cx, cy) or None when the parameters are unusable (status 2)."""
    roll, pitch, gv, cxr, cyr = [float(v) for v in params]
    if not all(math.isfinite(v) for v in (roll, pitch, gv, cxr, cyr)) or not 0.0 < gv < 180.0:
        return None
    f = float(general_vfov_to_focal(cxr, cyr, 1, gv, True))
    if not (math.isfinite(f) and f > 0.0):
        return None
    return roll * D2R, pitch * D2R, f, f * H, (cxr + 0.5) * W, (cyr + 0.5) * H


def fill_focal(R, F, cx, cy, H, W, Ho, Wo):
    """(1 / t_max: the least output focal length that keeps the four canvas corners inside the input, 0 when every focal length
    does; None when the output's principal ray is not strictly inside the input's cone)."""
    normals = np.array([[F, 0.0, cx], [-F, 0.0, W - cx], [0.0, F, cy], [0.0, -F, H - cy]])
    p = R[:, 2]
    np_ = normals @ p
    if not np.all(np_ > 0.0):
        return None
    tmax = math.inf
    for a in (-Wo / 2.0, Wo / 2.0):
        for b in (-Ho / 2.0, Ho / 2.0):
            q = R[:, 0] * a + R[:, 1] * b
            nq = normals @ q
            for k in range(4):
                if nq[k] < 0.0:
                    tmax = min(tmax, np_[k] / -nq[k])
    return 0.0 if tmax == math.inf else 1.0 / tmax


def setup(params, H, W, Ho, Wo, keep_pitch=False, focal="same"):
    """dict(status, M (3 x 3: input (X, Y, Z) = M (x', y', 1) at output pixel-centre coordinates, NaN for status 2), Fo,
    camera (roll, pitch, general vfov in degrees, cx_rel, cy_rel of the output), and the input camera's (r, e, f_rel, F, cx, cy))."""
    cam = input_camera(params, H, W)
    if cam is None:
        return {"status": 2, "M": np.full((3, 3), math.nan), "Fo": math.nan, "camera": [math.nan] * 5, "input": None}
    r, e, f, F, cx, cy = cam
    eo = e if keep_pitch else 0.0
    R = rz(-r) @ rx(eo - e)
    Fo = f * Ho
    status = 0
    if focal == "fill":
        ff = fill_focal(R, F, cx, cy, H, W, Ho, Wo)
        if ff is None:
            status = 1
        else:
            Fo = max(Fo, ff)
    elif focal != "same":
        Fo = Ho / (2.0 * math.tan(float(focal) * D2R / 2.0))
    K = np.array([[F, 0.0, cx], [0.0, F, cy], [0.0, 0.0, 1.0]])
    Koi = np.array([[1.0 / Fo, 0.0, -(Wo / 2.0) / Fo], [0.0, 1.0 / Fo, -(Ho / 2.0) / Fo], [0.0, 0.0, 1.0]])
    camera = [0.0, eo * R2D, 2.0 * math.atan(Ho / (2.0 * Fo)) * R2D, 0.0, 0.0]
    return {"status": status, "M": K @ R @ Koi, "Fo": Fo, "camera": camera, "input": cam, "R": R}


def positions(M, Ho, Wo, H, W):
    """(u, v, valid) float64 [Ho, Wo]: the input pixel-centre position of every output pixel centre."""
    y, x = np.meshgrid(np.arange(Ho, dtype=np.float64) + 0.5, np.arange(Wo, dtype=np.float64) + 0.5, indexing="ij")
    X = M[0, 0] * x + M[0, 1] * y + M[0, 2]
    Y = M[1, 0] * x + M[1, 1] * y + M[1, 2]
    Z = M[2, 0] * x + M[2, 1] * y + M[2, 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        u, v = X / Z, Y / Z
        valid = (Z > 0) & (u >= 0) & (u <= W) & (v >= 0) & (v <= H)
    return u, v, valid


def sample(img, u, v, valid, mode, fill):
    """img uint8 [H, W, C] -> uint8 [Ho, Wo, C]: bilinear in index space (u - 1/2, v - 1/2) with clamped taps, float64 weights,
    rounded half to even; or the nearest pixel floor(index + 1/2), clamped; ``fill`` (C values) where not valid."""
    H, W, C = img.shape
    uu, vv = np.where(valid, u, 0.5), np.where(valid, v, 0.5)
    s, t = uu - 0.5, vv - 0.5
    im = img.astype(np.float64)
    if mode == "nearest":
        xi = np.clip(np.floor(s + 0.5), 0, W - 1).astype(np.int64)
        yi = np.clip(np.floor(t + 0.5), 0, H - 1).astype(np.int64)
        out = img[yi, xi]
    elif mode == "bilinear":
        fs, ft = np.floor(s), np.floor(t)
        fx, fy = (s - fs)[..., None], (t - ft)[..., None]
        x0, x1 = np.clip(fs, 0, W - 1).astype(np.int64), np.clip(fs + 1, 0, W - 1).astype(np.int64)
        y0, y1 = np.clip(ft, 0, H - 1).astype(np.int64), np.clip(ft + 1, 0, H - 1).astype(np.int64)
        top = im[y0, x0] * (1.0 - fx) + im[y0, x1] * fx
        bot = im[y1, x0] * (1.0 - fx) + im[y1, x1] * fx
        out = np.clip(np.rint(top * (1.0 - fy) + bot * fy), 0, 255).astype(np.uint8)
    else:
        raise ValueError(f"unknown mode {mode!r}")
    return np.where(valid[..., None], out, np.asarray(fill, np.uint8).reshape(1, 1, C))


def upright(img, params, keep_pitch=False, focal="same", size=None, mode="bilinear", fill=0):
    """One image ([H, W] or [H, W, C] uint8) -> dict(im, mask, map (float32 [Ho, Wo, 2], NaN where invalid), camera, status,
    Fo, M, u, v (float64))."""
    img = np.asarray(img)
    flat = img.ndim == 2
    im3 = img[..., None] if flat else img
    H, W, C = im3.shape
    Ho, Wo = (H, W) if size is None else size
    fills = [fill] * C if np.isscalar(fill) else list(fill)
    st = setup(params, H, W, Ho, Wo, keep_pitch, focal)
    if st["status"] == 2:
        u = v = np.full((Ho, Wo), math.nan)
        valid = np.zeros((Ho, Wo), bool)
    else:
        u, v, valid = positions(st["M"], Ho, Wo, H, W)
    out = sample(im3, u, v, valid, mode, fills)
    xy = np.where(valid[..., None], np.stack([u, v], axis=2), math.nan).astype(np.float32)
    return {"im": out[..., 0] if flat else out, "mask": valid, "map": xy, "camera": st["camera"], "status": st["status"],
            "Fo": st["Fo"], "M": st["M"], "u": u, "v": v}


# ---------------------------------------------------------------- continuous camera model (the fields at any position)
def world_ray(x, y, r, e, F, cx, cy):
    """R_x(e) R_z(r) ((x - cx) / F, (y - cy) / F, 1) at pixel-centre positions x, y (arrays) -> (xw, yw, zw)."""
    a, b = (x - cx) / F, (y - cy) / F
    sr, cr, se, ce = math.sin(r), math.cos(r), math.sin(e), math.cos(e)
    xr, yr = a * cr - b * sr, a * sr + b * cr
    return xr, yr * ce - se, yr * se + ce


def latitude(x, y, r, e, F, cx, cy):
    """The latitude (radians) of the ray through the position (x, y): -atan2(yw, hypot(xw, zw)), y pointing down."""
    xw, yw, zw = world_ray(x, y, r, e, F, cx, cy)
    return -np.arctan2(yw, np.sqrt(xw * xw + zw * zw))


def up_vector(x, y, r, e, F, cx, cy):
    """get_up_general's up direction at the position (x, y), unnormalised:
    (-sin r cos e F + sin e (cx - x), -cos r cos e F + sin e (cy - y))."""
    sr, cr, se, ce = math.sin(r), math.cos(r), math.sin(e), math.cos(e)
    return -sr * ce * F + se * (cx - x), -cr * ce * F + se * (cy - y)


def push_direction(Minv, u, v, dx, dy):
    """The direction at the output position that the input direction (dx, dy) at the input position (u, v) maps to: the
    Jacobian of the projective map Minv there applied to (dx, dy)."""
    X = Minv[0, 0] * u + Minv[0, 1] * v + Minv[0, 2]
    Y = Minv[1, 0] * u + Minv[1, 1] * v + Minv[1, 2]
    Z = Minv[2, 0] * u + Minv[2, 1] * v + Minv[2, 2]
    x, y = X / Z, Y / Z
    ox = ((Minv[0, 0] - x * Minv[2, 0]) * dx + (Minv[0, 1] - x * Minv[2, 1]) * dy) / Z
    oy = ((Minv[1, 0] - y * Minv[2, 0]) * dx + (Minv[1, 1] - y * Minv[2, 1]) * dy) / Z
    return ox, oy
