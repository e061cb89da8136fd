"""CPU restatement of ``PanoCam.crop_distortion`` (perspective2d/utils/panocam.py:558-752): crop a perspective or Unified
Spherical Model view from an equirectangular panorama and compute its ground-truth fields.  TEST INFRASTRUCTURE (oracle).

Like oracle/panocam.py it is float64 numpy written in the reference's own order of operations (the same numpy calls, so on
one machine it reproduces the reference bit for bit), and it is pinned to the unmodified reference by tests/golden/pano.npz
(tests/golden/make_golden_pano.py runs the reference's own function with ``grid_sample_default`` below as its sampler).

``crop_distortion`` has the reference's signature, return tuple, warning and assertions; ``crop_distortion_full`` returns
every intermediate the GPU tests need (the sampler's pre-cast values, the unnormalised ``up`` vector and the offset status).
"""
import numpy as np
from numpy.lib.scimath import sqrt as csqrt

STATUS_OK, STATUS_MULTI, STATUS_ASSERT = 0, 1, 2
# sklearn's normalize divides a row by its l2 norm unless the norm is below 10 * eps (sklearn.preprocessing._data.
# _handle_zeros_in_scale): such a row, the exact zero vector included, is returned unscaled
UP_TINY = 10 * np.finfo(np.float64).eps


# ---------------------------------------------------------------------------------------------------------------------------
# The bilinear sampler.  PARITY UNPINNED: the reference calls ``equilib.grid_sample.numpy_grid_sample.default``
# (utils/panocam.py:693-695), and equilib 0.3.0 is neither part of the reference tree nor installable here, so the rule below is
# this project's choice (DESIGN.md section 5), not a restatement:
#   * coordinates in pixel-index units: nx in [0, Wp - 1], ny in [0, Hp - 1] (what crop_distortion's (1/a)(theta - b) produces);
#   * x0 = floor(nx), wx = nx - x0, columns wrap: x0 mod Wp and x1 = (x0 + 1) mod Wp (the panorama is periodic in azimuth);
#   * ny is clamped to [0, Hp - 1], y0 = floor(ny), wy = ny - y0, y1 = min(y0 + 1, Hp - 1);
#   * v = (1 - wy) ((1 - wx) p00 + wx p01) + wy ((1 - wx) p10 + wx p11) in float64, then clipped to [0, 255] and truncated to
#     uint8 (the float -> uint8 cast the reference itself applies in its masked branch, :707).
def grid_sample_precast(img_chw, grid):
    """img_chw: [C, Hp, Wp] uint8; grid: [2, H, W] = (ny, nx) -> float64 [C, H, W] before the cast."""
    _, hp, wp = img_chw.shape
    ny, nx = np.asarray(grid[0], np.float64), np.asarray(grid[1], np.float64)
    x0f = np.floor(nx)
    wx = nx - x0f
    x0 = np.mod(x0f.astype(np.int64), wp)
    x1 = np.mod(x0 + 1, wp)
    nyc = np.minimum(np.maximum(ny, 0.0), hp - 1.0)
    y0f = np.floor(nyc)
    wy = nyc - y0f
    y0 = y0f.astype(np.int64)
    y1 = np.minimum(y0 + 1, hp - 1)
    p = img_chw.astype(np.float64)
    hx, hy = 1.0 - wx, 1.0 - wy
    return hy * (hx * p[:, y0, x0] + wx * p[:, y0, x1]) + wy * (hx * p[:, y1, x0] + wx * p[:, y1, x1])


def grid_sample_default(img_chw, grid):
    """Drop-in for ``equilib.grid_sample.numpy_grid_sample.default(img, grid)`` as crop_distortion calls it: [C, H, W] uint8."""
    return np.clip(grid_sample_precast(img_chw, grid), 0.0, 255.0).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------------
def _deg2rad(deg):        # utils/panocam.py:73-75
    return deg * np.pi / 180


def _minfocal(u0, v0, xi, xref=1, yref=1):    # :64-70
    fmin = np.sqrt(-(1 - xi * xi) * ((xref - u0) * (xref - u0) + (yref - v0) * (yref - v0)))
    return fmin * 1.0001


def _diskradius(xi, f):   # :18-19
    return np.sqrt(-(f * f) / (1 - xi * xi))


def rotations(az, el, roll):
    """The three 3 x 3 matrices of :617-655 (degrees in)."""
    rot_el = np.array([1.0, 0.0, 0.0, 0.0, np.cos(_deg2rad(el)), -np.sin(_deg2rad(el)), 0.0, np.sin(_deg2rad(el)),
                       np.cos(_deg2rad(el))]).reshape((3, 3))
    rot_az = np.array([np.cos(_deg2rad(az)), 0.0, np.sin(_deg2rad(az)), 0.0, 1.0, 0.0, -np.sin(_deg2rad(az)), 0.0,
                       np.cos(_deg2rad(az))]).reshape((3, 3))
    rot_roll = np.array([np.cos(_deg2rad(roll)), -np.sin(_deg2rad(roll)), 0.0, np.sin(_deg2rad(roll)), np.cos(_deg2rad(roll)), 0.0,
                         0.0, 0.0, 1.0]).reshape((3, 3))
    return rot_el, rot_az, rot_roll


def horizon_offset(col):
    """:709-722 on nphi[:, W // 2] -> (offset, status).  status 0: one zero crossing (offset) or none (nan); 1: several (the
    reference prints its WARNING and uses the first); 2: one of the reference's three assertions fails (offset nan)."""
    rows = np.where(np.diff(np.sign(col)))[0]
    status = STATUS_OK
    if len(rows) >= 2:
        status = STATUS_MULTI
        rows = [rows[0]]
    if len(rows) == 0:
        return np.nan, status
    r = rows[0]
    if not (col[r] >= 0) or not (col[r + 1] <= 0):
        return np.nan, STATUS_ASSERT
    dy = col[r + 1] - col[r]
    offset = r - col[r] / dy
    if not (col[r] / dy <= 1.0):
        return np.nan, STATUS_ASSERT
    return offset, status


def crop_distortion_full(image360, f, xi, H, W, az, el, roll):
    """Every output of :559-752 plus what the tests compare against: dict with im (uint8 [H,W,3]), sample (float64 [H,W,3], the
    sampler's values before the cast, before the mask), mask (bool [H,W] or None), ntheta, nphi, lat, xy_map, up (normalised),
    up_raw (the vector before ``normalize``), up_len (its length), offset, status."""
    u0 = W / 2.0                                                          # :577-580
    v0 = H / 2.0
    grid_x, grid_y = np.meshgrid(list(range(W)), list(range(H)))
    image360 = np.asarray(image360)
    pano_w, pano_h = np.shape(image360)[1], np.shape(image360)[0]        # :587-588
    fmin = _minfocal(u0, v0, xi, 1, 1)                                    # :592-594 (nan unless xi > 1)

    x_cam = np.divide(grid_x - u0, f)                                     # :598-599
    y_cam = -np.divide(grid_y - v0, f)
    aux = np.multiply(x_cam, x_cam) + np.multiply(y_cam, y_cam)           # :603-613
    alpha_cam = np.real(xi + csqrt(1 + np.multiply((1 - xi * xi), aux)))  # csqrt of a negative argument: real part 0 -> alpha = xi
    alpha_cam_div = np.divide(alpha_cam, aux + 1)
    x_sph = np.multiply(x_cam, alpha_cam_div)
    y_sph = np.multiply(y_cam, alpha_cam_div)
    z_sph = alpha_cam_div - xi

    rot_el, rot_az, rot_roll = rotations(az, el, roll)                    # :616-660
    coords = np.vstack((x_sph.ravel(), y_sph.ravel(), z_sph.ravel()))
    sph = rot_az.dot(rot_roll.T.dot(rot_el.dot(coords)))
    sph = sph.reshape((3, H, W)).transpose((1, 2, 0))
    x_sph, y_sph, z_sph = sph[:, :, 0], sph[:, :, 1], sph[:, :, 2]

    ntheta = np.arctan2(x_sph, z_sph)                                     # :663-664
    nphi = np.arctan2(y_sph, np.sqrt(z_sph ** 2 + x_sph ** 2))

    min_theta, max_theta, min_phi, max_phi = -np.pi, np.pi, -np.pi / 2.0, np.pi / 2.0      # :666-677
    min_x, max_x, min_y, max_y = 0, pano_w - 1.0, 0, pano_h - 1.0
    ax = (max_theta - min_theta) / (max_x - min_x)                        # :680-687
    bx = max_theta - ax * max_x
    nx = (1.0 / ax) * (ntheta - bx)
    ay = (min_phi - max_phi) / (max_y - min_y)
    by = max_phi - ay * min_y
    ny = (1.0 / ay) * (nphi - by)
    lat = nphi.copy()                                                     # :688-689
    xy_map = np.stack((nx, ny)).transpose(1, 2, 0)

    chw = image360.transpose(2, 0, 1)                                     # :693-695
    sample = grid_sample_precast(chw, np.stack((ny, nx))).transpose(1, 2, 0)
    im = grid_sample_default(chw, np.stack((ny, nx))).transpose(1, 2, 0)
    mask = None
    if f < fmin:                                                          # :696-707
        r = _diskradius(xi, f)
        ci = (np.round(H / 2), np.round(W / 2))                           # numpy rounds half to even
        xx, yy = np.meshgrid(list(range(H)) - ci[0], list(range(W)) - ci[1])
        mask = ((np.multiply(xx, xx) + np.multiply(yy, yy)) < r * r).T
        m3 = np.stack([np.double(mask.T)] * 3, axis=-1).transpose((1, 0, 2))
        im = np.array(np.multiply(im, m3), dtype=np.uint8)

    offset, status = horizon_offset(nphi[:, W // 2])                      # :709-722

    end_x = nx.copy()                                                     # :724-734
    end_y = ny.copy() - 1e-5
    ntheta_end = end_x * ax + bx
    nphi_end = end_y * ay + by
    y_s = np.sin(nphi)                                                    # :736-738 (sin(nphi), not sin(nphi_end))
    x_s = np.cos(nphi_end) * np.sin(ntheta_end)
    z_s = np.cos(nphi_end) * np.cos(ntheta_end)
    coords = np.vstack((x_s.ravel(), y_s.ravel(), z_s.ravel()))           # :740-743
    sph = rot_el.T.dot(rot_roll.dot(rot_az.T.dot(coords)))
    sph = sph.reshape((3, H, W)).transpose((1, 2, 0))
    x_s, y_s, z_s = sph[:, :, 0], sph[:, :, 1], sph[:, :, 2]
    x_c = x_s * f / (xi * csqrt(x_s ** 2 + y_s ** 2 + z_s ** 2) + z_s) + u0    # :747-749
    y_c = -y_s * f / (xi * csqrt(x_s ** 2 + y_s ** 2 + z_s ** 2) + z_s) + v0
    up_raw = np.stack((x_c - grid_x, y_c - grid_y)).transpose(1, 2, 0)
    flat = up_raw.reshape(-1, 2)                                          # :750: sklearn.preprocessing.normalize (l2, rows)
    norms = np.sqrt(np.einsum("ij,ij->i", flat, flat))
    up_len = norms.reshape(H, W).copy()
    norms[norms < UP_TINY] = 1.0                                          # a zero (or near-zero) vector is left as it is
    up = (flat / norms[:, None]).reshape(up_raw.shape)
    return {"im": im, "sample": sample, "mask": mask, "ntheta": ntheta, "nphi": nphi, "lat": lat, "xy_map": xy_map, "up": up,
            "up_raw": up_raw, "up_len": up_len, "offset": offset, "status": status}


def crop_distortion(image360, f, xi, H, W, az, el, roll):
    """:559-752 -> (im, ntheta, nphi, offset, up, lat, xy_map), with the reference's WARNING (several zero crossings of the
    horizon column) and AssertionError (e.g. an upside-down camera)."""
    o = crop_distortion_full(image360, f, xi, H, W, az, el, roll)
    if o["status"] == STATUS_ASSERT:
        raise AssertionError("crop_distortion: the horizon column crosses zero from below (upside-down camera)")
    if o["status"] == STATUS_MULTI:
        col = o["nphi"][:, W // 2]
        print("WARNING | Number of zero crossings:", len(np.where(np.diff(np.sign(col)))[0]))
    return o["im"], o["ntheta"], o["nphi"], o["offset"], o["up"], o["lat"], o["xy_map"]


def make_panorama(seed, hp, wp):
    """A seeded, smooth-plus-noise uint8 RGB panorama [hp, wp, 3] (the goldens and benchmarks regenerate it instead of storing it)."""
    rs = np.random.RandomState(seed)
    y = np.linspace(0.0, 1.0, hp)[:, None, None]
    x = np.linspace(0.0, 1.0, wp)[None, :, None]
    ph = rs.uniform(0, 2 * np.pi, (1, 1, 3))
    base = 127.5 + 80.0 * np.sin(2 * np.pi * (3 * x) + ph) * np.cos(np.pi * (2 * y) + ph)
    noise = rs.uniform(-40.0, 40.0, (hp, wp, 3))
    return np.clip(base + noise, 0, 255).astype(np.uint8)
