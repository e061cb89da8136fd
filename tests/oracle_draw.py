"""CPU restatement of the project's rendering rule for the reference's perspective-field drawings (DESIGN.md section 1), and
of the pinhole ``PanoCam.get_up`` / ``get_lat`` they draw from.  TEST INFRASTRUCTURE (oracle), float64 numpy.

The drawings are ``draw_perspective_fields`` / ``draw_up_field`` / ``draw_latitude_field`` (perspective2d/utils/utils.py:165-430),
which call ``VisualizerPerspective.draw_lati`` (contourf + contour, utils/visualizer.py:236-279) and ``draw_arrow`` (quiver,
:193-234) on a matplotlib figure of the image's own size at 100 dpi, with the image at extent (0, W, H, 0) (:47-53).
matplotlib is not available, so this file states the rule the CUDA kernel implements; its constants are checked against the
reference's own rendering ``assets/vancouver/pred_pers.png`` (tests/test_oracle_draw.py, PARITY UNPINNED otherwise):

* every pixel (i, j) covers [j, j+1] x [i, i+1] and is the mean of 4 x 4 samples at (j + (a + .5)/4, i + (b + .5)/4),
  rounded half to even;
* fill: contourf(x, y, lat) with x, y = mgrid indices puts the values on the nodes (j, i); a sample in the domain
  [0, W-1] x [0, H-1] takes the bilinear value v of its node cell and, in band k (levels linspace(-pi/2, pi/2, 19),
  lev[k] <= v < lev[k+1], the last band closed), becomes c + alpha_contourf (band_k - c), band_k = seismic((k + .5) / 18);
* lines (contour, linewidths=5 at 100 dpi): a sample with |v - lev[k]| <= (lw / 2) |grad v| becomes
  c + alpha_contour (line_k - c), line_k = seismic(k / 18), in increasing k;
* arrows (quiver with scale_units="xy", scale=1, angles="uv", headaxislength=3.5, default headwidth 3, headlength 5,
  minshaft 1, minlength 1), drawn last: opaque polygons, shaft width 0.06 W / clip(sqrt(N), 8, 25) px (quiver's default
  width).  pred_pers.png shows them over the contour lines (fully covered shaft pixels stay (0, 255, 0) inside the horizon line);
* seismic: matplotlib's anchors (0, 0, .3) (0, 0, 1) (1, 1, 1) (1, 0, 0) (.5, 0, 0) at 0, 1/4, 1/2, 3/4, 1, sampled into a
  256-entry table at i / 255; t -> entry min(floor(256 t), 255).
"""
import math

import numpy as np

LEVELS = np.linspace(-np.pi / 2, np.pi / 2, 19)                  # visualizer.py:243-244: bands = 20, linspace(.., bands - 1)
HALF_LINE = 0.5 * 5 * 100 / 72                                   # linewidths=5 (:263) points at the figure's 100 dpi, halved
GREEN = (0.0, 1.0, 0.0)                                          # utils.py:200-201
C0 = (0x1F / 255, 0x77 / 255, 0xB4 / 255)                       # matplotlib's default colour cycle, first entry
_ANCHORS = np.array([(0.0, 0.0, 0.3), (0.0, 0.0, 1.0), (1.0, 1.0, 1.0), (1.0, 0.0, 0.0), (0.5, 0.0, 0.0)])


def seismic_table():
    """[256, 3] float64: LinearSegmentedColormap.from_list("seismic", anchors) sampled at i / 255."""
    x = np.arange(256) / 255.0
    s = np.minimum((x * 4).astype(int), 3)
    dist = (x - s / 4.0) / 0.25
    return dist[:, None] * (_ANCHORS[s + 1] - _ANCHORS[s]) + _ANCHORS[s]


def seismic(t):
    return seismic_table()[min(int(math.floor(256 * t)), 255)]


BAND = np.array([seismic((k + 0.5) / 18) for k in range(18)]) * 255.0
LINE = np.array([seismic(k / 18) for k in range(19)]) * 255.0


def arrow_lattice(h, w, density, arrow_inv_len):
    """utils.py:192-199: tails x = arange(0, W, W // density), y likewise (meshgrid, y outer), length factor
    sqrt(W^2 + H^2) // arrow_inv_len."""
    x, y = np.meshgrid(np.arange(0, w, w // density), np.arange(0, h, h // density))
    return x.ravel(), y.ravel(), np.sqrt(w ** 2 + h ** 2) // arrow_inv_len


def shaft_width(w, n):
    """quiver's default width (0.06 of the axes span over clip(sqrt(N), 8, 25)) in canvas pixels."""
    return 0.06 * w / np.clip(np.sqrt(n), 8, 25)


def arrow_hit(rx, ry, d, inv, lp):
    """Samples (rx, ry) relative to the tail, unit direction d, 1 / (k w), polygon length lp in units of k w (< 0: hexagon).
    The polygon (0, .5) (lp-3.5, .5) (lp-5, 1.5) (lp, 0) and its mirror image; the hexagon of circumradius 1/2 with a vertex
    along d (quiver's _h_arrows for vectors shorter than minlength)."""
    a = (rx * d[0] + ry * d[1]) * inv
    b = np.abs(ry * d[0] - rx * d[1]) * inv
    if lp < 0:
        apo = math.sqrt(3) / 4
        return (b <= apo) & (math.sqrt(3) / 2 * np.abs(a) + 0.5 * b <= apo)
    tip = b <= 0.3 * (lp - a)
    return tip & np.where(b <= 0.5, a >= 0, a >= lp - 3.5 - 1.5 * (b - 0.5))


def draw(img, up=None, lat=None, color=GREEN, density=10, arrow_inv_len=20, alpha_fill=0.4, alpha_line=0.9):
    """img uint8 [H, W, 3]; up [H, W, 2] (float32 values, as the kernel reads them) or None; lat [H, W] radians or None.
    Returns the drawn uint8 [H, W, 3]."""
    h, w = img.shape[:2]
    off = (np.arange(4) + 0.5) / 4
    sy = (np.arange(h)[:, None] + off[None, :]).reshape(-1)            # [4H] sample rows
    sx = (np.arange(w)[:, None] + off[None, :]).reshape(-1)            # [4W]
    col = np.repeat(np.repeat(img.astype(np.float64), 4, 0), 4, 1)     # [4H, 4W, 3]
    dom = np.zeros((4 * h, 4 * w), bool)
    if lat is not None:
        lat = np.asarray(lat, np.float64)
        i0 = np.minimum(np.floor(sy).astype(int), max(h - 2, 0))
        j0 = np.minimum(np.floor(sx).astype(int), max(w - 2, 0))
        dom = (np.floor(sy)[:, None] < h - 1) & (np.floor(sx)[None, :] < w - 1)
        if h >= 2 and w >= 2:
            fy, fx = (sy - i0)[:, None], (sx - j0)[None, :]
            v00, v01 = lat[i0][:, j0], lat[i0][:, j0 + 1]
            v10, v11 = lat[i0 + 1][:, j0], lat[i0 + 1][:, j0 + 1]
            v = (1 - fy) * ((1 - fx) * v00 + fx * v01) + fy * ((1 - fx) * v10 + fx * v11)
            gx = (1 - fy) * (v01 - v00) + fy * (v11 - v10)
            gy = (1 - fx) * (v10 - v00) + fx * (v11 - v01)
        else:
            v = gx = gy = np.zeros(dom.shape)
        with np.errstate(invalid="ignore"):
            band = np.clip(np.searchsorted(LEVELS, v, side="right") - 1, 0, 17)
            fill = dom & (v >= LEVELS[0]) & (v <= LEVELS[-1])
        col = np.where(fill[..., None], col + alpha_fill * (BAND[band] - col), col)
    if lat is not None:
        g = HALF_LINE * np.hypot(gx, gy)
        for k in range(19):
            with np.errstate(invalid="ignore"):
                on = dom & (np.abs(v - LEVELS[k]) <= g)
            col = np.where(on[..., None], col + alpha_line * (LINE[k] - col), col)
    if up is not None:
        up = np.asarray(up, np.float64)
        x, y, length = arrow_lattice(h, w, density, arrow_inv_len)
        sw = shaft_width(w, len(x))
        hit = np.zeros((4 * h, 4 * w), bool)
        for tx, ty in zip(x, y):
            u = up[ty, tx] * length
            ln = math.hypot(u[0], u[1])
            d = u / ln if ln > 0 else np.array([1.0, 0.0])
            l = ln / sw
            if l < 1:
                inv, lp, reach = 1 / sw, -1.0, 0.5 * sw
            elif l < 5:
                inv, lp, reach = 5 / ln, 5.0, 1.3 * ln
            else:
                inv, lp, reach = 1 / sw, l, ln + 1.5 * sw
            r0, r1 = np.searchsorted(sy, ty - reach), np.searchsorted(sy, ty + reach, side="right")
            c0, c1 = np.searchsorted(sx, tx - reach), np.searchsorted(sx, tx + reach, side="right")
            if r0 < r1 and c0 < c1:
                hit[r0:r1, c0:c1] |= arrow_hit(sx[None, c0:c1] - tx, sy[r0:r1, None] - ty, d, inv, lp)
        col = np.where(hit[..., None], np.asarray(color, np.float64) * 255.0, col)
    return np.rint(col.reshape(h, 4, w, 4, 3).mean(axis=(1, 3))).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------------
# PanoCam.get_lat / get_up (perspective2d/utils/panocam.py:384-448), with the helpers they call (:271-382); sklearn's
# normalize restated (rows divided by their l2 norm unless it is below 10 eps)

def _normalize(x):
    n = np.sqrt(np.einsum("ij,ij->i", x, x))
    n[n < 10 * np.finfo(np.float64).eps] = 1.0
    return x / n[:, None]


def get_lat(vfov, im_w, im_h, elevation, roll):
    """:384-420, degrees."""
    focal_length = im_h / 2 / np.tan(vfov / 2)
    dy = np.linspace(-im_h / 2, im_h / 2, im_h)
    dx = np.linspace(-im_w / 2, im_w / 2, im_w)
    x, y = np.meshgrid(dx, dy)
    x, y = x.ravel() / focal_length, y.ravel() / focal_length
    focal_length = 1
    x_world = x * np.cos(roll) - y * np.sin(roll)
    y_world = x * np.cos(elevation) * np.sin(roll) + y * np.cos(elevation) * np.cos(roll) - focal_length * np.sin(elevation)
    z_world = x * np.sin(elevation) * np.sin(roll) + y * np.sin(elevation) * np.cos(roll) + focal_length * np.cos(elevation)
    l = -np.arctan2(y_world, np.sqrt(x_world ** 2 + z_world ** 2)) / np.pi * 180
    return l.reshape(im_h, im_w)


def get_up(vfov, im_w, im_h, elevation, roll):
    """:422-448: unit vectors from every pixel index (j, i) to the vertical vanishing point (:302-333), or at elevation == 0
    to a point 1e8 px away along the horizon's normal (:288-300)."""
    if elevation == np.pi / 2 or elevation == -np.pi / 2:
        mid = np.inf * np.sign(elevation)
    else:
        mid = 0.5 + 0.5 * np.tan(elevation) / np.cos(roll) / np.tan(vfov / 2)
    dh = np.inf * np.sign(roll) if roll == np.pi / 2 or roll == -np.pi / 2 else -im_w / im_h * np.tan(roll) / 2
    horizon = (mid - dh, mid + dh)
    if elevation == 0:
        vvp_abs = 1e8 * _normalize(np.array([[im_h * (horizon[1] - horizon[0]), -im_w]]))[0]
        absvvp = np.array([vvp_abs[0] + 0.5 * im_w - 0.5, vvp_abs[1] + 0.5 * im_h - 0.5, 1])
    else:
        vx = 0.5 - 0.5 / im_w - 0.5 * np.sin(roll) / np.tan(elevation) / np.tan(vfov / 2) * im_h / im_w
        vy = 0.5 - 0.5 / im_h - 0.5 * np.cos(roll) / np.tan(elevation) / np.tan(vfov / 2)
        absvvp = np.array([vx * im_w, vy * im_h, np.sign(elevation)])
    gridx, gridy = np.meshgrid(np.arange(0, im_w), np.arange(0, im_h))
    start = np.stack((gridx.reshape(-1), gridy.reshape(-1))).T
    arrow = _normalize(absvvp[:2] - start) * absvvp[2]
    return arrow.reshape(im_h, im_w, 2)
