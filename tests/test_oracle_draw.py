"""CPU: the constants of the drawing rule (tests/oracle_draw.py, DESIGN.md section 1) against the reference's own rendering
assets/vancouver/pred_pers.png (windows in tests/golden/draw_vancouver.npz, with the demo's cv2-resized input image), the
pinhole PanoCam.get_up / get_lat restatement against the unmodified reference (tests/golden/pinhole.npz), and the drawing
functions' argument checks, which raise before any GPU work."""
import inspect
import os

import numpy as np
import pytest

import oracle_draw as od
from perspectivefields_b200 import viz

GOLD = os.path.join(os.path.dirname(__file__), "golden")
V = np.load(os.path.join(GOLD, "draw_vancouver.npz"))
P, I = V["pred_a"].astype(np.float64), V["img_a"].astype(np.float64)
R0, _, C0, _ = V["window_a"]
ARROW_X = (192, 256)                                     # lattice columns in window a: arange(0, 640, 64)


def _away_from_arrows(cols, margin=9):
    return np.array([all(abs(c - x) > margin for x in ARROW_X) for c in cols])


def test_fill_alpha_and_band_colour():
    """Between the horizon line and the next line up (band 9): pred = (1 - alpha) img + alpha 255 band_9 per channel."""
    rows = slice(300 - R0, 350 - R0)
    cols = np.nonzero(_away_from_arrows(np.arange(P.shape[1]) + C0))[0]
    p, x = P[rows][:, cols].reshape(-1, 3), I[rows][:, cols].reshape(-1, 3)
    keep = (x.min(1) > 5) & (x.max(1) < 250)                  # clipped pixels of the JPEG say nothing about the blend
    p, x = p[keep], x[keep]
    # one alpha for the three channels (least squares of pred - img = alpha (255 colour - img) with a free colour), then each
    # channel's colour at that alpha (median: robust to the JPEG's and the resize's noise)
    eqs = []
    for ch in range(3):
        e = np.zeros((len(x), 4))
        e[:, 0] = -x[:, ch]
        e[:, 1 + ch] = 1.0
        eqs.append(e)
    sol = np.linalg.lstsq(np.concatenate(eqs), np.concatenate([p[:, ch] - x[:, ch] for ch in range(3)]), rcond=None)[0]
    alpha = float(sol[0])
    colours = np.median((p - (1 - alpha) * x) / alpha, axis=0) / 255
    assert abs(alpha - 0.40) <= 0.02, alpha
    assert np.abs(np.array(colours) - od.BAND[9] / 255).max() <= 0.02, (colours, od.BAND[9] / 255)
    assert np.allclose(od.BAND[9] / 255, [1.0, 0.882, 0.882], atol=1e-3)


def test_arrow_shaft_colour_and_width():
    """Shaft rows of the arrow at x = 192 (tail y = 312): fully covered pixels are exactly (0, 255, 0); the coverage summed
    across the shaft (1 - red / background red, background = the band-9 fill) is the rule's 0.06 W / sqrt(110) = 3.66 px."""
    widths = []
    for y in range(292, 308):
        row, img = P[y - R0], I[y - R0]
        cols = np.arange(184 - C0, 201 - C0)
        full = [c for c in cols if tuple(row[c]) == (0.0, 255.0, 0.0)]
        assert len(full) >= 2, y
        bg = 0.6 * img[cols, 0] + 0.4 * od.BAND[9][0]
        widths.append(np.clip(1 - row[cols, 0] / bg, 0, 1).sum())
    w = od.shaft_width(640, 110)
    assert abs(w - 3.66) < 0.01
    assert abs(np.mean(widths) - w) <= 0.3, widths


def test_contour_line_width():
    """The horizon line (level 9) across columns without arrows: the coverage summed down each column (green channel, band 9
    above the line's centre, band 8 below, full coverage = alpha 0.9 of line 9's colour) is 5 pt at 100 dpi = 6.94 px."""
    widths = []
    for c in np.nonzero(_away_from_arrows(np.arange(P.shape[1]) + C0, 12))[0]:
        p, x = P[350 - R0:395 - R0, c, 1], I[350 - R0:395 - R0, c, 1]
        centre = int(np.argmax(p))
        cov = []
        for r in range(len(p)):
            bg = 0.6 * x[r] + 0.4 * (od.BAND[9] if r <= centre else od.BAND[8])[1]
            full = bg + 0.9 * (od.LINE[9][1] - bg)
            cov.append(np.clip((p[r] - bg) / (full - bg), 0, 1))
        widths.append(sum(cov))
    lw = 2 * od.HALF_LINE
    assert abs(lw - 6.94) < 0.01
    assert abs(np.median(widths) - lw) <= 0.5, widths


def test_arrows_are_drawn_over_the_contour_lines():
    """Window b: the shaft at x = 576 crosses the horizon line.  Its fully covered column stays exactly (0, 255, 0) on rows
    where the columns beside it carry the line (a line over the arrow would leave at least 0.9 * 255 in red)."""
    pb = V["pred_b"].astype(np.float64)
    r0, _, c0, _ = V["window_b"]
    for y in range(358, 363):
        assert tuple(pb[y - r0, 576 - c0]) == (0.0, 255.0, 0.0), y
        assert pb[y - r0, 579 - c0:584 - c0].min() > 0.9 * 255 * 0.95, y


def test_seismic_table():
    t = od.seismic_table()
    assert t.shape == (256, 3) and np.allclose(t[0], (0, 0, 0.3)) and np.allclose(t[255], (0.5, 0, 0))
    assert np.allclose(od.seismic(0.5), (1, 1 - 4 / 510, 1 - 4 / 510))


def test_pinhole_restatement_matches_reference_golden():
    g = np.load(os.path.join(GOLD, "pinhole.npz"))
    for i, (vfov, w, h, el, roll) in enumerate(g["cases"]):
        assert np.abs(od.get_up(vfov, int(w), int(h), el, roll) - g[f"up{i}"]).max() <= 1e-12, i
        assert np.abs(od.get_lat(vfov, int(w), int(h), el, roll) - g[f"lat{i}"]).max() <= 1e-12, i


def test_constant_in_band_fill_rounds_away_from_half():
    """The GPU test of a constant in-band latitude compares bit for bit with round(0.6 img + 0.4 colour): no value of that
    formula lies within 1e-3 of a rounding tie, so float32 and float64 agree on every byte."""
    img = np.arange(256, dtype=np.float64)[:, None]
    for k in (3, 9, 12):
        v = 0.6 * img + 0.4 * od.BAND[k][None, :]
        assert np.abs(v - np.floor(v) - 0.5).min() > 1e-3, k


def test_drop_in_signatures():
    from perspectivefields_b200 import panocam

    sig = lambda f: [(p.name, p.default) for p in inspect.signature(f).parameters.values()]
    e = inspect.Parameter.empty
    assert sig(viz.draw_perspective_fields) == [("img_rgb", e), ("up", e), ("latimap", e), ("color", None), ("density", 10),
                                                ("arrow_inv_len", 20), ("return_img", True)]
    assert sig(viz.draw_up_field) == [("img_rgb", e), ("vector_field", e), ("color", None), ("density", 10), ("arrow_inv_len", 20),
                                      ("return_img", True)]
    assert sig(viz.draw_latitude_field) == [("img_rgb", e), ("latimap", None), ("binmap", None), ("alpha_contourf", 0.4),
                                            ("alpha_contour", 0.9), ("return_img", True)]
    assert sig(viz.draw_from_r_p_f) == [("img", e), ("roll", e), ("pitch", e), ("vfov", e), ("mode", e), ("up_color", None),
                                        ("alpha_contourf", 0.4), ("alpha_contour", 0.9), ("draw_up", True), ("draw_lat", True),
                                        ("lati_alpha", 0.5)]
    assert sig(viz.draw_from_r_p_f_cx_cy) == [("img", e), ("roll", e), ("pitch", e), ("vfov", e), ("rel_cx", e), ("rel_cy", e),
                                              ("mode", e), ("up_color", None), ("alpha_contourf", 0.4), ("alpha_contour", 0.9),
                                              ("draw_up", True), ("draw_lat", True)]
    assert [p for p, _ in sig(panocam.PanoCam.get_up)][:5] == ["vfov", "im_w", "im_h", "elevation", "roll"]
    assert [p for p, _ in sig(panocam.PanoCam.get_lat)][:5] == ["vfov", "im_w", "im_h", "elevation", "roll"]


def test_bad_arguments_raise_value_error_before_gpu_work():
    img = np.zeros((48, 64, 3), np.uint8)
    up = np.zeros((48, 64, 2), np.float32)
    lat = np.zeros((48, 64), np.float32)
    bad = [
        lambda: viz.draw_perspective_fields(img, up, lat, density=0),
        lambda: viz.draw_perspective_fields(img, up, lat, density=65),          # 64 // 65 == 0
        lambda: viz.draw_perspective_fields(img, up, lat, arrow_inv_len=0),
        lambda: viz.draw_perspective_fields(img, up[:, :-1], lat),
        lambda: viz.draw_perspective_fields(img, up, lat[:-1]),
        lambda: viz.draw_perspective_fields(img[..., :2], up, lat),
        lambda: viz.draw_perspective_fields(img, up, lat, color=(0, 2, 0)),
        lambda: viz.draw_up_field(img, up, color=(0, 1)),
        lambda: viz.draw_latitude_field(img),
        lambda: viz.draw_latitude_field(img, lat, alpha_contourf=1.5),
        lambda: viz.draw_from_r_p_f(img, 1.0, 2.0, 60.0, "grad"),
        lambda: viz.draw_from_r_p_f_cx_cy(img, 1.0, 2.0, 60.0, 0.0, 0.0, "degrees"),
        lambda: viz.draw_fields_batch([img, img], [up], [lat, lat]),
        lambda: viz.draw_predictions([img], []),
    ]
    for k, f in enumerate(bad):
        with pytest.raises(ValueError):
            f()
