"""CPU: the oracle's restatement of PanoCam.crop_distortion (tests/oracle_pano.py) against golden outputs of the unmodified
reference (tests/golden/pano.npz, make_golden_pano.py), the horizon-offset status cases, the sampler rule, and the argument
checks of the Python API (which run before any GPU work)."""
import ctypes
import os
import warnings

import numpy as np
import pytest

import oracle_pano as op

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "pano.npz"))
PANO = op.make_panorama(*[int(x) for x in GOLD["pano"]])
CASES = [tuple(c) for c in GOLD["cases"]]
KEEP = [i for i in range(len(CASES)) if not GOLD["raises"][i]]


def _full(i):
    f, xi, h, w, az, el, roll = CASES[i]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)      # minfocal's sqrt of a negative number (nan unless xi > 1)
        return op.crop_distortion_full(PANO, f, xi, int(h), int(w), az, el, roll)


@pytest.mark.parametrize("i", KEEP)
def test_oracle_matches_reference_golden(i):
    o = _full(i)
    h, w = int(CASES[i][2]), int(CASES[i][3])
    for k in ("ntheta", "nphi", "lat"):
        assert o[k].shape == (h, w) and np.abs(o[k] - GOLD[f"{k}{i}"]).max() <= 1e-12, k
    xy = GOLD[f"xy_map{i}"]
    assert o["xy_map"].shape == (h, w, 2) and (np.abs(o["xy_map"] - xy) <= 1e-12 * np.maximum(1.0, np.abs(xy))).all()
    assert o["im"].dtype == np.uint8 and np.array_equal(o["im"], GOLD[f"im{i}"])
    g_off = float(GOLD[f"offset{i}"])
    assert (np.isnan(g_off) and np.isnan(o["offset"])) or abs(o["offset"] - g_off) <= 1e-12
    up, g_up = o["up"], GOLD[f"up{i}"]
    big = o["up_len"] >= 1e-6
    assert np.abs(up - g_up)[big].max(initial=0.0) <= 1e-6
    assert (o["up_len"][(g_up == 0).all(axis=2)] < 1e-12).all()
    # the reference's crop lies on the panorama: every xy inside [0, Wp - 1] x [0, Hp - 1] up to rounding
    assert xy[..., 0].min() > -1e-9 and xy[..., 0].max() < PANO.shape[1] - 1 + 1e-9
    assert xy[..., 1].min() > -1e-9 and xy[..., 1].max() < PANO.shape[0] - 1 + 1e-9


def test_golden_cases_cover_the_issue_list():
    c = np.array(CASES)
    assert {0.0, 0.5, 0.9, 1.2}.issubset(set(c[:, 1]))
    assert any(_full(i)["mask"] is not None for i in KEEP)                       # catadioptric disk
    assert any(int(h) % 2 and int(w) % 2 and _full(i)["mask"] is not None for i, (_, _, h, w, *_r) in enumerate(CASES) if i in KEEP)
    seam = [i for i in KEEP if GOLD[f"xy_map{i}"][..., 0].min() < 2 and GOLD[f"xy_map{i}"][..., 0].max() > PANO.shape[1] - 3]
    assert seam
    ys = np.concatenate([GOLD[f"xy_map{i}"][..., 1].ravel() for i in KEEP])
    assert ys.min() < 2 and ys.max() > PANO.shape[0] - 3                        # both poles
    assert GOLD["raises"].sum() == 1


def test_offset_status_cases(capsys):
    # level camera, even H: nphi is exactly 0 on row H / 2, two crossings -> the reference's WARNING and the first crossing
    i = [k for k in KEEP if CASES[k][4:] == (0.0, 0.0, 0.0)][0]
    o = _full(i)
    assert o["status"] == op.STATUS_MULTI and o["offset"] == CASES[i][2] / 2
    assert (o["nphi"][int(CASES[i][2]) // 2] == 0).all()
    f, xi, h, w, az, el, roll = CASES[i]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        op.crop_distortion(PANO, f, xi, int(h), int(w), az, el, roll)
        assert "WARNING | Number of zero crossings: 2" in capsys.readouterr().out
        # upside down: the reference raises AssertionError
        j = int(np.nonzero(GOLD["raises"])[0][0])
        f, xi, h, w, az, el, roll = CASES[j]
        assert roll == 180.0
        with pytest.raises(AssertionError):
            op.crop_distortion(PANO, f, xi, int(h), int(w), az, el, roll)
        assert op.crop_distortion_full(PANO, f, xi, int(h), int(w), az, el, roll)["status"] == op.STATUS_ASSERT
        # camera pointing at a pole: no crossing -> nan, status 0
        o = op.crop_distortion_full(PANO, 20.0, 0.0, 32, 48, 0.0, 88.0, 0.0)
        assert o["status"] == op.STATUS_OK and np.isnan(o["offset"])
        # a tilted camera: one crossing
        o = op.crop_distortion_full(PANO, 30.0, 0.0, 48, 64, 10.0, 7.0, 3.0)
        assert o["status"] == op.STATUS_OK and 0 < o["offset"] < 47
    assert op.horizon_offset(np.array([-0.2, -0.1, 0.1]))[1] == op.STATUS_ASSERT
    assert op.horizon_offset(np.array([0.3, 0.1, -0.1, -0.2])) == (pytest.approx(1.5), op.STATUS_OK)


def test_sampler_rule():
    img = np.zeros((3, 4, 5), np.uint8)                 # [C, Hp, Wp]
    img[0] = np.arange(20).reshape(4, 5) * 10
    grid = np.array([[[0.0, 0.0, 3.0, 3.7, -1e-17]], [[4.5, 0.25, 2.0, 1.0, 0.0]]])   # (ny, nx), [2, 1, 5]
    v = op.grid_sample_precast(img, grid)[0, 0]
    assert v[0] == pytest.approx(0.5 * 40 + 0.5 * 0)       # x = Wp - 1 + 0.5 wraps to column 0
    assert v[1] == pytest.approx(2.5)
    assert v[2] == 170.0                                    # the last row: y1 clamps to Hp - 1
    assert v[3] == 160.0                                    # ny beyond Hp - 1 clamps
    assert v[4] == 0.0                                      # ny slightly below 0 clamps
    assert op.grid_sample_default(img, np.array([[[0.0]], [[0.99]]]))[0, 0, 0] == 9       # 9.9 truncates to 9


def test_python_api_checks_arguments_before_gpu_work(tmp_path):
    from perspectivefields_b200 import panocam as pc
    pano = np.zeros((16, 32, 3), np.uint8)
    good = (10.0, 0.0, 8, 8, 0.0, 0.0, 0.0)
    bad_views = [(0.0, 0.0, 8, 8, 0, 0, 0), (float("nan"), 0.0, 8, 8, 0, 0, 0), (10.0, float("inf"), 8, 8, 0, 0, 0),
                 (10.0, 0.0, 0, 8, 0, 0, 0), (10.0, 0.0, 8, 2.5, 0, 0, 0), (10.0, 0.0, True, 8, 0, 0, 0),
                 (10.0, 0.0, 8, 8, 0, "x", 0), (10.0, 0.0, 8, 8, 0, 0), {"f": 10.0, "xi": 0.0, "H": 8}]
    for v in bad_views:
        with pytest.raises(ValueError):
            pc.crop_distortion_views(pano, [good, v])
    with pytest.raises(ValueError):
        pc.crop_distortion_views(pano, [])
    with pytest.raises(ValueError):
        pc.crop_distortion_views(pano, [good], outputs=("up", "depth"))
    for p in (pano.astype(np.float32), pano[:, :, :2], pano[:, :, 0]):
        with pytest.raises(TypeError):
            pc.crop_distortion_views(p, [good])
    with pytest.raises(ValueError):
        pc.crop_distortion_views(pano[:1], [good])
    with pytest.raises(ValueError):
        pc.PanoCam.crop_distortion(pano, -1.0, 0.0, 8, 8, 0.0, 0.0, 0.0)
    # a path is read with Pillow as RGB (what imageio.imread returns for an 8-bit file)
    from PIL import Image
    rgb = op.make_panorama(3, 16, 32)
    Image.fromarray(rgb).convert("P").save(tmp_path / "pano.png")       # palette image: converted to RGB on reading
    assert np.array_equal(pc._check_panorama(str(tmp_path / "pano.png")), np.asarray(Image.fromarray(rgb).convert("P").convert("RGB")))


def test_pf_pano_view_struct_layout():
    from perspectivefields_b200 import _native
    assert ctypes.sizeof(_native.pf_pano_view) == 64          # include/pf_b200.h: 2 x int32, 5 x double, 2 x int64
    assert _native.pf_pano_view.f.offset == 8 and _native.pf_pano_view.im_offset.offset == 48
    assert _native.pf_pano_view.field_offset.offset == 56
