"""GPU: pf_draw_fields (csrc/draw.cuh) against the numpy restatement of the drawing rule (tests/oracle_draw.py), its exact
properties, the viz drop-ins of the reference's draw_* functions, and the pinhole PanoCam.get_up / get_lat.

Kernel vs oracle: the kernel decides each of the 16 samples of a pixel in float32, the oracle in float64, so a sample that lies
within rounding distance of a band, line or arrow boundary may flip; one flipped sample moves a byte by at most 255 / 16.
Hence >= 99.9 % of bytes within 1 and every byte within 16."""
import math
import os

import numpy as np
import pytest
import torch

import oracle_draw as od
import pf_test_util as U
from oracle import weights_gen as wg
from perspectivefields_b200 import _native, panocam as pc, viz

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _img(h, w, seed):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


def _close(got, ref, what):
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    assert got.shape == ref.shape, what
    assert (d <= 1).mean() >= 0.999, (what, (d <= 1).mean())
    assert d.max() <= 16, (what, d.max())


def _fields(h, w, el=-0.25, roll=0.2, f=0.9):
    ups, lats = pc.camera_fields([f], [h], [w], [el], [roll], [0.05], [-0.03])
    return ups[0], torch.deg2rad(lats[0])


def test_kernel_matches_oracle_on_camera_fields():
    cases = [(480, 640, 10, 20), (13, 17, 2, 20), (100, 70, 10, 7), (233, 301, 1, 20), (480, 640, 64, 20), (1, 50, 1, 20)]
    for k, (h, w, density, inv) in enumerate(cases):
        img = _img(h, w, k)
        up, lat = _fields(h, w)
        lat_in = lat if h > 1 else None
        got = viz.draw_fields_batch([img], [up], [lat_in], density=density, arrow_inv_len=inv)[0]
        ref = od.draw(img, up.cpu().numpy(), None if lat_in is None else lat.cpu().numpy(), density=density, arrow_inv_len=inv)
        _close(got, ref, (h, w, density))
        # latitude only, arrows only
        _close(viz.draw_latitude_field(img, lat.cpu().numpy()), od.draw(img, lat=lat.cpu().numpy()), ("lat", h, w))
        _close(viz.draw_up_field(img, up, density=density, arrow_inv_len=inv),
               od.draw(img, up=up.cpu().numpy(), color=od.C0, density=density, arrow_inv_len=inv), ("up", h, w))


def test_kernel_matches_oracle_on_short_and_degenerate_arrows():
    """Vectors scaled to lengths between 1 and 5 shaft widths (the scaled-down polygon), below one (the hexagon) and zero."""
    h, w = 240, 320
    img = _img(h, w, 5)
    up, _ = _fields(h, w)
    length = math.sqrt(w * w + h * h) // 20
    sw = od.shaft_width(w, len(od.arrow_lattice(h, w, 10, 20)[0]))
    for scale in (3.0 * sw / length, 0.6 * sw / length, 0.0):
        u = up * scale
        _close(viz.draw_up_field(img, u, color=(1, 0, 0)), od.draw(img, up=u.cpu().numpy(), color=(1, 0, 0)), scale)
    rs = np.random.RandomState(3)
    u = torch.tensor(rs.uniform(-1, 1, (h, w, 2)) * rs.uniform(0, 8 * sw / length, (h, w, 1)), dtype=torch.float32).cuda()
    _close(viz.draw_up_field(img, u, density=20), od.draw(img, up=u.cpu().numpy(), color=od.C0, density=20), "mixed lengths")


def test_kernel_matches_oracle_on_a_prediction_at_640_wide():
    version = "Paramnet-360Cities-edina-centered"
    m, _ = U.make_model(version)
    src = wg.smooth_images(1, 768, 1024, 3)[0]
    pred = m.inference(src)
    up, lat = viz.resize_fields(pred["pred_gravity_original"], pred["pred_latitude_original"], 640)
    h, w = lat.shape
    img = _img(h, w, 9)
    lat = torch.deg2rad(lat)
    got = viz.draw_perspective_fields(img, up, lat)
    ref = od.draw(img, up.cpu().numpy().transpose(1, 2, 0), lat.cpu().numpy())
    _close(got, ref, "prediction")


def test_nothing_drawn_leaves_the_image():
    img = _img(70, 90, 1)
    _, lat = _fields(70, 90)
    out = viz.draw_latitude_field(img, lat, alpha_contourf=0.0, alpha_contour=0.0)
    assert np.array_equal(out, img)


def test_constant_in_band_latitude():
    h, w = 37, 53
    img = _img(h, w, 2)
    for k in (3, 9, 12):
        v = (od.LEVELS[k] + od.LEVELS[k + 1]) / 2
        out = viz.draw_latitude_field(img, np.full((h, w), v, np.float32))
        ref = np.rint(0.6 * img[:-1, :-1] + 0.4 * od.BAND[k]).astype(np.uint8)
        assert np.array_equal(out[:-1, :-1], ref), k
        assert np.array_equal(out[-1], img[-1]) and np.array_equal(out[:, -1], img[:, -1]), k


def test_interior_arrow_pixels_are_the_arrow_colour():
    h, w = 120, 160
    up = torch.tensor([0.3, -1.0]).cuda().expand(h, w, 2).contiguous()
    color = (0.2, 0.6, 1.0)
    img = _img(h, w, 4)
    out = viz.draw_up_field(img, up, color=color)
    full = od.draw(np.zeros((h, w, 3), np.uint8), up=up.cpu().numpy(), color=(1, 1, 1)).min(axis=2) == 255
    assert full.sum() > 50
    assert (out[full] == np.array([51, 153, 255], np.uint8)).all()


def test_batch_over_chunks_equals_single_calls_and_in_place_equals_out_of_place():
    rs = np.random.RandomState(6)
    sizes = [(int(rs.randint(20, 130)), int(rs.randint(20, 200))) for _ in range(30)]     # 30 > 24 canvases per launch
    imgs = [_img(h, w, 100 + k) for k, (h, w) in enumerate(sizes)]
    ups, lats = [], []
    for k, (h, w) in enumerate(sizes):
        u, l = _fields(h, w, el=rs.uniform(-0.6, 0.6), roll=rs.uniform(-0.5, 0.5))
        ups.append(u.permute(2, 0, 1).contiguous() if k % 2 else u)      # both layouts, read in place
        lats.append(l if k % 3 else None)
    batch = viz.draw_fields_batch(imgs, ups, lats, density=5)
    for k in range(len(sizes)):
        one = viz.draw_fields_batch([imgs[k]], [ups[k]], [lats[k]], density=5)[0]
        assert np.array_equal(batch[k], one), k
    dev = [torch.from_numpy(im).cuda() for im in imgs]
    inplace = viz._draw([d.clone() for d in dev], [u if u.shape[-1] == 2 else u.permute(1, 2, 0) for u in ups], lats,
                        [od.GREEN] * len(dev), 5, 20, 0.4, 0.9, in_place=True)
    for k in range(len(sizes)):
        assert np.array_equal(inplace[k].cpu().numpy(), batch[k]), k


def test_drop_in_types_and_save(tmp_path):
    h, w = 96, 128
    img = _img(h, w, 8)
    up, lat = _fields(h, w)
    out = viz.draw_perspective_fields(img, up.permute(2, 0, 1).cpu(), lat.cpu().numpy())   # the demo's CPU [2, H, W] tensor
    assert isinstance(out, np.ndarray) and out.dtype == np.uint8 and out.shape == (h, w, 3)
    dev = viz.draw_perspective_fields(torch.from_numpy(img).cuda(), up, lat)
    assert isinstance(dev, torch.Tensor) and dev.is_cuda and dev.dtype == torch.uint8
    assert np.array_equal(dev.cpu().numpy(), out)
    vis = viz.draw_perspective_fields(img, up, lat, color=(0, 1, 0), return_img=False)
    assert np.array_equal(vis.get_image(), out)
    vis.save(str(tmp_path / "perspective_pred"))
    from PIL import Image
    assert np.array_equal(np.array(Image.open(tmp_path / "perspective_pred.png")), out)
    assert isinstance(viz.draw_latitude_field(img, lat, return_img=False), viz.DrawnImage)
    assert isinstance(viz.draw_up_field(img, up, return_img=False), viz.DrawnImage)


def test_draw_from_r_p_f_and_predictions_draw_lat_then_up():
    h, w = 90, 120
    img = _img(h, w, 12)
    out = viz.draw_from_r_p_f(img, 4.0, -10.0, 60.0, "deg")
    up = pc.PanoCam.get_up(math.radians(60), w, h, math.radians(-10), math.radians(4)).cpu().numpy()
    lat = np.radians(pc.PanoCam.get_lat(math.radians(60), w, h, math.radians(-10), math.radians(4)).cpu().numpy())
    _close(out, od.draw(od.draw(img, lat=lat), up=up, color=od.C0), "draw_from_r_p_f")
    assert np.array_equal(viz.draw_from_r_p_f(img, math.radians(4.0), math.radians(-10.0), math.radians(60.0), "rad"), out)
    preds = [{"pred_roll": torch.tensor(2.0), "pred_pitch": torch.tensor(8.0), "pred_general_vfov": torch.tensor(50.0),
              "pred_rel_cx": torch.tensor(0.0625), "pred_rel_cy": torch.tensor(-0.03125)}] * 2
    imgs = [img, _img(64, 80, 13)]
    drawn = viz.draw_predictions(imgs, preds)
    for im, d, p in zip(imgs, drawn, preds):
        one = viz.draw_from_r_p_f_cx_cy(im, 2.0, 8.0, 50.0, 0.0625, -0.03125, "deg", up_color=(0, 1, 0))
        assert np.array_equal(d, one)


def test_abi_rejects_bad_canvases():
    L = _native.lib()
    img = torch.zeros(16 * 16 * 3, dtype=torch.uint8, device="cuda")
    lat = torch.zeros(16 * 16, dtype=torch.float32, device="cuda")

    def call(**kw):
        c = _native.pf_draw_canvas(height=16, width=16, img_offset=0, out_offset=0, lat_offset=0, up_offset=-1, density=10,
                                   arrow_inv_len=20, alpha_fill=0.4, alpha_line=0.9, draw_lat=1, draw_up=0)
        for k, v in kw.items():
            setattr(c, k, v)
        cs = (_native.pf_draw_canvas * 1)(c)
        before = L.pf_kernel_launch_count()
        r = L.pf_draw_fields(0, cs, 1, img.data_ptr(), img.data_ptr(), lat.data_ptr(), None, None)
        assert L.pf_kernel_launch_count() == before
        return r

    assert call(height=0) == -1
    assert call(img_offset=-3) == -1
    assert call(lat_offset=-1) == -1
    assert call(alpha_fill=1.5) == -1
    assert call(draw_up=1) == -1                    # no up field
    assert L.pf_draw_fields(0, None, 1, img.data_ptr(), img.data_ptr(), None, None, None) == -1


def test_pinhole_fields_match_reference_golden():
    g = np.load(os.path.join(GOLD, "pinhole.npz"))
    for i, (vfov, w, h, el, roll) in enumerate(g["cases"]):
        up = pc.PanoCam.get_up(vfov, int(w), int(h), el, roll)
        lat = pc.PanoCam.get_lat(vfov, int(w), int(h), el, roll)
        assert up.is_cuda and up.dtype == torch.float32 and tuple(up.shape) == (int(h), int(w), 2)
        tol = 1e-5 if el == 0 else 2e-6               # the 1e8 px far point: ~5e-6 of direction variation float32 cannot hold
        assert np.abs(up.cpu().numpy() - g[f"up{i}"]).max() < tol, i
        assert np.abs(lat.cpu().numpy() - g[f"lat{i}"]).max() < 2e-5, i
