"""Visualisation hand-off on the GPU (SURVEY.md 8f-4): what the reference's demo does to the predicted fields between the path
and matplotlib -- ``resize_fix_aspect_ratio`` (demo/demo.py:30-51: ``cv2.resize`` of the up field and the latitude map to a
640-pixel-wide canvas) and the arrow grid of ``draw_perspective_fields`` / ``draw_up_field`` (utils/utils.py:190-200,
:236-247: ``up[y, x] * arrow_len`` on a ``density`` x ``density`` lattice) -- evaluated on the device, so that only the
canvas-sized latitude map (for the contour plot) and a few hundred arrow coordinates cross PCIe instead of the full-resolution
fields (37 MB per 2048x1536 image).

The resampling is ``pf_op_resize_f32`` (bilinear, pixel-centre aligned, no antialias: the sampling positions of
``cv2.resize(..., INTER_LINEAR)`` and of ``F.interpolate(align_corners=False)`` coincide).  No CPU path.

The drawing itself: ``draw_perspective_fields``, ``draw_up_field``, ``draw_latitude_field``, ``draw_from_r_p_f`` and
``draw_from_r_p_f_cx_cy`` are drop-ins for the reference's functions of the same names (utils/utils.py:165-430: same
signatures and defaults), rasterised by ``pf_draw_fields`` (csrc/draw.cuh) instead of matplotlib, by the rule of DESIGN.md
section 1 (parity with matplotlib unpinned).  Numpy images give numpy results, CUDA uint8 tensors give CUDA uint8 tensors.
``draw_fields_batch`` draws a list in one library call; ``draw_predictions`` draws ``inference_batch`` results as the demo's
ParamNet panel.  No CPU path.
"""
import math
import os

import numpy as np
import torch

from . import _batch, _native
from . import panocam


def _resize_plane(t, th, tw):
    """[H, W] float32 CUDA tensor -> [th, tw]."""
    L = _native.lib()
    t = t.contiguous()
    out = torch.empty((th, tw), dtype=torch.float32, device=t.device)
    stream = torch.cuda.current_stream(t.device).cuda_stream
    _native.check(L.pf_op_resize_f32(t.data_ptr(), t.shape[0], t.shape[1], 1, th, tw, out.data_ptr(), stream))
    return out


def target_size(height, width, target_width=None, target_height=None):
    """demo/demo.py:30-40: the canvas size ``resize_fix_aspect_ratio`` picks."""
    if target_width is None and target_height is None:
        raise ValueError("target_width or target_height must be given")
    if target_height is None:
        factor = target_width / width
    elif target_width is None:
        factor = target_height / height
    else:
        factor = max(target_width / width, target_height / height)
    if target_width is not None and factor == target_width / width:
        target_height = int(height * factor)
    else:
        target_width = int(width * factor)
    return target_height, target_width


def resize_fields(up, lati, target_width=640, target_height=None):
    """``resize_fix_aspect_ratio`` for the fields (demo/demo.py:41-51): ``up`` [2, H, W] and ``lati`` [H, W] CUDA tensors ->
    ([2, th, tw], [th, tw]) CUDA tensors."""
    if up.device.type != "cuda":
        raise RuntimeError("perspectivefields_b200.viz needs CUDA tensors (there is no CPU path)")
    h, w = lati.shape
    th, tw = target_size(h, w, target_width, target_height)
    with torch.cuda.device(up.device):
        up_r = torch.stack([_resize_plane(up[0].float(), th, tw), _resize_plane(up[1].float(), th, tw)])
        lat_r = _resize_plane(lati.float(), th, tw)
    return up_r, lat_r


def arrow_grid(up, density=10, arrow_inv_len=20):
    """utils/utils.py:190-200: lattice ``x = arange(0, w, w // density)``, ``y = arange(0, h, h // density)``; arrows
    ``up[:, y, x] * (sqrt(w^2 + h^2) // arrow_inv_len)``, drawn with (u, -v).  ``up``: [2, H, W] (CUDA).  Returns host arrays
    x, y (int64) and u, v (float32, v already negated as ``draw_arrow`` receives it)."""
    _, h, w = up.shape
    xs = torch.arange(0, w, w // density, device=up.device)
    ys = torch.arange(0, h, h // density, device=up.device)
    yy, xx = torch.meshgrid(ys, xs, indexing="ij")          # np.meshgrid(x, y) ravel order: y outer, x inner
    x, y = xx.reshape(-1), yy.reshape(-1)
    arrow_len = math.sqrt(w ** 2 + h ** 2) // arrow_inv_len
    end = up[:, y, x] * arrow_len
    return x.cpu().numpy(), y.cpu().numpy(), end[0].cpu().numpy(), (-end[1]).cpu().numpy()


def handoff(pred, target_width=640, density=10, arrow_inv_len=20):
    """Everything ``demo.log_results`` needs from one prediction to draw ``perspective_pred`` (demo/demo.py:53-62): the latitude
    map in RADIANS on the canvas (host float32, for ``draw_lati``'s contours) and the arrow lattice of the up field."""
    up_r, lat_r = resize_fields(pred["pred_gravity_original"], pred["pred_latitude_original"], target_width)
    x, y, u, v = arrow_grid(up_r, density, arrow_inv_len)
    return {"latitude_rad": torch.deg2rad(lat_r).cpu().numpy(), "arrow_x": x, "arrow_y": y, "arrow_u": u, "arrow_v": v,
            "canvas_hw": tuple(lat_r.shape)}


# ---------------------------------------------------------------------------------------------------------------------------
# Drawing (utils/utils.py:165-430)

GREEN = (0.0, 1.0, 0.0)                                      # draw_perspective_fields' colour for color=None (utils.py:200-201)
C0 = (0x1F / 255.0, 0x77 / 255.0, 0xB4 / 255.0)              # matplotlib's default face colour: quiver(color=None)


class DrawnImage:
    """What the reference's ``draw_*`` return with ``return_img=False`` (its ``VisImage``): ``get_image()`` and ``save(path)``."""

    def __init__(self, img):
        self._img = img

    def get_image(self):
        """The drawn canvas: numpy uint8 [H, W, 3] RGB, or a CUDA uint8 tensor when the input image was one."""
        return self._img

    def save(self, filepath):
        """Write the canvas as an image file, PNG when the path has no extension (``.png`` is appended, as ``savefig`` does)."""
        from PIL import Image

        path = os.fspath(filepath)
        if not os.path.splitext(path)[1]:
            path += ".png"
        img = self._img.cpu().numpy() if isinstance(self._img, torch.Tensor) else self._img
        Image.fromarray(np.ascontiguousarray(img)).save(path)


def _check_image(img, i):
    if isinstance(img, torch.Tensor):
        if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
            raise ValueError(f"image {i}: expected a uint8 [H, W, 3] tensor, got {img.dtype} {list(img.shape)}")
        return img
    img = np.asarray(img)
    if img.ndim != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError(f"image {i}: expected an [H, W, 3] image, got shape {list(img.shape)}")
    if img.dtype.kind not in "uif":
        raise ValueError(f"image {i}: expected a numeric image, got {img.dtype}")
    return img.astype(np.uint8, copy=False)                   # VisImage.reset_image: img.astype("uint8")


def _check_up(up, h, w, i):
    """[2, H, W] torch tensor (the reference's torch branch) or [H, W, 2] (numpy, or a tensor such as PanoCam.get_up's) ->
    float32 tensor ([H, W, 2] view) or numpy array."""
    if isinstance(up, torch.Tensor):
        t = _batch.up_view(up, h, w)
        if t is None:
            raise ValueError(f"up field {i}: expected [2, {h}, {w}] or [{h}, {w}, 2], got {list(up.shape)}")
        if not t.is_floating_point():
            raise ValueError(f"up field {i}: expected a float tensor, got {t.dtype}")
        return t
    a = np.asarray(up)
    if a.shape != (h, w, 2) or a.dtype.kind not in "uif":
        raise ValueError(f"up field {i}: expected a numeric [{h}, {w}, 2] array, got {a.dtype} {list(a.shape)}")
    return a


def _check_lat(lat, h, w, i):
    shape = tuple(lat.shape) if isinstance(lat, torch.Tensor) else np.shape(lat)
    if tuple(shape) != (h, w):
        raise ValueError(f"latitude map {i}: expected [{h}, {w}], got {list(shape)}")
    return lat


def _check_color(color, default):
    color = default if color is None else tuple(color)
    if len(color) != 3:
        raise ValueError(f"color must be an (r, g, b) triple in [0, 1], got {color!r}")
    return tuple(_batch.unit(c, "color component") for c in color)


def _check_lattice(density, arrow_inv_len, h, w, i):
    _batch.positive_int(density, "density")
    _batch.positive_int(arrow_inv_len, "arrow_inv_len")
    if w // density == 0 or h // density == 0:
        raise ValueError(f"canvas {i} ({h} x {w}): density {density} leaves no arrow step (W // density or H // density is 0)")


def _on_device(items, dtype, dev):
    """Host arrays / CPU tensors of a list -> one packed upload; CUDA tensors of ``dtype`` stay where they are."""
    out, host = list(items), []
    for k, t in enumerate(items):
        if t is None:
            continue
        if isinstance(t, torch.Tensor) and t.is_cuda:
            if t.device != dev:
                raise ValueError(f"all tensors must be on {dev}, got one on {t.device}")
            if t.dtype != dtype:
                out[k] = t.to(dtype)
        else:
            host.append(k)
    if host:
        arrs = [items[k].cpu().numpy() if isinstance(items[k], torch.Tensor) else items[k] for k in host]
        for k, t in zip(host, _batch.upload(arrs, dtype, dev)):
            out[k] = t
    return out


def _draw(imgs, ups, lats, colors, density, arrow_inv_len, alpha_fill, alpha_line, in_place=False):
    """Checked inputs -> list of CUDA uint8 [H, W, 3] canvases drawn by one pf_draw_fields call.  ``in_place``: the images are
    CUDA tensors that receive the drawing."""
    n = len(imgs)
    dev = _batch.device(__name__, list(imgs) + [u for u in ups if u is not None] + [l for l in lats if l is not None])
    L = _native.lib()
    with torch.cuda.device(dev):
        imgs_d = _on_device(imgs, torch.uint8, dev)
        lats_d = _on_device(lats, torch.float32, dev)
        ups_d = _on_device(ups, torch.float32, dev)
        imgs_d = [t if t.is_contiguous() else t.contiguous() for t in imgs_d]
        lats_d = [t if t is None or t.is_contiguous() else t.contiguous() for t in lats_d]
        if in_place:
            outs = imgs_d
        else:
            offs, total = _batch.layout([t.numel() for t in imgs_d])
            outs = _batch.views(torch.empty(total, dtype=torch.uint8, device=dev), offs, [t.shape for t in imgs_d])
        ib, ob, lb, ub = _batch.base(imgs_d), _batch.base(outs), _batch.base(lats_d), _batch.base(ups_d)
        descs = (_native.pf_draw_canvas * n)()
        for k in range(n):
            h, w = imgs_d[k].shape[:2]
            d = descs[k]
            d.height, d.width = h, w
            d.img_offset, d.out_offset = _batch.offset(imgs_d[k], ib), _batch.offset(outs[k], ob)
            d.alpha_fill, d.alpha_line = alpha_fill, alpha_line
            d.lat_offset, d.up_offset = _batch.offset(lats_d[k], lb), _batch.offset(ups_d[k], ub)
            d.draw_lat = int(lats_d[k] is not None)
            if ups_d[k] is not None:
                d.draw_up, d.up_stride[:] = 1, ups_d[k].stride()
                d.density, d.arrow_inv_len = int(density), int(arrow_inv_len)
                d.arrow_rgb[:] = colors[k]
        ptr = lambda b: b if b else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_draw_fields(dev.index, descs, n, ib, ob, ptr(lb), ptr(ub), stream))
    return outs


def _finish(outs, imgs, return_img=True):
    """Device canvases -> numpy for numpy inputs (one copy), CUDA tensors for CUDA inputs; ``DrawnImage`` when not return_img."""
    host = [k for k, im in enumerate(imgs) if not isinstance(im, torch.Tensor)]
    res = list(outs)
    if host:
        flat = torch.cat([outs[k].reshape(-1) for k in host]).cpu().numpy()
        off = 0
        for k in host:
            s = outs[k].numel()
            res[k] = flat[off:off + s].reshape(tuple(outs[k].shape))
            off += s
    return res if return_img else [DrawnImage(r) for r in res]


def draw_fields_batch(imgs, ups=None, lats=None, color=None, density=10, arrow_inv_len=20, alpha_contourf=0.4, alpha_contour=0.9):
    """``draw_perspective_fields`` for a list of canvases in ONE library call (sizes may differ).  ``imgs``: RGB [H, W, 3]
    (numpy or CUDA uint8); ``ups``: per canvas an up field ([2, H, W] tensor or [H, W, 2]) or None for no arrows; ``lats``: per
    canvas a latitude map in RADIANS [H, W] or None for no contours.  ``color`` None draws (0, 1, 0).  Returns a list of
    numpy arrays / CUDA tensors like the inputs."""
    n = len(imgs)
    if n == 0:
        return []
    ups = [None] * n if ups is None else list(ups)
    lats = [None] * n if lats is None else list(lats)
    if len(ups) != n or len(lats) != n:
        raise ValueError(f"{n} images but {len(ups)} up fields and {len(lats)} latitude maps")
    imgs = [_check_image(im, k) for k, im in enumerate(imgs)]
    col = _check_color(color, GREEN)
    af, al = _batch.unit(alpha_contourf, "alpha_contourf"), _batch.unit(alpha_contour, "alpha_contour")
    for k, im in enumerate(imgs):
        h, w = im.shape[:2]
        if ups[k] is not None:
            _check_lattice(density, arrow_inv_len, h, w, k)
            ups[k] = _check_up(ups[k], h, w, k)
        if lats[k] is not None:
            lats[k] = _check_lat(lats[k], h, w, k)
    return _finish(_draw(imgs, ups, lats, [col] * n, density, arrow_inv_len, af, al), imgs)


def draw_perspective_fields(img_rgb, up, latimap, color=None, density=10, arrow_inv_len=20, return_img=True):
    """utils/utils.py:165-206: latitude contours (alpha 0.4 / 0.9), then the up-vector arrows ((0, 1, 0) for color=None) with the
    contour lines over them.  ``up``: [2, H, W] tensor or [H, W, 2]; ``latimap``: [H, W] radians."""
    img = _check_image(img_rgb, 0)
    h, w = img.shape[:2]
    _check_lattice(density, arrow_inv_len, h, w, 0)
    up = _check_up(up, h, w, 0)
    lat = _check_lat(latimap, h, w, 0)
    col = _check_color(color, GREEN)
    return _finish(_draw([img], [up], [lat], [col], density, arrow_inv_len, 0.4, 0.9), [img], return_img)[0]


def draw_up_field(img_rgb, vector_field, color=None, density=10, arrow_inv_len=20, return_img=True):
    """utils/utils.py:209-250: the up-vector arrows alone (matplotlib's default colour C0 for color=None)."""
    img = _check_image(img_rgb, 0)
    h, w = img.shape[:2]
    _check_lattice(density, arrow_inv_len, h, w, 0)
    up = _check_up(vector_field, h, w, 0)
    col = _check_color(color, C0)
    return _finish(_draw([img], [up], [None], [col], density, arrow_inv_len, 0.4, 0.9), [img], return_img)[0]


def draw_latitude_field(img_rgb, latimap=None, binmap=None, alpha_contourf=0.4, alpha_contour=0.9, return_img=True):
    """utils/utils.py:403-429: the latitude contours alone.  ``latimap``: [H, W] radians (``binmap`` is deprecated, unused)."""
    img = _check_image(img_rgb, 0)
    if latimap is None:
        raise ValueError("latimap is required")
    lat = _check_lat(latimap, img.shape[0], img.shape[1], 0)
    af, al = _batch.unit(alpha_contourf, "alpha_contourf"), _batch.unit(alpha_contour, "alpha_contour")
    return _finish(_draw([img], [None], [lat], [None], 10, 20, af, al), [img], return_img)[0]


def _radians(mode, *angles):
    if mode == "deg":
        return [math.radians(float(a)) for a in angles]
    if mode == "rad":
        return [float(a) for a in angles]
    raise ValueError("Bad argument")


def _draw_lat_then_up(imgs, ups, lats_deg, up_color, alpha_contourf, alpha_contour, draw_up, draw_lat):
    """draw_from_r_p_f*'s two steps on device fields: draw_latitude_field, then draw_up_field over ITS result (the arrows go over
    the contour lines here, utils.py:312-320), the second call drawing in place."""
    af, al = _batch.unit(alpha_contourf, "alpha_contourf"), _batch.unit(alpha_contour, "alpha_contour")
    col = _check_color(up_color, C0)
    n = len(imgs)
    cur = list(imgs)
    if draw_lat:
        cur = _draw(cur, [None] * n, [torch.deg2rad(l) for l in lats_deg], [None] * n, 10, 20, af, al)
    if draw_up:
        cur = _draw(cur, ups, [None] * n, [col] * n, 10, 20, af, al, in_place=draw_lat)
    if not draw_lat and not draw_up:
        return [im.copy() if isinstance(im, np.ndarray) else im.clone() for im in imgs]
    return _finish(cur, imgs)


def draw_from_r_p_f(img, roll, pitch, vfov, mode, up_color=None, alpha_contourf=0.4, alpha_contour=0.9, draw_up=True, draw_lat=True,
                    lati_alpha=0.5):
    """utils/utils.py:253-321: the fields of a pinhole camera (``PanoCam.get_lat`` / ``get_up``) drawn over ``img``.
    ``lati_alpha`` is deprecated and unused, as in the reference."""
    img = _check_image(img, 0)
    roll, pitch, vfov = _radians(mode, roll, pitch, vfov)
    h, w = img.shape[:2]
    if draw_up:
        _check_lattice(10, 20, h, w, 0)
    dev = _batch.device(__name__, [img])
    ups, lats = panocam.pinhole_fields([vfov], [h], [w], [pitch], [roll], dev, up=True, lat=True)
    return _draw_lat_then_up([img], ups, lats, up_color, alpha_contourf, alpha_contour, draw_up, draw_lat)[0]


def draw_from_r_p_f_cx_cy(img, roll, pitch, vfov, rel_cx, rel_cy, mode, up_color=None, alpha_contourf=0.4, alpha_contour=0.9,
                          draw_up=True, draw_lat=True):
    """utils/utils.py:324-400: the fields of a camera with an off-centre principal point (``get_lat_general`` /
    ``get_up_general``, focal length from the general vertical field of view) drawn over ``img``."""
    img = _check_image(img, 0)
    roll, pitch, vfov = _radians(mode, roll, pitch, vfov)
    h, w = img.shape[:2]
    if draw_up:
        _check_lattice(10, 20, h, w, 0)
    dev = _batch.device(__name__, [img])
    focal = panocam.general_vfov_to_focal(rel_cx, rel_cy, 1, vfov, False)
    ups, lats = panocam.camera_fields([float(focal)], [h], [w], [pitch], [roll], [float(rel_cx)], [float(rel_cy)], dev)
    return _draw_lat_then_up([img], ups, lats, up_color, alpha_contourf, alpha_contour, draw_up, draw_lat)[0]


def draw_predictions(imgs, preds, up_color=GREEN, alpha_contourf=0.4, alpha_contour=0.9, draw_up=True, draw_lat=True):
    """The demo's ParamNet panel (demo/demo.py:64-75: ``draw_from_r_p_f_cx_cy(img, roll, pitch, general vfov, rel_cx, rel_cy,
    "deg", up_color=(0, 1, 0))``) for a list of ``inference_batch`` results, at each image's own size: the fields of all images
    in one ``fields_from_predictions`` call, then two library calls for the whole list.  Resizing the images (the demo's
    640-wide canvas, ``target_size``) is the caller's, as in the reference."""
    if len(imgs) != len(preds):
        raise ValueError(f"{len(imgs)} images but {len(preds)} predictions")
    if not imgs:
        return []
    imgs = [_check_image(im, k) for k, im in enumerate(imgs)]
    _check_color(up_color, C0)
    if draw_up:
        for k, im in enumerate(imgs):
            _check_lattice(10, 20, im.shape[0], im.shape[1], k)
    dev = _batch.device(__name__, imgs)
    ups, lats = panocam.fields_from_predictions(preds, [im.shape[:2] for im in imgs], "deg", dev)
    return _draw_lat_then_up(imgs, ups, lats, up_color, alpha_contourf, alpha_contour, draw_up, draw_lat)
