"""Camera parameters -> dense perspective fields on the GPU (SURVEY.md 8f-1, the step callers run right after the
inference path): drop-in for the two static methods of the reference's ``perspective2d.utils.panocam.PanoCam`` that turn
ParamNet's output into an up-vector field and a latitude map (utils/panocam.py:451-556; called from
utils/utils.py:367-385 and demo/demo.py:69-78).

Also ``PanoCam.crop_distortion`` (utils/panocam.py:559-752, the reference's notebooks/camera2perspective.ipynb workflow): a
perspective or Unified Spherical Model view cropped from an equirectangular panorama with its ground-truth fields, and its batched
form ``crop_distortion_views``, whose crops can go straight into ``PerspectiveFields.inference_batch`` on the device.

And the pinhole crop of that workflow: ``PanoCam.crop_equi``, ``PanoCam(pano_path).get_image`` with its horizon line and vertical
vanishing point (utils/panocam.py:121-382), and the batched ``crop_equi_views``, under the crop rule of DESIGN.md section 1.

Same names, argument order and meaning as the reference.  Differences: results are float32 CUDA tensors (the reference returns
float64 numpy arrays), and ``camera_fields`` evaluates a whole batch (images may differ in size) in one launch per 24 images.
There is no CPU path: the functions raise when the CUDA library or a CUDA device is missing.
"""
import ctypes
import math
import os

import numpy as np
import torch

from . import _batch, _native


def general_vfov(d_cx, d_cy, h, focal, degree):
    """utils/utils.py:13-44: the general vertical field of view, the angle at the pinhole between the rays through the
    midpoints of the image's top and bottom edges, for a principal point offset (d_cx, d_cy) from the centre.  Lengths relative
    to the image height (h = 1) or in pixels (h = the height).  The inverse of ``general_vfov_to_focal``.  Scalars or numpy
    arrays (float64), or torch tensors (computed with torch ops on their device, without synchronising)."""
    xp = torch if any(isinstance(v, torch.Tensor) for v in (d_cx, d_cy, focal)) else np
    p_sqr = focal ** 2 + d_cx ** 2 + (d_cy + 0.5 * h) ** 2
    q_sqr = focal ** 2 + d_cx ** 2 + (d_cy - 0.5 * h) ** 2
    cos_fov = (p_sqr + q_sqr - h ** 2) / 2 / xp.sqrt(p_sqr) / xp.sqrt(q_sqr)
    fov = xp.arccos(cos_fov)
    return xp.rad2deg(fov) if degree else fov


def general_vfov_to_focal(rel_cx, rel_cy, h, gvfov, degree):
    """utils/utils.py:47-91 (SciPy ``fsolve`` there): relative focal length from the general vertical field of view, the
    angle between the rays through the top-centre and bottom-centre pixels, for an off-centre principal point.  Closed form
    (DESIGN.md section 4): with c = cos(gvfov), A = f^2 + cx^2 + cy^2 + h^2/4:  4 (c^2 - 1) A^2 + 4 h^2 A - h^2 (h^2 + 4 c^2 cy^2) = 0,
    root with sign(2A - h^2) = sign(c).  Scalars or arrays; float64."""
    cx, cy, g = np.asarray(rel_cx, np.float64), np.asarray(rel_cy, np.float64), np.asarray(gvfov, np.float64)
    if degree:
        g = np.radians(g)
    c = np.cos(g)
    h = float(h)
    # p^2 = f^2 + cx^2 + (cy + h/2)^2 = A + h cy,  q^2 = A - h cy,  cos(gvfov) = (p^2 + q^2 - h^2) / (2 p q)
    # => (2A - h^2)^2 = 4 c^2 (A^2 - h^2 cy^2), a quadratic in A; squaring adds the root of the supplementary angle, which
    #    the sign condition removes
    a2 = 4.0 * (c * c - 1.0)
    a1 = 4.0 * h * h
    a0 = -(h ** 4 + 4.0 * c * c * h * h * cy * cy)
    disc = np.sqrt(np.maximum(a1 * a1 - 4.0 * a2 * a0, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        r1, r2 = (-a1 + disc) / (2.0 * a2), (-a1 - disc) / (2.0 * a2)
        pick = np.where(np.sign(2.0 * r1 - h * h) == np.sign(c), r1, r2)
        lin = -a0 / a1                                   # c^2 == 1 never happens for a real field of view; guard anyway
        A = np.where(np.abs(a2) < 1e-300, lin, pick)
        f2 = A - cx * cx - cy * cy - h * h / 4.0
        return np.sqrt(f2)


def camera_fields(focal_rel, heights, widths, elevation, roll, cx_rel, cy_rel, device=None, up=True, lat=True, vp=None):
    """Batched ``get_up_general`` / ``get_lat_general``: every argument is a sequence of length n (radians for the angles).
    ``vp``: None or a sequence of n (x, y) points in pixel-centre coordinates (pixel (i, j) at (j + .5, i + .5)) that the up
    fields point to instead, (nan, nan) keeping the camera's own (``PanoCam.get_up`` at elevation 0).
    Returns (list of [H_i, W_i, 2] float32 tensors or None, list of [H_i, W_i] float32 tensors in degrees or None)."""
    L = _native.lib()
    dev = _batch.device(__name__, (), device)
    n = len(heights)
    sizes = [(int(h), int(w)) for h, w in zip(heights, widths)]
    up_offs, up_total = _batch.layout([2 * h * w for h, w in sizes])
    lat_offs, lat_total = _batch.layout([h * w for h, w in sizes])
    cams = (_native.pf_camera * n)()
    for i, (h, w) in enumerate(sizes):
        cams[i] = _native.pf_camera(h, w, float(focal_rel[i]), float(elevation[i]), float(roll[i]), float(cx_rel[i]), float(cy_rel[i]),
                                    up_offs[i], lat_offs[i])
    with torch.cuda.device(dev):
        up_blob = torch.empty(up_total, dtype=torch.float32, device=dev) if up else None
        lat_blob = torch.empty(lat_total, dtype=torch.float32, device=dev) if lat else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        up_ptr, lat_ptr = up_blob.data_ptr() if up else None, lat_blob.data_ptr() if lat else None
        if vp is None:
            _native.check(L.pf_camera_fields(dev.index, cams, n, up_ptr, lat_ptr, stream))
        else:
            vps = (ctypes.c_double * (2 * n))(*[float(c) for p in vp for c in p])
            _native.check(L.pf_camera_fields_vp(dev.index, cams, vps, n, up_ptr, lat_ptr, stream))
    ups = _batch.views(up_blob, up_offs, [(h, w, 2) for h, w in sizes]) if up else None
    lats = _batch.views(lat_blob, lat_offs, sizes) if lat else None
    return ups, lats


PANO_OUTPUTS = ("ntheta", "nphi", "up", "lat", "xy_map")


def _check_view(view, i):
    """(f, xi, H, W, az, el, roll) -- crop_distortion's argument order -- or a dict with those keys -> checked tuple."""
    keys = ("f", "xi", "H", "W", "az", "el", "roll")
    if isinstance(view, dict):
        missing = [k for k in keys if k not in view]
        if missing:
            raise ValueError(f"view {i}: missing {missing}")
        view = [view[k] for k in keys]
    view = tuple(view)
    if len(view) != 7:
        raise ValueError(f"view {i}: expected (f, xi, H, W, az, el, roll), got {len(view)} values")
    f, xi, h, w, az, el, roll = view
    f = _batch.real(f, f"view {i}: f")
    if f <= 0:
        raise ValueError(f"view {i}: f must be > 0, got {f}")
    return (f, _batch.real(xi, f"view {i}: xi"), _batch.positive_int(h, f"view {i}: H"), _batch.positive_int(w, f"view {i}: W"), _batch.real(az, f"view {i}: az"),
            _batch.real(el, f"view {i}: el"), _batch.real(roll, f"view {i}: roll"))


def _check_panorama(image360):
    """numpy / torch uint8 [Hp, Wp, 3] or a path (read with Pillow as RGB, what imageio.imread returns for an 8-bit file) ->
    the array or tensor, checked; no GPU work."""
    if isinstance(image360, (str, os.PathLike)):
        from PIL import Image
        with Image.open(image360) as im:
            image360 = np.array(im.convert("RGB"))
    if isinstance(image360, torch.Tensor):
        if image360.dtype != torch.uint8:
            raise TypeError(f"the panorama must be uint8, got {image360.dtype}")
        shape = tuple(image360.shape)
    else:
        image360 = np.asarray(image360)
        if image360.dtype != np.uint8:
            raise TypeError(f"the panorama must be uint8, got {image360.dtype}")
        shape = image360.shape
    if len(shape) != 3 or shape[2] != 3:
        raise TypeError(f"the panorama must be [H, W, 3], got {list(shape)}")
    if shape[0] < 2 or shape[1] < 2:
        raise ValueError(f"the panorama must be at least 2 x 2, got {shape[0]} x {shape[1]}")
    return image360


def crop_distortion_views(image360, views, outputs=("up", "lat"), device=None):
    """Batched ``PanoCam.crop_distortion`` (utils/panocam.py:559-752): many views of ONE panorama, one upload, one launch per 12 views,
    no synchronisation.  ``views``: sequence of ``(f, xi, H, W, az, el, roll)`` (or dicts with those keys; sizes may differ);
    ``outputs``: any of ``ntheta, nphi, up, lat, xy_map``.  Returns a dict: ``im`` (list of uint8 [H, W, 3] views into one device
    blob, the panorama's channel order), one list of float32 tensors per selected output ([H, W] radians or [H, W, 2]), ``offset``
    (float64 [n], the horizon row at column W // 2, nan without a zero crossing) and ``status`` (int32 [n]: 0 fine, 1 several zero
    crossings (the reference warns), 2 the reference's assertions fail) as device tensors."""
    outputs = tuple(outputs)
    bad = [o for o in outputs if o not in PANO_OUTPUTS]
    if bad:
        raise ValueError(f"unknown outputs {bad}; choose from {PANO_OUTPUTS}")
    vs = [_check_view(v, i) for i, v in enumerate(views)]
    if not vs:
        raise ValueError("no views")
    pano = _check_panorama(image360)
    dev = _pano_device(pano, device)
    L = _native.lib()
    n = len(vs)
    # 16-byte aligned crops and 4-float aligned fields: full-width vector stores
    im_offs, im_total = _batch.layout([3 * v[2] * v[3] for v in vs], 16)
    fld_offs, fld_total = _batch.layout([v[2] * v[3] for v in vs], 4)
    descs = (_native.pf_pano_view * n)()
    for i, (f, xi, h, w, az, el, roll) in enumerate(vs):
        descs[i] = _native.pf_pano_view(h, w, f, xi, az, el, roll, im_offs[i], fld_offs[i])
    with torch.cuda.device(dev):
        src = torch.as_tensor(pano).to(dev).contiguous()
        im = torch.empty(im_total, dtype=torch.uint8, device=dev)
        blobs = {o: torch.empty((2 if o in ("up", "xy_map") else 1) * fld_total, dtype=torch.float32, device=dev) for o in outputs}
        offset = torch.empty(n, dtype=torch.float64, device=dev)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        ptr = lambda o: blobs[o].data_ptr() if o in blobs else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_pano_views(dev.index, src.data_ptr(), src.shape[0], src.shape[1], descs, n, im.data_ptr(), ptr("ntheta"),
                                      ptr("nphi"), ptr("up"), ptr("lat"), ptr("xy_map"), offset.data_ptr(), status.data_ptr(), stream))
    hw = [(v[2], v[3]) for v in vs]
    out = {"im": _batch.views(im, im_offs, [(h, w, 3) for h, w in hw])}
    for o in outputs:
        two = o in ("up", "xy_map")
        out[o] = _batch.views(blobs[o], [2 * f for f in fld_offs] if two else fld_offs, [(h, w, 2) if two else (h, w) for h, w in hw])
    out["offset"], out["status"] = offset, status
    return out


EQUI_MODES = {"bilinear": _native.PF_EQUI_BILINEAR, "nearest": _native.PF_EQUI_NEAREST}


def _rad(deg):
    return deg / 180 * math.pi          # the reference's expression (utils/panocam.py:171-173, :188-193)


def _check_equi_view(view, i):
    """(vfov, im_w, im_h, azimuth, elevation, roll, ar) -- crop_equi's argument order -- or a dict with those keys -> checked tuple."""
    keys = ("vfov", "im_w", "im_h", "azimuth", "elevation", "roll", "ar")
    if isinstance(view, dict):
        missing = [k for k in keys if k not in view]
        if missing:
            raise ValueError(f"view {i}: missing {missing}")
        view = [view[k] for k in keys]
    view = tuple(view)
    if len(view) != 7:
        raise ValueError(f"view {i}: expected (vfov, im_w, im_h, azimuth, elevation, roll, ar), got {len(view)} values")
    vfov, w, h, az, el, roll, ar = view
    vfov, ar = _batch.real(vfov, f"view {i}: vfov"), _batch.real(ar, f"view {i}: ar")
    if not 0.0 < vfov < 180.0:
        raise ValueError(f"view {i}: vfov must lie in (0, 180) degrees, got {vfov}")
    if ar <= 0.0:
        raise ValueError(f"view {i}: ar must be > 0, got {ar}")
    fov_x = 2 * math.atan(math.tan(vfov * math.pi / 180.0 / 2) * ar) * 180 / math.pi
    if not fov_x < 180.0:
        raise ValueError(f"view {i}: the horizontal field of view 2 atan(tan(vfov / 2) ar) = {fov_x} degrees must be < 180")
    return (vfov, _batch.positive_int(w, f"view {i}: im_w"), _batch.positive_int(h, f"view {i}: im_h"), _batch.real(az, f"view {i}: azimuth"),
            _batch.real(el, f"view {i}: elevation"), _batch.real(roll, f"view {i}: roll"), ar)


def _check_equi_panorama(equi_img):
    """numpy / torch uint8 or float32 [Hp, Wp] or [Hp, Wp, 3] -> (array or tensor, dtype code, channels); no GPU work."""
    if isinstance(equi_img, torch.Tensor):
        codes = {torch.uint8: _native.PF_EQUI_U8, torch.float32: _native.PF_EQUI_F32}
    else:
        equi_img = np.asarray(equi_img)
        codes = {np.dtype(np.uint8): _native.PF_EQUI_U8, np.dtype(np.float32): _native.PF_EQUI_F32}
    if equi_img.dtype not in codes:
        raise TypeError(f"the panorama must be uint8 or float32, got {equi_img.dtype}")
    shape = tuple(equi_img.shape)
    if len(shape) not in (2, 3) or (len(shape) == 3 and shape[2] != 3):
        raise TypeError(f"the panorama must be [H, W] or [H, W, 3], got {list(shape)}")
    if shape[0] < 1 or shape[1] < 1:
        raise ValueError(f"the panorama must be at least 1 x 1, got {shape[0]} x {shape[1]}")
    return equi_img, codes[equi_img.dtype], 1 if len(shape) == 2 else 3


def _pano_device(pano, device):
    """The CUDA device a call runs on: the panorama's own when it is a CUDA tensor (``device`` must agree), else ``device`` or the
    current one."""
    if isinstance(pano, torch.Tensor) and pano.is_cuda and device is not None and torch.device(device) != pano.device:
        raise ValueError(f"the panorama is on {pano.device}, not on {device}")
    return _batch.device(__name__, [pano], device)


def horizon_vvp(vfov, im_w, im_h, elevation, roll):
    """get_image's horizon line and relative vertical vanishing point (utils/panocam.py:188-193), degrees in; the reference's tuples."""
    args = (_rad(elevation), _rad(roll), _rad(vfov), im_h, im_w)
    return PanoCam.getRelativeHorizonLineFromAngles(*args), PanoCam.getRelativeVVP(*args)


def _equi_views(equi_img, views, outputs, mode, img_format, unit, device):
    outputs = tuple(outputs)
    bad = [o for o in outputs if o not in ("up", "lat")]
    if bad:
        raise ValueError(f"unknown outputs {bad}; choose from ('up', 'lat')")
    if mode not in EQUI_MODES:
        raise ValueError(f"unknown mode {mode!r}; choose from {tuple(EQUI_MODES)}")
    if img_format not in ("RGB", "BGR"):
        raise ValueError(f"unknown img_format {img_format!r}; choose 'RGB' or 'BGR'")
    vs = [_check_equi_view(v, i) for i, v in enumerate(views)]
    if not vs:
        raise ValueError("no views")
    pano, dtype, channels = _check_equi_panorama(equi_img)
    swap = img_format == "BGR"
    if swap and channels != 3:
        raise ValueError("img_format='BGR' needs a 3-channel panorama")
    if unit and dtype != _native.PF_EQUI_U8:
        raise TypeError("get_image's crop needs a uint8 panorama")
    dev = _pano_device(pano, device)
    L = _native.lib()
    n = len(vs)
    tdt = torch.float32 if dtype == _native.PF_EQUI_F32 else torch.uint8
    esize = 4 if dtype == _native.PF_EQUI_F32 else 1
    shapes = [(v[2], v[1], 3) if channels == 3 else (v[2], v[1]) for v in vs]
    offs, total = _batch.layout([math.prod(s) * esize for s in shapes], 16)     # 16-byte aligned crops: full-width vector stores
    descs = (_native.pf_equi_view * n)()
    for i, (vfov, w, h, az, el, roll, ar) in enumerate(vs):
        descs[i] = _native.pf_equi_view(h, w, vfov, az, el, roll, ar, offs[i])
    with torch.cuda.device(dev):
        src = torch.as_tensor(pano).to(dev).contiguous()
        blob = torch.empty(total, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _native.check(L.pf_equi_views(dev.index, src.data_ptr(), src.shape[0], src.shape[1], channels, dtype, descs, n, EQUI_MODES[mode],
                                      _native.PF_EQUI_UNIT if unit else _native.PF_EQUI_CAST, int(swap), blob.data_ptr(), stream))
    out = {"im": _batch.views(blob.view(tdt), [o // esize for o in offs], shapes)}
    if outputs:
        ups, lats = pinhole_fields([_rad(v[0]) for v in vs], [v[2] for v in vs], [v[1] for v in vs], [_rad(v[4]) for v in vs],
                                   [_rad(v[5]) for v in vs], dev, up="up" in outputs, lat="lat" in outputs)
        out.update({k: f for k, f in (("up", ups), ("lat", lats)) if k in outputs})
    hv = [horizon_vvp(v[0], v[1], v[2], v[4], v[5]) for v in vs]
    out["horizon"] = np.array([h for h, _ in hv], np.float64).reshape(n, 2)
    out["vvp"] = np.array([tuple(p) + (math.nan,) * (3 - len(p)) for _, p in hv], np.float64).reshape(n, 3)
    return out


def crop_equi_views(equi_img, views, outputs=("up", "lat"), mode="bilinear", img_format="RGB", device=None):
    """Batched ``PanoCam.crop_equi`` (utils/panocam.py:196-249): pinhole views of ONE equirectangular panorama, one upload, one
    launch per 24 views, no synchronisation.  ``equi_img``: numpy / torch uint8 or float32 [Hp, Wp] or [Hp, Wp, 3]; ``views``:
    sequence of ``(vfov, im_w, im_h, azimuth, elevation, roll, ar)`` in degrees (or dicts with those keys; sizes may differ);
    ``outputs``: any of ``up, lat``; ``mode``: ``bilinear`` or ``nearest``; ``img_format="BGR"`` writes the channels in the order
    2, 1, 0.  Returns a dict: ``im`` (list of CUDA views into one 16-byte-aligned blob, in the panorama's dtype, [H, W, 3] or
    [H, W]; the uint8 [H, W, 3] crops are valid ``PerspectiveFields.inference_batch`` input), ``up`` / ``lat`` (lists of float32
    CUDA tensors: the reference's ``get_up`` / ``get_lat`` of each camera, ``lat`` in degrees), ``horizon`` (float64 [n, 2]) and
    ``vvp`` (float64 [n, 3]; ``(inf, inf, nan)`` for a view at elevation 0, where the reference returns ``(inf, inf)``) as host
    arrays."""
    return _equi_views(equi_img, views, outputs, mode, img_format, False, device)


class PanoCam:
    """``perspective2d.utils.panocam.PanoCam``: the panorama given as a path (``get_image``) and the static methods (same
    signatures), except ``getGravityField`` / ``getAbsVVP``."""

    def __init__(self, pano_path, device=None):
        """Reads the panorama once (Pillow, converted to RGB as the reference's ``preprocess`` does) and keeps it on the CUDA
        ``device`` (the reference re-reads the file on every ``get_image``)."""
        from PIL import Image
        self.pano_path = pano_path
        with Image.open(pano_path) as im:
            pano = np.array(im.convert("RGB"))
        self.device = _pano_device(None, device)
        self.pano = torch.from_numpy(pano).to(self.device)

    def get_image(self, vfov=85, im_w=640, im_h=480, azimuth=0, elevation=30, roll=0, ar=4.0 / 3.0, img_format="RGB"):
        """utils/panocam.py:132-194 -> (crop, horizon, vvp): the crop as a CUDA uint8 [im_h, im_w, 3] tensor in ``img_format``
        order (the reference returns a PIL image for RGB and a numpy array for BGR), computed as the reference's ToTensor ->
        sampler -> ToPILImage chain does; horizon and vvp are the reference's tuples."""
        crop = _equi_views(self.pano, [(vfov, im_w, im_h, azimuth, elevation, roll, ar)], (), "bilinear", img_format, True, self.device)["im"][0]
        horizon, vvp = horizon_vvp(vfov, im_w, im_h, elevation, roll)
        return crop, horizon, vvp

    @staticmethod
    def crop_equi(equi_img, vfov, im_w, im_h, azimuth, elevation, roll, ar, mode):
        """utils/panocam.py:196-249 -> CUDA tensor in the panorama's dtype, [im_h, im_w, 3] or [im_h, im_w] (degrees in)."""
        return crop_equi_views(equi_img, [(vfov, im_w, im_h, azimuth, elevation, roll, ar)], (), mode)["im"][0]

    @staticmethod
    def getRelativeVVP(elevation, roll, vfov, im_h, im_w):
        """utils/panocam.py:302-333 (radians): the vertical vanishing point over the image size and whether the up vectors point
        to it (+1) or away (-1); the 2-tuple (inf, inf) at elevation 0."""
        if elevation == 0:
            return np.inf, np.inf
        te, tv = np.tan(elevation), np.tan(vfov / 2)
        vx = 0.5 - 0.5 / im_w - 0.5 * np.sin(roll) / te / tv * im_h / im_w
        vy = 0.5 - 0.5 / im_h - 0.5 * np.cos(roll) / te / tv
        return vx, vy, np.sign(elevation)

    @staticmethod
    def getRelativeHorizonLineFromAngles(elevation, roll, vfov, im_h, im_w):
        """utils/panocam.py:335-351 (radians): the horizon's heights at the left and right image borders over the image height."""
        mid = PanoCam.getMidpointFromAngle(elevation, roll, vfov)
        dh = PanoCam.getDeltaHeightFromRoll(roll, im_h, im_w)
        return mid - dh, mid + dh

    @staticmethod
    def getMidpointFromAngle(elevation, roll, vfov):
        """utils/panocam.py:353-367 (radians): the horizon's height at the image centre over the image height; inf * sign at ±pi/2."""
        if elevation in (np.pi / 2, -np.pi / 2):
            return np.inf * np.sign(elevation)
        return 0.5 + 0.5 * np.tan(elevation) / np.cos(roll) / np.tan(vfov / 2)

    @staticmethod
    def getDeltaHeightFromRoll(roll, im_h, im_w):
        """utils/panocam.py:369-382 (radians): half the horizon's height change across the image over the image height; inf * sign
        at ±pi/2."""
        if roll in (np.pi / 2, -np.pi / 2):
            return np.inf * np.sign(roll)
        return -im_w / im_h * np.tan(roll) / 2

    @staticmethod
    def crop_distortion(image360, f, xi, H, W, az, el, roll, device=None):
        """utils/panocam.py:559-752 -> (im, ntheta, nphi, offset, up, lat, xy_map): CUDA tensors (uint8 [H, W, 3]; float32 [H, W]
        radians; float32 [H, W, 2]) and ``offset`` as a Python float (nan when the horizon does not cross column W // 2).
        ``image360``: numpy / CUDA uint8 [Hp, Wp, 3] or a path.  Prints the reference's WARNING when the horizon column crosses zero
        several times and raises AssertionError where the reference's assertions fail (e.g. an upside-down camera).  This call
        synchronises (for the offset); ``crop_distortion_views`` does not."""
        out = crop_distortion_views(image360, [(f, xi, H, W, az, el, roll)], PANO_OUTPUTS, device)
        status = int(out["status"][0].item())
        if status == 2:
            raise AssertionError("crop_distortion: the horizon column crosses zero from below (e.g. an upside-down camera)")
        nphi = out["nphi"][0]
        if status == 1:
            s = torch.sign(nphi[:, int(W) // 2])
            print("WARNING | Number of zero crossings:", int((s[1:] != s[:-1]).sum().item()))
        return (out["im"][0], out["ntheta"][0], nphi, float(out["offset"][0].item()), out["up"][0], out["lat"][0], out["xy_map"][0])

    @staticmethod
    def get_up(vfov, im_w, im_h, elevation, roll, device=None):
        """utils/panocam.py:422-448 (pinhole camera, centred principal point) -> float32 CUDA tensor [im_h, im_w, 2]."""
        return pinhole_fields([vfov], [im_h], [im_w], [elevation], [roll], device, up=True, lat=False)[0][0]

    @staticmethod
    def get_lat(vfov, im_w, im_h, elevation, roll, device=None):
        """utils/panocam.py:384-420 -> float32 CUDA tensor [im_h, im_w], degrees."""
        return pinhole_fields([vfov], [im_h], [im_w], [elevation], [roll], device, up=False, lat=True)[1][0]

    @staticmethod
    def get_up_general(focal_rel, im_w, im_h, elevation, roll, cx_rel, cy_rel, device=None):
        """utils/panocam.py:451-513 -> float32 CUDA tensor [im_h, im_w, 2]."""
        return camera_fields([focal_rel], [im_h], [im_w], [elevation], [roll], [cx_rel], [cy_rel], device, up=True, lat=False)[0][0]

    @staticmethod
    def get_lat_general(focal_rel, im_w, im_h, elevation, roll, cx_rel, cy_rel, device=None):
        """utils/panocam.py:515-556 -> float32 CUDA tensor [im_h, im_w], degrees."""
        return camera_fields([focal_rel], [im_h], [im_w], [elevation], [roll], [cx_rel], [cy_rel], device, up=False, lat=True)[1][0]


def far_vanishing_point(im_w, im_h, roll):
    """utils/panocam.py:288-300, :336-382 at elevation 0 (getRelativeVVP returns inf there): the point 1e8 px away along the
    horizon's normal, in pixel-centre coordinates (the reference's pixel-index point + 0.5).  float64."""
    dh = PanoCam.getDeltaHeightFromRoll(roll, im_h, im_w)
    d = np.array([im_h * ((0.5 + dh) - (0.5 - dh)), -im_w], np.float64)
    norm = np.sqrt(d @ d)
    if norm >= 10 * np.finfo(np.float64).eps:                # sklearn's normalize leaves (near-)zero rows unscaled
        d = d / norm
    return 1e8 * d[0] + 0.5 * im_w, 1e8 * d[1] + 0.5 * im_h


def pinhole_fields(vfov, heights, widths, elevation, roll, device=None, up=True, lat=True):
    """Batched ``PanoCam.get_up`` / ``get_lat`` (utils/panocam.py:384-448), radians: the ``_general`` fields with focal_rel =
    1 / (2 tan(vfov / 2)) and a centred principal point, except that at elevation == 0 the up field points to the reference's
    far vanishing point (``far_vanishing_point``) rather than being constant."""
    n = len(heights)
    focal = [1.0 / (2.0 * math.tan(float(v) / 2.0)) for v in vfov]
    nan = (math.nan, math.nan)
    vp = [far_vanishing_point(int(widths[i]), int(heights[i]), float(roll[i])) if float(elevation[i]) == 0 else nan for i in range(n)]
    return camera_fields(focal, heights, widths, elevation, roll, [0.0] * n, [0.0] * n, device, up=up, lat=lat, vp=vp)


def fields_from_predictions(preds, sizes, mode="deg", device=None):
    """The parameter -> field step of ``draw_from_r_p_f_cx_cy`` (utils/utils.py:359-385) for a list of ``inference`` results:
    ``roll, pitch, general vfov, rel_cx, rel_cy`` (degrees when mode == "deg") -> focal by ``general_vfov_to_focal(cx, cy, 1,
    vfov, False)`` -> (up fields, latitude maps in degrees) at the given (H, W) sizes."""
    if mode not in ("deg", "rad"):
        raise ValueError("Bad argument")
    val = lambda d, k: float(d[k].item() if hasattr(d[k], "item") else d[k])
    roll = [val(p, "pred_roll") for p in preds]
    pitch = [val(p, "pred_pitch") for p in preds]
    vfov = [val(p, "pred_general_vfov") for p in preds]
    cx = [val(p, "pred_rel_cx") for p in preds]
    cy = [val(p, "pred_rel_cy") for p in preds]
    if mode == "deg":
        roll, pitch, vfov = [math.radians(v) for v in roll], [math.radians(v) for v in pitch], [math.radians(v) for v in vfov]
    focal = general_vfov_to_focal(cx, cy, 1, vfov, False)
    return camera_fields(list(focal), [s[0] for s in sizes], [s[1] for s in sizes], pitch, roll, cx, cy, device)
