"""Generate tests/golden/equi.npz from the UNMODIFIED reference (build container only; needs torchvision and cv2):

    PF_REFERENCE_ROOT=<reference checkout> python tests/golden/make_golden_equi.py

Runs ``PanoCam.crop_equi``, ``PanoCam(path).get_image``, the horizon / vertical-vanishing-point helpers and ``get_lat`` /
``get_up`` (perspective2d/utils/panocam.py:121-448) themselves.  ``equilib.equi2pers``, which the first two wrap, comes from
equilib 0.3.0, which is neither in the reference tree nor installed: the script sets the oracle's ``equi2pers``
(tests/oracle_equi.py: this project's geometry and sampler) as the module's ``equi2pers`` and records the arguments the wrapper
passes it.  Everything else -- fov_x, the rot dict, the dtype handling, ToTensor / ToPILImage and the cv2 colour conversion, the
helpers and the fields -- is the reference's code.  The panorama is regenerated from a seed (``oracle_pano.make_panorama``)."""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.ref_shim import load_reference  # noqa: E402
import oracle_equi  # noqa: E402
import oracle_pano  # noqa: E402

PANO_SEED, PANO_H, PANO_W = 9, 256, 512
# (vfov, im_w, im_h, azimuth, elevation, roll, ar), degrees
CROP_CASES = [
    (70.0, 64, 48, 30.0, 20.0, 0.0, 64 / 48),
    (60.0, 64, 48, -50.0, -15.0, 10.0, 64 / 48),
    (80.0, 48, 64, 100.0, 35.0, -25.0, 48 / 64),
    (50.0, 64, 48, 10.0, 5.0, 3.0, 4 / 3),
    (90.0, 64, 48, -120.0, -40.0, 30.0, 4 / 3),
    (60.0, 48, 40, 180.0, 0.0, 0.0, 1.5),          # ar != W / H, across the seam, level
    (40.0, 40, 30, 0.0, 85.0, 0.0, 4 / 3),         # looking at the north pole: rows clamp
    (50.0, 40, 30, 45.0, -20.0, 180.0, 4 / 3),     # upside down
]
# (vfov, im_w, im_h, azimuth, elevation, roll, ar) of get_image, RGB and BGR
IMAGE_CASES = [(85.0, 64, 48, 0.0, 30.0, 0.0, 4 / 3), (60.0, 48, 64, -70.0, -10.0, 12.0, 0.75)]
# (vfov, im_w, im_h, elevation, roll), degrees, of the horizon / VVP helpers
HV_CASES = [(85.0, 640, 480, 30.0, 0.0), (60.0, 64, 48, -15.0, 10.0), (70.0, 64, 48, 0.0, 5.0), (70.0, 64, 48, 90.0, 0.0),
            (70.0, 64, 48, -90.0, 20.0), (50.0, 48, 64, 10.0, 90.0), (50.0, 48, 64, -10.0, -90.0), (50.0, 48, 64, 10.0, 180.0),
            (60.0, 40, 30, 0.0, 180.0), (45.0, 33, 17, 90.0, 90.0), (100.0, 320, 240, 45.0, -135.0)]


def rad(x):
    return x / 180 * np.pi       # the expression get_image uses (:188-193)


def main():
    load_reference()
    import perspective2d.utils.panocam as ref
    from PIL import Image

    ref.equi2pers = oracle_equi.equi2pers
    pano = oracle_pano.make_panorama(PANO_SEED, PANO_H, PANO_W)
    gray = np.ascontiguousarray(pano[:, :, 1])
    pano_f32 = (pano.astype(np.float32) * np.float32(1.0 / 64)) - np.float32(1.5)
    out = {"pano": np.array([PANO_SEED, PANO_H, PANO_W], np.int64), "crop_cases": np.array(CROP_CASES, np.float64),
           "image_cases": np.array(IMAGE_CASES, np.float64), "hv_cases": np.array(HV_CASES, np.float64)}
    wrapper = []
    for i, (vfov, w, h, az, el, roll, ar) in enumerate(CROP_CASES):
        w, h = int(w), int(h)
        for key, img, mode in (("u8", pano, "bilinear"), ("gray", gray, "bilinear"), ("f32", pano_f32, "bilinear"), ("near", pano, "nearest")):
            oracle_equi.CALLS.clear()
            out[f"{key}{i}"] = ref.PanoCam.crop_equi(img, vfov, w, h, az, el, roll, ar, mode)
        c = oracle_equi.CALLS[0]
        wrapper.append([c["fov_x"], c["roll"], c["pitch"], c["yaw"]])
        out[f"lat{i}"] = ref.PanoCam.get_lat(rad(vfov), w, h, rad(el), rad(roll))
        out[f"up{i}"] = ref.PanoCam.get_up(rad(vfov), w, h, rad(el), rad(roll))
    out["wrapper"] = np.array(wrapper, np.float64)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "pano.png")
        Image.fromarray(pano).save(path)
        cam = ref.PanoCam(path)
        for k, (vfov, w, h, az, el, roll, ar) in enumerate(IMAGE_CASES):
            for fmt in ("RGB", "BGR"):
                crop, horizon, vvp = cam.get_image(vfov, int(w), int(h), az, el, roll, ar, fmt)
                out[f"image_{fmt}{k}"] = np.array(crop)
                out[f"image_horizon{k}"] = np.array(horizon, np.float64)
                out[f"image_vvp{k}"] = np.array(vvp, np.float64)
    hv = []
    for vfov, w, h, el, roll in HV_CASES:
        args = (rad(el), rad(roll), rad(vfov), int(h), int(w))
        horizon = ref.PanoCam.getRelativeHorizonLineFromAngles(*args)
        vvp = ref.PanoCam.getRelativeVVP(*args)
        mid = ref.PanoCam.getMidpointFromAngle(*args[:3])
        dh = ref.PanoCam.getDeltaHeightFromRoll(rad(roll), int(h), int(w))
        hv.append([*horizon, *vvp, *([np.nan] * (3 - len(vvp))), len(vvp), mid, dh])
    out["hv"] = np.array(hv, np.float64)     # horizon (2), vvp padded with nan (3), len(vvp), midpoint, delta height
    path = os.path.join(HERE, "equi.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
