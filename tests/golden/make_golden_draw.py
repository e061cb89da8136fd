"""Generate the two fixtures of the drawing tests (build container only; needs the reference checkout and cv2):

    PF_REFERENCE_ROOT=/path/to/PerspectiveFields python tests/golden/make_golden_draw.py

* draw_vancouver.npz: two windows of the reference's own ``draw_perspective_fields`` output ``assets/vancouver/pred_pers.png``
  (640 x 528, 10 x 11 arrows) and of ``assets/vancouver/IMG_2481.jpg`` resized as the demo does (``cv2.resize`` to 640 x 528,
  RGB).  Window a (rows 280:400, columns 150:320) holds the horizon line (level 9) with band 9 above it and band 8 below and two
  arrow shafts (x = 192, 256); window b (rows 350:390, columns 560:600) the shaft at x = 576 where it crosses the horizon line.
* pinhole.npz: ``PanoCam.get_up`` / ``get_lat`` (utils/panocam.py:384-448) of the UNMODIFIED reference for the cases below.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_shim import REFERENCE_ROOT, load_reference  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
WINDOWS = {"a": (280, 400, 150, 320), "b": (350, 390, 560, 600)}
# (vfov, im_w, im_h, elevation, roll), radians
CASES = [
    (0.90, 32, 24, 0.30, -0.20),
    (1.10, 40, 30, -0.45, 0.60),
    (0.80, 24, 36, 0.00, 0.35),        # elevation == 0: the far vanishing point
    (1.30, 17, 11, -0.0, -1.30),       # -0.0 == 0 too
    (0.70, 33, 33, -0.05, 0.00),
    (1.00, 48, 20, 0.75, 3.00),
    (0.60, 21, 29, 0.00, 2.50),        # elevation 0 with cos(roll) < 0
    (1.50, 3, 2, 0.20, 0.10),          # 2 x 3
    (1.20, 64, 48, -0.15, 0.05),
]


def main():
    import cv2
    from PIL import Image

    assets = os.path.join(REFERENCE_ROOT, "assets", "vancouver")
    pred = np.array(Image.open(os.path.join(assets, "pred_pers.png")).convert("RGB"))
    img = cv2.cvtColor(cv2.imread(os.path.join(assets, "IMG_2481.jpg")), cv2.COLOR_BGR2RGB)
    img = cv2.resize(img, (pred.shape[1], pred.shape[0]))
    out = {"canvas_hw": np.array(pred.shape[:2])}
    for k, (r0, r1, c0, c1) in WINDOWS.items():
        out[f"window_{k}"] = np.array((r0, r1, c0, c1))
        out[f"pred_{k}"], out[f"img_{k}"] = pred[r0:r1, c0:c1], img[r0:r1, c0:c1]
    path = os.path.join(HERE, "draw_vancouver.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")

    load_reference()
    from perspective2d.utils.panocam import PanoCam
    out = {"cases": np.array(CASES, np.float64)}
    for i, (vfov, w, h, el, roll) in enumerate(CASES):
        out[f"up{i}"] = PanoCam.get_up(vfov=vfov, im_w=int(w), im_h=int(h), elevation=el, roll=roll)
        out[f"lat{i}"] = PanoCam.get_lat(vfov=vfov, im_w=int(w), im_h=int(h), elevation=el, roll=roll)
    path = os.path.join(HERE, "pinhole.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
