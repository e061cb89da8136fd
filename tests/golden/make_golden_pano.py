"""Generate tests/golden/pano.npz from the UNMODIFIED reference (build container only):

    PF_REFERENCE_ROOT=<reference checkout> python tests/golden/make_golden_pano.py

Runs ``PanoCam.crop_distortion`` (perspective2d/utils/panocam.py:559-752) itself.  Its sampler,
``equilib.grid_sample.numpy_grid_sample.default``, comes from equilib 0.3.0, which is neither in the reference tree nor installed;
the script sets the oracle's sampler (tests/oracle_pano.py: ``grid_sample_default``, parity unpinned) as the module's
``grid_sample`` before the calls.  Everything else -- projection, rotations, the catadioptric mask, the horizon offset and its
assertions, the reverse projection and sklearn's ``normalize`` -- is the reference's code.  The panorama is regenerated from a
seed (``oracle_pano.make_panorama``) and not stored."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.ref_shim import load_reference  # noqa: E402
import oracle_pano  # noqa: E402

PANO_SEED, PANO_H, PANO_W = 7, 384, 768
# (f, xi, H, W, az, el, roll), degrees; every view is at most 48 x 72
CASES = [
    (40.0, 0.0, 40, 56, 30.0, 10.0, 5.0),        # 0 pinhole
    (30.0, 0.5, 32, 48, -60.0, -15.0, -8.0),     # 1 xi = 0.5
    (12.0, 0.9, 48, 64, 120.0, 5.0, 12.0),       # 2 xi = 0.9, wide
    (20.0, 1.2, 48, 72, 0.0, 20.0, 0.0),         # 3 xi = 1.2 with f < fmin: catadioptric disk mask
    (14.0, 1.3, 31, 45, 45.0, -10.0, 3.0),       # 4 odd H / W: disk centre (round-half-even(H/2), round-half-even(W/2))
    (24.0, 0.0, 33, 47, -20.0, 25.0, -15.0),     # 5 odd H / W, no mask
    (30.0, 0.0, 32, 48, 180.0, 3.0, 2.0),        # 6 view straddling the panorama seam (x near 0 and Wp - 1)
    (20.0, 0.3, 32, 48, 10.0, 88.0, 0.0),        # 7 el near +90: rows near 0
    (20.0, 0.0, 32, 48, -40.0, -89.0, 7.0),      # 8 el near -90: rows near Hp - 1
    (30.0, 0.0, 32, 48, 0.0, 0.0, 0.0),          # 9 level camera, even H: exact-zero horizon row (two crossings: WARNING)
    (30.0, 0.0, 24, 32, 0.0, 0.0, 180.0),        # 10 upside down: the reference raises AssertionError
]
KEYS = ("im", "ntheta", "nphi", "offset", "up", "lat", "xy_map")


def main():
    load_reference()
    import perspective2d.utils.panocam as ref

    ref.grid_sample = types.SimpleNamespace(numpy_grid_sample=types.SimpleNamespace(default=oracle_pano.grid_sample_default))
    pano = oracle_pano.make_panorama(PANO_SEED, PANO_H, PANO_W)
    out = {"cases": np.array(CASES, np.float64), "pano": np.array([PANO_SEED, PANO_H, PANO_W], np.int64)}
    raises = []
    for i, (f, xi, h, w, az, el, roll) in enumerate(CASES):
        try:
            res = ref.PanoCam.crop_distortion(pano, f, xi, int(h), int(w), az, el, roll)
        except AssertionError:
            raises.append(1)
            continue
        raises.append(0)
        for k, v in zip(KEYS, res):
            out[f"{k}{i}"] = np.asarray(v)
    out["raises"] = np.array(raises, np.int64)
    path = os.path.join(HERE, "pano.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
