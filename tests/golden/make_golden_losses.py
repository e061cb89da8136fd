"""Generate tests/golden/losses.npz from the UNMODIFIED reference (build container only; needs the reference checkout):

    PF_REFERENCE_ROOT=/path/to/PerspectiveFields python tests/golden/make_golden_losses.py

The inputs are regenerated from the seeds in tests/oracle_metrics.py; only the reference's outputs are stored:
* ``enc_special``: ``encode_bin`` of the special vectors (axes, bin centres, zero vectors, exact rounding ties), num_bin 73;
* ``enc_lat_special``: ``encode_bin_latitude`` of every class boundary, its float32 neighbours and the ends, num_classes 180;
* ``msgil``: ``msgil_norm_loss`` of a small case with a random mask;
* per case of ``LOSS_CASES``: checksums of the reference's labels (classification) and the values of
  ``GravityDecoder.losses`` / ``LatitudeDecoder.losses`` called unbound on an object carrying loss_type, loss_weight and
  ignore_value, with the targets of the rule (oracle_metrics.targets).
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_metrics as om  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def special_latitudes():
    b = om.latitude_boundaries(om.NUM_LAT)
    vals = [b, np.nextafter(b, np.float32(-np.inf)), np.nextafter(b, np.float32(np.inf)),
            np.array([-90.0, 90.0, -89.99, 89.99, 0.0, -0.0, -100.0, 100.0], np.float32)]
    return np.concatenate(vals).astype(np.float32)


def main():
    load_reference()
    from perspective2d.modeling.persformer_heads.gravity_head import GravityDecoder
    from perspective2d.modeling.persformer_heads.latitude_head import LatitudeDecoder
    from perspective2d.modeling.persformer_heads.loss_fns import msgil_norm_loss
    from perspective2d.utils.utils import encode_bin, encode_bin_latitude

    out = {}
    v, ties = om.special_vectors()
    print(f"{ties} exact rounding ties among {v.shape[-1]} special vectors")
    out["enc_special"] = encode_bin(v, om.NUM_BIN).numpy().astype(np.int16)
    out["enc_lat_special"] = encode_bin_latitude(torch.from_numpy(special_latitudes()), om.NUM_LAT).numpy().astype(np.int16)

    g = torch.Generator().manual_seed(3)
    p, t = torch.randn((2, 2, 37, 53), generator=g), torch.randn((2, 2, 37, 53), generator=g)
    mask = torch.rand((2, 2, 37, 53), generator=g) < 0.7
    out["msgil"] = np.float64(msgil_norm_loss(p, t, mask).item())

    for name, loss_type, n, h, w, seed in om.LOSS_CASES:
        pg, pl, up, lat = om.loss_inputs(loss_type, n, h, w, seed)
        if loss_type == "regression":
            gg, gl = om.targets(up, lat, loss_type)
        else:
            gg = torch.stack([encode_bin(u.permute(2, 0, 1), om.NUM_BIN) for u in up])
            gl = torch.stack([encode_bin_latitude(d, om.NUM_LAT) for d in lat])
            out[name + "/gt_gravity_checksum"] = np.int64(om.label_checksum(gg))
            out[name + "/gt_latitude_checksum"] = np.int64(om.label_checksum(gl))
        head = types.SimpleNamespace(loss_type=loss_type, loss_weight=1.0, ignore_value=om.IGNORE_GRAVITY)
        vals = GravityDecoder.losses(head, pg, gg)
        head = types.SimpleNamespace(loss_type=loss_type, loss_weight=1.0, ignore_value=om.IGNORE_LATITUDE)
        vals.update(LatitudeDecoder.losses(head, pl, gl))
        for k, val in vals.items():
            out[f"{name}/{k}"] = np.float32(val.item())
        print(name, {k: float(val) for k, val in vals.items()})
    path = os.path.join(HERE, "losses.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
