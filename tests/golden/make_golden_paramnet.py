"""Generate tests/golden/paramnet.npz from the UNMODIFIED reference (build container only; needs the reference checkout):

    PF_REFERENCE_ROOT=/path/to/PerspectiveFields python tests/golden/make_golden_paramnet.py

For each configuration of tests/oracle_paramnet.CONFIGS the reference's ``build_param_net(cfg)`` (cfg: the defaults merged
with the variant's yaml, as perspectivefields.py:124-131 builds it) is loaded with the seeded ``param_net.*`` weights of
oracle/weights_gen.py and run on the seeded inputs of tests/oracle_paramnet.py, the camera fields coming from the reference's
own ``PanoCam.get_up_general`` / ``get_lat_general``.  Only outputs are stored, under ``<config>/``:
* ``raw``: the ConvNeXt backbone's output x [n, 5];
* ``eval/<key>``: the eval branch's dict ``pn(preds)``;
* ``loss/<key>``: the training branch's dict ``pn.train(); pn(preds, batched_inputs)`` for ``oracle_paramnet.targets(n)``.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_paramnet as op  # noqa: E402
from oracle import panocam as oracle_panocam  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402
from oracle.variants import VARIANTS  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    mod = load_reference()
    from perspective2d.config.config import get_perspective2d_cfg_defaults
    from perspective2d.modeling.param_network import build_param_net
    from perspective2d.utils.panocam import PanoCam

    grav, lat = op.inputs(PanoCam.get_up_general, PanoCam.get_lat_general)
    og, ol = op.inputs(oracle_panocam.get_up_general, oracle_panocam.get_lat_general)
    print("oracle fields vs the reference's: max |diff| gravity %.3g, sin(latitude) %.3g" % ((og - grav).abs().max(), (ol - lat).abs().max()))
    preds = {"pred_gravity": grav, "pred_latitude": lat}
    batched_inputs = op.targets(grav.shape[0])
    out = {}
    for name, version, seed in op.CONFIGS:
        cfg = get_perspective2d_cfg_defaults()
        cfg.merge_from_file(os.path.join(os.path.dirname(mod.__file__), "config", VARIANTS[version]["ckpt"].replace(".pth", ".yaml")))
        pn = build_param_net(cfg)
        sd = {k[len("param_net."):]: v for k, v in op.param_state(version, seed).items()}
        pn.load_state_dict(sd, strict=True)
        pn.eval()
        raw = []
        pn.backbone.register_forward_hook(lambda m, i, o: raw.append(o.detach().clone()))
        with torch.no_grad():
            ev = pn(preds)
            out[f"{name}/raw"] = raw[0].numpy()
            for k, v in ev.items():
                out[f"{name}/eval/{k}"] = np.asarray(v.numpy() if isinstance(v, torch.Tensor) else v, np.float32)
            pn.train()
            for k, v in pn(preds, batched_inputs).items():
                out[f"{name}/loss/{k}"] = np.float32(v.item())
        print(name, cfg.MODEL.PARAM_DECODER.NAME, "LOSS_WEIGHT", cfg.MODEL.PARAM_DECODER.LOSS_WEIGHT,
              {k[len(name) + 6:]: float(v) for k, v in out.items() if k.startswith(name + "/loss/")})
    path = os.path.join(HERE, "paramnet.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
