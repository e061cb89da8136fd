"""Generate tests/golden/paramnet_grads.npz from the UNMODIFIED reference (build container only; needs the reference checkout):

    PF_REFERENCE_ROOT=/path/to/PerspectiveFields python tests/golden/make_golden_paramnet_grads.py

For each configuration of tests/oracle_paramnet.CONFIGS the reference's ``build_param_net(cfg)`` is loaded with the seeded
``param_net.*`` weights (as in make_golden_paramnet.py) and run in its training branch on the seeded fields and targets of
tests/oracle_paramnet.py: ``pn.train(); sum(pn(preds, batched_inputs).values()).backward()``.  The full gradients are about
112 MB per configuration, so only summaries are stored, as a few arrays per configuration (one array per tensor would cost
more in zip headers than in data), values in float32 (the reference computes in float32).  For the T gradient tensors of a
configuration -- every parameter in ``named_parameters()`` order, then ``input/pred_gravity`` and ``input/pred_latitude``:
* ``<config>/names`` [T] and ``<config>/numel`` [T];
* ``<config>/norm`` and ``<config>/sum`` [T]: each tensor's L2 norm and sum (taken in float64);
* ``<config>/val`` [T, 64]: each tensor at 64 flat indices drawn by ``paramnet_grads_fixture.sample_idx`` (seeded by the name, so not stored);
* ``<config>/full``: the tensors with at most 384 elements (the stem and the first two stages' LayerNorms, biases and gamma,
  the head bias), concatenated in order.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_paramnet as op  # noqa: E402
import paramnet_grads_fixture as fx  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402
from oracle.variants import VARIANTS  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

def summarize(config, tensors):
    """{name: gradient} in order -> the arrays stored for ``config``."""
    names, numel, norm, tot, val, full = [], [], [], [], [], []
    for k, g in tensors.items():
        g = g.detach().double().reshape(-1)
        names.append(k)
        numel.append(g.numel())
        norm.append(g.norm().item())
        tot.append(g.sum().item())
        val.append(g[torch.from_numpy(fx.sample_idx(k, g.numel()))].numpy())
        if g.numel() <= fx.FULL_MAX:
            full.append(g.numpy())
    return {f"{config}/names": np.array(names), f"{config}/numel": np.array(numel, np.int64), f"{config}/norm": np.array(norm),
            f"{config}/sum": np.array(tot), f"{config}/val": np.stack(val).astype(np.float32),
            f"{config}/full": np.concatenate(full).astype(np.float32)}


def main():
    mod = load_reference()
    from perspective2d.config.config import get_perspective2d_cfg_defaults
    from perspective2d.modeling.param_network import build_param_net
    from perspective2d.utils.panocam import PanoCam

    grav, lat = op.inputs(PanoCam.get_up_general, PanoCam.get_lat_general)
    batched_inputs = op.targets(grav.shape[0])
    out = {}
    for name, version, seed in op.CONFIGS:
        cfg = get_perspective2d_cfg_defaults()
        cfg.merge_from_file(os.path.join(os.path.dirname(mod.__file__), "config", VARIANTS[version]["ckpt"].replace(".pth", ".yaml")))
        pn = build_param_net(cfg)
        sd = {k[len("param_net."):]: v for k, v in op.param_state(version, seed).items()}
        pn.load_state_dict(sd, strict=True)
        pn.train()
        g = grav.clone().requires_grad_(True)
        la = lat.clone().requires_grad_(True)
        losses = pn({"pred_gravity": g, "pred_latitude": la}, batched_inputs)
        sum(losses.values()).backward()
        tensors = {f"param_net.{k}": p.grad for k, p in pn.named_parameters()}
        tensors["input/pred_gravity"] = g.grad
        tensors["input/pred_latitude"] = la.grad
        out.update(summarize(name, tensors))
        print(name, {k: float(v) for k, v in losses.items()})
    path = os.path.join(HERE, "paramnet_grads.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
