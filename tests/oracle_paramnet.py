"""Seeded inputs of the ParamNet parity tests (tests/test_oracle_paramnet.py, tests/golden/make_golden_paramnet.py).

The golden file stores the reference's outputs only; both sides rebuild the inputs from the seeds here:
* ``cameras``: pinhole cameras (roll, pitch in degrees, vfov in degrees) whose fields at 320 x 320 are ``get_up_general`` /
  ``get_lat_general`` (the reference's PanoCam in the generator, oracle/panocam.py's restatement in the test), latitude as
  sin(latitude) as the regression head returns it;
* ``random_fields``: unnormalised Gaussian up fields and uniform sin(latitude) maps, which no camera produces;
* ``targets``: the ``batched_inputs`` of the training branch (every key either ParamNet class reads), host floats.
"""
import math

import numpy as np
import torch

SIZE = 320
N_CAMERAS = 6
N_RANDOM = 2
# (name, model version, weight seed): the three ParamNet configurations with ParamNet weights
CONFIGS = (("centered", "Paramnet-360Cities-edina-centered", 0),
           ("uncentered_360", "Paramnet-360Cities-edina-uncentered", 1),
           ("uncentered_gsv", "PersNet_Paramnet-GSV-uncentered", 2))


def cameras(seed=11):
    rs = np.random.RandomState(seed)
    return [(float(rs.uniform(-30, 30)), float(rs.uniform(-40, 40)), float(rs.uniform(40, 90))) for _ in range(N_CAMERAS)]


def camera_fields(get_up_general, get_lat_general):
    """(gravity float32 [N_CAMERAS, 2, SIZE, SIZE], sin(latitude) float32 [N_CAMERAS, 1, SIZE, SIZE]) of ``cameras()`` with the
    given ``PanoCam.get_up_general`` / ``get_lat_general``."""
    ups, lats = [], []
    for roll, pitch, vfov in cameras():
        f = 1.0 / (2.0 * math.tan(math.radians(vfov) / 2.0))
        args = (f, SIZE, SIZE, math.radians(pitch), math.radians(roll), 0.0, 0.0)
        ups.append(np.asarray(get_up_general(*args), np.float64).transpose(2, 0, 1))
        lats.append(np.sin(np.radians(np.asarray(get_lat_general(*args), np.float64)))[None])
    return torch.from_numpy(np.stack(ups).astype(np.float32)), torch.from_numpy(np.stack(lats).astype(np.float32))


def random_fields(seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((N_RANDOM, 2, SIZE, SIZE), generator=g), torch.rand((N_RANDOM, 1, SIZE, SIZE), generator=g) * 2 - 1


def inputs(get_up_general, get_lat_general):
    cg, cl = camera_fields(get_up_general, get_lat_general)
    rg, rl = random_fields()
    return torch.cat([cg, rg]).contiguous(), torch.cat([cl, rl]).contiguous()


def targets(n, seed=23):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        roll, pitch, vfov = rs.uniform(-30, 30), rs.uniform(-40, 40), rs.uniform(40, 90)
        out.append({"roll": float(roll), "pitch": float(pitch), "vfov": float(vfov), "general_vfov": float(vfov + rs.uniform(-5, 5)),
                    "rel_cx": float(rs.uniform(-0.1, 0.1)), "rel_cy": float(rs.uniform(-0.1, 0.1))})
    return out


def param_state(version, seed):
    """The ``param_net.*`` entries of oracle/weights_gen.py's seeded checkpoint of ``version``."""
    from oracle import weights_gen as wg
    from oracle.schema import state_dict_schema

    return {k: wg.synth_tensor(k, s, seed) for k, s in state_dict_schema(version) if k.startswith("param_net.")}
