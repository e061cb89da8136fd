"""Layout of tests/golden/paramnet_grads.npz, shared by its generator (tests/golden/make_golden_paramnet_grads.py) and
tests/test_oracle_paramnet_grads.py: how many entries of each gradient tensor are stored, which ones, and up to which size a
tensor is stored whole."""
import zlib

import numpy as np

SAMPLES = 64
FULL_MAX = 384


def sample_idx(name, numel):
    """The SAMPLES flat indices of tensor ``name`` (e.g. ``param_net.backbone.norm.weight``) whose gradient the fixture stores."""
    return np.random.RandomState(zlib.crc32(name.encode())).randint(0, numel, SAMPLES).astype(np.int64)
