"""CPU: the ``resize`` option of ``PerspectiveFields`` (working sizes other than DATALOADER.RESIZE = [320, 320]) on the host
side -- validation, the configuration and ``aug`` it produces, the distributed blob sizes -- and the oracle at 384 x 512 and
448 x 448 (tests/oracle_resize.py) against the unmodified reference's outputs (tests/golden/golden_resize.npz, made by
tests/golden/make_golden_resize.py).  A model is built without a GPU: its engine is created on first use."""
import os

import numpy as np
import pytest
import torch

import oracle_resize as ro
import pf_test_util as U
from golden_util import GOLDEN_DIR, golden_images
from oracle import model as om
from oracle import weights_gen as wg
from oracle.variants import VARIANTS
from perspectivefields_b200 import dist
from perspectivefields_b200.perspectivefields import check_resize

VERSION = "Paramnet-360Cities-edina-centered"


@pytest.mark.parametrize("bad", [(320, 330), (330, 320), (32, 320), (320, 32), (672, 320), (320, 672), (640, 448), (512, 576),
                                 (0, 320), (-320, 320), (320.0, 320), (True, 320), 320, (320,), (320, 320, 3), "320x320"])
def test_resize_validation(bad):
    with pytest.raises(ValueError):
        check_resize(bad)


@pytest.mark.parametrize("good,keys", [((64, 64), 4), ((320, 448), 140), ((384, 512), 192), ((512, 512), 256), ((640, 384), 240),
                                      ((64, 640), 40), ((np.int64(448), 448), 196)])
def test_resize_accepted(good, keys):
    h, w = check_resize(good)
    assert (h, w) == tuple(int(x) for x in good) and (h // 32) * (w // 32) == keys


def test_default_is_the_yaml_resize():
    assert check_resize(None) == (320, 320)
    U.write_synthetic_checkpoint(VERSION)
    from perspectivefields_b200 import PerspectiveFields

    a, b = PerspectiveFields(VERSION), PerspectiveFields(VERSION, resize=(320, 320))
    for m in (a, b):
        assert m.cfg.DATALOADER.RESIZE == [320, 320] and m.net_size() == (320, 320)
        assert (m.aug.new_h, m.aug.new_w, m.aug.interp) == (320, 320, 2)


def test_bad_resize_raises_before_any_gpu_work():
    from perspectivefields_b200 import PerspectiveFields

    with pytest.raises(ValueError, match="multiples of 32"):
        PerspectiveFields(VERSION, resize=(300, 400))
    with pytest.raises(ValueError, match="256"):
        PerspectiveFields(VERSION, resize=(640, 448))


@pytest.mark.parametrize("version", sorted(VARIANTS))
def test_cfg_and_aug_follow_resize(version):
    U.write_synthetic_checkpoint(version)
    from perspectivefields_b200 import PerspectiveFields

    m = PerspectiveFields(version, resize=(384, 512), precision="bf16")
    assert m.cfg.DATALOADER.RESIZE == [384, 512] and m.cfg["DATALOADER"]["RESIZE"] == [384, 512]
    assert (m.aug.new_h, m.aug.new_w) == (384, 512)
    assert m.net_size() == (384, 512) and m._engine is None
    m.load_state_dict(m.state_dict())         # the option is a model attribute: it survives a reload
    assert m.net_size() == (384, 512) and m.cfg.DATALOADER.RESIZE == [384, 512]
    # the configuration of a default model is not shared with it
    assert PerspectiveFields(version).cfg.DATALOADER.RESIZE == [320, 320]


def test_dist_blob_sizes_at_a_non_square_size():
    sizes = [(480, 640), (10, 20)]
    n = dist.blob_numels((2, 1), sizes, (320, 448))
    assert n["pred_gravity"] == 2 * 2 * 320 * 448 and n["pred_latitude"] == 2 * 320 * 448
    assert n["gravity_original"] == 2 * (480 * 640 + 200) and n["params"] == 16
    raw = dist.empty_raw((73, 180), sizes, "cpu", (320, 448))
    assert raw["pred_gravity"].shape == (2, 73, 320, 448) and raw["pred_latitude"].shape == (2, 180, 320, 448)
    assert dist.blob_numels((2, 1), sizes) == dist.blob_numels((2, 1), sizes, (320, 320))
    spec = dict(dist._result_spec(VARIANTS[VERSION], 480, 640, (448, 320)))
    assert spec["pred_gravity"] == (2, 448, 320) and spec["pred_latitude_original"] == (480, 640)


# ------------------------------------------------------------------------------------------------ oracle vs reference
_SKIP = {"PersNet-360Cities": ("pred_gravity_original", "pred_latitude_original")}   # argmax-decoded: the logits are compared
_GOLDEN = None


def _golden():
    global _GOLDEN
    if _GOLDEN is None:
        _GOLDEN = dict(np.load(os.path.join(GOLDEN_DIR, "golden_resize.npz")))
    return _GOLDEN


@pytest.mark.parametrize("net_hw", [(384, 512), (448, 448)])
@pytest.mark.parametrize("version", sorted(VARIANTS))
def test_oracle_matches_reference_at_other_sizes(version, net_hw):
    """The oracle at another working size (tests/oracle_resize.py) against the unmodified reference run with that
    DATALOADER.RESIZE (tests/golden/make_golden_resize.py): a seeded sample of 768 elements of every returned tensor at 1e-4
    relative to the tensor's maximum magnitude, and the abs-sum checksum of the whole tensor."""
    g = _golden()
    assert [tuple(x) for x in g["sizes"]] == [(384, 512), (448, 448)]
    tag = "%dx%d" % net_hw
    out = ro.inference_batch(wg.synth_state_dict(version, 0), version, golden_images(), net_hw)
    for i, res in enumerate(out):
        base = f"{tag}/{version}/{i}"
        assert list(res.keys()) == list(g[f"{base}/keys"])
        for k, v in res.items():
            if isinstance(v, str) or k in _SKIP.get(version, ()):
                continue
            key = f"{base}/{k}"
            a = v.detach().double().numpy().reshape(-1)
            absmax, _, sa, *shape = g[key + "/meta"]
            assert tuple(v.shape) == tuple(int(x) for x in shape), k
            idx = ro.sample_index(key, a.size)
            got = a if idx is None else a[idx]
            e = np.abs(got - g[key]).max() / max(float(absmax), 1e-30)
            assert e <= 1e-4, (version, i, k, e)
            assert abs(np.abs(a).sum() - sa) <= 4e-4 * max(sa, 1e-30), (k, "abs-sum checksum")
    assert tuple(out[0]["pred_gravity"].shape[1:]) == net_hw


def test_resize_oracle_at_320_is_the_oracle():
    """tests/oracle_resize.py at (320, 320) computes exactly what oracle/model.py computes."""
    version = "Paramnet-360Cities-edina-uncentered"
    sd = wg.synth_state_dict(version, 0)
    img = wg.smooth_images(1, 150, 200, 3)[0]
    a, b = ro.inference(sd, version, img, (320, 320)), om.inference(sd, version, img)
    assert list(a.keys()) == list(b.keys())
    for k, v in b.items():
        assert (a[k] == v) if isinstance(v, str) else torch.equal(a[k], v), k
