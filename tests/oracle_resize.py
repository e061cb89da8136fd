"""The oracle (oracle/model.py) at a working size other than DATALOADER.RESIZE = [320, 320].  TEST INFRASTRUCTURE.

The network itself is shape-generic in the reference and in oracle/model.py (MiT has no position embedding, the heads upsample
by fixed factors, ConvNeXt runs on whatever map it gets), so the network functions of oracle/model.py are reused as they are.
The working size enters in exactly the places the reference reads ``cfg.DATALOADER.RESIZE``:

* the Pillow resize of the pre-process, ``ResizeTransform(RESIZE[0], RESIZE[1])`` (perspectivefields.py:155) -- ``preprocess``;
* the heads' ``image_size`` (gravity_head.py:136, latitude_head.py:135): the crop to it and the
  ``[[W / image_size[1]], [H / image_size[0]]]`` scale of the post-process (gravity_head.py:248-256, latitude_head.py:201-209,
  utils/utils.py:503) -- ``pf_postprocess`` / ``postprocess_gravity`` / ``postprocess_latitude``.

At ``net_hw = (320, 320)`` every function here computes exactly what its oracle/model.py namesake computes
(tests/test_resize_host.py checks it).  ``sample_index`` is the element sample of tests/golden/golden_resize.npz.
"""
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import model as om
from oracle.pillow_resize import resize_bilinear_u8
from oracle.variants import PIXEL_MEAN, PIXEL_STD, VARIANTS

SAMPLE = 768      # elements kept of a larger golden array (tests/golden/make_golden_resize.py)


def sample_index(key, size):
    """Sorted seeded sample of SAMPLE flat indices of an array of `size` elements, a function of the golden key only (the
    generator and the test draw the same one, so the indices need not be stored); None when the array is kept whole."""
    if size <= SAMPLE:
        return None
    return np.sort(np.random.default_rng(zlib.crc32(key.encode())).choice(size, SAMPLE, replace=False))


def pf_postprocess(result, out_h, out_w, net_hw):
    """utils/utils.py:483-507: crop to the network size (image_size = DATALOADER.RESIZE), bilinear (no antialias) to (H, W)."""
    result = result[:, :net_hw[0], :net_hw[1]].expand(1, -1, -1, -1)
    return F.interpolate(result, size=(out_h, out_w), mode="bilinear", align_corners=False)[0]


def postprocess_gravity(cfg, result, height, width, net_hw):
    """gravity_head.py:237-261."""
    vec = result if cfg["gravity"] == "regression" else om.decode_bin(result.argmax(dim=0), cfg["gravity_classes"])
    scale = torch.tensor([[width / net_hw[1]], [height / net_hw[0]]]).unsqueeze(-1)
    vec = pf_postprocess(vec * scale, height, width, net_hw)
    return F.normalize(vec, dim=0)


def postprocess_latitude(cfg, result, height, width, net_hw):
    """latitude_head.py:195-219."""
    if cfg["latitude"] == "regression":
        lat = pf_postprocess(result, height, width, net_hw)[0]
        return torch.rad2deg(torch.asin(lat))
    lat = om.decode_bin_latitude(result.argmax(dim=0), cfg["latitude_classes"]).unsqueeze(0)
    return pf_postprocess(lat, height, width, net_hw)[0]


def preprocess(img_bgr, net_hw):
    """perspectivefields.py:196-202 with ResizeTransform(H, W): copy, (BGR kept), Pillow resize, float32 CHW."""
    assert img_bgr.dtype == np.uint8 and img_bgr.ndim == 3 and img_bgr.shape[2] == 3
    image = resize_bilinear_u8(img_bgr, net_hw[0], net_hw[1])
    return torch.as_tensor(image.astype("float32").transpose(2, 0, 1))


@torch.no_grad()
def forward(sd, version, batched_inputs, net_hw, taps=None):
    """perspectivefields.py:223-272 on CPU fp32 (oracle/model.py:forward) with images [3, H, W] at the working size."""
    cfg = VARIANTS[version]
    mean = torch.tensor(PIXEL_MEAN).view(-1, 1, 1)
    std = torch.tensor(PIXEL_STD).view(-1, 1, 1)
    images = torch.stack([(x["image"] - mean) / std for x in batched_inputs])
    assert tuple(images.shape[2:]) == tuple(net_hw)
    hl = om.mit_b3(sd, images, taps)
    ll = om.low_level_encoder(sd, images)
    if taps is not None:
        taps["ll"] = ll
    g, l = om.heads_inference(sd, cfg, hl, ll, taps)
    results = []
    for i, inp in enumerate(batched_inputs):
        h, w = inp["height"], inp["width"]
        results.append({
            "pred_gravity": g[i],
            "pred_gravity_original": postprocess_gravity(cfg, g[i], h, w, net_hw),
            "pred_latitude": l[i],
            "pred_latitude_original": postprocess_latitude(cfg, l[i], h, w, net_hw),
            "pred_latitude_original_mode": "deg",
        })
    if cfg["param_net"] is not None:
        param = om.param_net(sd, cfg, g, l, taps)
        for i in range(len(results)):
            results[i].update({k: v[i] for k, v in param.items()})
    return results


def inference_batch(sd, version, img_bgr_list, net_hw, taps=None):
    """perspectivefields.py:207-221."""
    inputs = [{"image": preprocess(im, net_hw), "height": im.shape[0], "width": im.shape[1]} for im in img_bgr_list]
    return forward(sd, version, inputs, net_hw, taps)


def inference(sd, version, img_bgr, net_hw):
    """perspectivefields.py:194-205."""
    return inference_batch(sd, version, [img_bgr], net_hw)[0]
