"""CPU restatement (float32 numpy, in the kernels' order of operations) of flip test-time augmentation (DESIGN.md section 1, "Flip
test-time augmentation"; engine option "flip_tta", ``PerspectiveFields(tta="flip")``), and the oracle forward with it.

For each image x the network runs on x and on its mirror x[:, ::-1] (taken before the pre-process); with a the image's head output,
b the mirror's and M(b) = b[..., ::-1] (column W-1-x read at x), the merged outputs at the working size are
  regression up        normalize(a + M(b) * (-1, 1)), normalize(v) = v / max(|v|, 1e-12)
  regression latitude  (a + M(b)) * 0.5
  classification       (a + P(M(b))) * 0.5, P: up class c -> (36 - c) mod 72 (c < 72), 72 and every latitude class fixed,
each a sum, then a scale, rounded one at a time.  Decode, confidence, post-process and ParamNet then run on the merged outputs.
"""
import numpy as np
import torch

import oracle_confidence as ocf
import oracle_resize as ro
import oracle_subbin as osb
from oracle import model as om
from oracle.variants import NET_H, NET_W, PIXEL_MEAN, PIXEL_STD, VARIANTS

F32 = np.float32


def class_map(NC, is_gravity):
    """P as an index array: merged class c reads the mirror's class P[c]."""
    c = np.arange(NC)
    if not is_gravity:
        return c
    m = NC - 1
    return np.where(c < m, (m + m // 2 - c) % m, c)


def mirror(x):
    """M: the last (column) axis reversed."""
    return np.ascontiguousarray(np.asarray(x)[..., ::-1])


def merge_up(a, b):
    """a, b [..., 2, H, W] unit up vectors -> normalize(a + M(b) * (-1, 1))."""
    a, b = np.asarray(a, F32), mirror(np.asarray(b, F32))
    vx, vy = a[..., 0, :, :] - b[..., 0, :, :], a[..., 1, :, :] + b[..., 1, :, :]
    nrm = np.maximum(np.sqrt(vx * vx + vy * vy), F32(1e-12))
    return np.stack([vx / nrm, vy / nrm], -3).astype(F32)


def merge_lat(a, b):
    """a, b [..., H, W] sin-latitudes -> (a + M(b)) * 0.5."""
    return ((np.asarray(a, F32) + mirror(np.asarray(b, F32))) * F32(0.5)).astype(F32)


def merge_logits(a, b, is_gravity):
    """a, b [..., NC, H, W] logits -> (a + P(M(b))) * 0.5."""
    a, b = np.asarray(a, F32), mirror(np.asarray(b, F32))
    p = class_map(a.shape[-3], is_gravity)
    return ((a + np.take(b, p, axis=-3)) * F32(0.5)).astype(F32)


def merge_heads(cfg, g, l):
    """Head outputs of the 2n slots (slot n + i: image i's mirror) -> the n merged ones (numpy float32)."""
    g, l = np.asarray(g, F32), np.asarray(l, F32)
    n = g.shape[0] // 2
    if cfg["gravity"] == "regression":
        return merge_up(g[:n], g[n:]), merge_lat(l[:n, 0], l[n:, 0])[:, None]
    return merge_logits(g[:n], g[n:], True), merge_logits(l[:n], l[n:], False)


@torch.no_grad()
def forward(sd, version, batched_inputs, net_hw=(NET_H, NET_W), decode="argmax", confidence=False, logits=True, mirrored=None):
    """oracle forward (oracle_resize.forward) with flip TTA.  ``batched_inputs``: list of {"image" [3, H, W] at the working size,
    "height", "width"}; ``mirrored``: the images the mirror slots run on ([3, H, W] each; default: each image flipped, the
    engine's float path).  The result dicts have the engine's keys: the merged logits (logits=True) or the decoded fields at
    the working size, the post-processed fields, the confidences when asked for, and ParamNet's outputs."""
    cfg = VARIANTS[version]
    mean = torch.tensor(PIXEL_MEAN).view(-1, 1, 1)
    std = torch.tensor(PIXEL_STD).view(-1, 1, 1)
    if mirrored is None:
        mirrored = [x["image"].flip(-1) for x in batched_inputs]
    images = torch.stack([(x["image"] - mean) / std for x in batched_inputs] + [(m - mean) / std for m in mirrored])
    assert tuple(images.shape[2:]) == tuple(net_hw)
    g2, l2 = om.heads_inference(sd, cfg, om.mit_b3(sd, images), om.low_level_encoder(sd, images))
    g, l = (torch.from_numpy(t) for t in merge_heads(cfg, g2.numpy(), l2.numpy()))
    results = []
    for i, inp in enumerate(batched_inputs):
        h, w = inp["height"], inp["width"]
        r = {}
        if cfg["gravity"] == "regression":
            r["pred_gravity"] = g[i]
            r["pred_gravity_original"] = ro.postprocess_gravity(cfg, g[i], h, w, net_hw)
            r["pred_latitude"] = l[i]
            r["pred_latitude_original"] = ro.postprocess_latitude(cfg, l[i], h, w, net_hw)
        else:
            if decode == "subbin":
                up, lat = osb.decode_gravity(g[i].numpy(), axis=0), osb.decode_latitude(l[i].numpy(), axis=0)
                go = osb.postprocess_gravity(g[i].numpy(), h, w, net_hw)
                lo = osb.postprocess_latitude(l[i].numpy(), h, w, net_hw)
            else:
                up = om.decode_bin(g[i].argmax(0), cfg["gravity_classes"]).numpy()
                lat = om.decode_bin_latitude(l[i].argmax(0), cfg["latitude_classes"]).numpy()
                go = ro.postprocess_gravity(cfg, g[i], h, w, net_hw)
                lo = ro.postprocess_latitude(cfg, l[i], h, w, net_hw)
            r["pred_gravity"] = g[i] if logits else torch.from_numpy(np.asarray(up, F32))
            r["pred_gravity_original"] = go
            r["pred_latitude"] = l[i] if logits else torch.from_numpy(np.asarray(lat, F32))[None]
            r["pred_latitude_original"] = lo
        r["pred_latitude_original_mode"] = "deg"
        if confidence:
            r["pred_gravity_confidence"] = torch.from_numpy(ocf.confidence(g[i].numpy()).astype(F32))
            r["pred_latitude_confidence"] = torch.from_numpy(ocf.confidence(l[i].numpy()).astype(F32))
        results.append(r)
    if cfg["param_net"] is not None:
        param = om.param_net(sd, cfg, g, l)
        for i in range(len(results)):
            results[i].update({k: v[i] for k, v in param.items()})
    return results


def inference_batch(sd, version, img_bgr_list, net_hw=(NET_H, NET_W), **kw):
    """uint8 BGR images of any size: the mirror slot runs on the Pillow resize of x[:, ::-1] (Pillow's resize does not commute
    with a flip bit for bit, so this is not the flipped resized image)."""
    inputs = [{"image": ro.preprocess(im, net_hw), "height": im.shape[0], "width": im.shape[1]} for im in img_bgr_list]
    mirrored = [ro.preprocess(np.ascontiguousarray(im[:, ::-1]), net_hw) for im in img_bgr_list]
    return forward(sd, version, inputs, net_hw, mirrored=mirrored, **kw)
