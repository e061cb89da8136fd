"""CPU restatement (float32 numpy, in the kernels' order of operations) of the sub-bin decode of the classification heads (DESIGN.md
section 1, "Sub-bin decode"; engine option "subbin", ``PerspectiveFields(decode="subbin")``), and the post-process of
oracle/model.py with only the decode step swapped for it.

For one pixel with logits l of one head: c = the first maximal index; neighbours c-, c+ (up head, NC = 73: the 72 direction
bins as a circle, (c -+ 1) mod (NC - 1), and no refinement in the no-direction bin NC - 1; latitude head: c -+ 1, no refinement in
the two pole bins); a = l(c) - l(c-), b = l(c) - l(c+); delta = (a - b) / (2 (a + b)) when a and b are finite and a + b > 0, else 0;
the field is decode_bin / decode_bin_latitude's formula at p = c + delta.
"""
import numpy as np
import torch
import torch.nn.functional as F

import oracle_resize as ro
from oracle import model as om
from oracle.variants import NET_H, NET_W

F32 = np.float32


def neighbours(c, NC, is_gravity):
    """Classes of the lower and upper neighbour of the argmax c (c itself where the bin is not refined) and the refined mask."""
    c = np.asarray(c, np.int64)
    if is_gravity:
        m = NC - 1   # direction bins 0 .. NC-2 on a circle
        refined = c < NC - 1
        lo = np.where(refined, (c - 1) % max(m, 1), c)
        hi = np.where(refined, (c + 1) % max(m, 1), c)
    else:
        refined = (c > 0) & (c < NC - 1)
        lo, hi = np.maximum(c - 1, 0), np.minimum(c + 1, NC - 1)
    return lo, hi, refined


def delta_of(l0, lm, lp):
    """delta of the parabola vertex through (-1, lm), (0, l0), (1, lp), in float32; 0 for non-finite or flat (a + b <= 0) input."""
    l0, lm, lp = (np.asarray(x, F32) for x in (l0, lm, lp))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        a, b = l0 - lm, l0 - lp
        s = a + b
        ok = np.isfinite(a) & np.isfinite(b) & (s > 0)
        d = (a - b) / (F32(2) * np.where(ok, s, F32(1)))
    return np.where(ok, d, F32(0)).astype(F32)


def position(logits, is_gravity, axis=-1):
    """(c, delta) of every pixel: the argmax and its sub-bin offset (delta = 0 where the bin is not refined), class axis removed."""
    l = np.moveaxis(np.asarray(logits, F32), axis, -1)
    NC = l.shape[-1]
    c = l.argmax(-1)
    lo, hi, refined = neighbours(c, NC, is_gravity)
    take = lambda i: np.take_along_axis(l, i[..., None], -1)[..., 0]
    d = delta_of(take(c), take(lo), take(hi))
    return c, np.where(refined, d, F32(0)).astype(F32)


def decode_gravity(logits, axis=-1):
    """Up vectors of the 73-bin head: [..., 2] for [..., NC] logits, the component on ``axis`` otherwise ([n, 2, H, W])."""
    l = np.asarray(logits)
    NC = l.shape[axis]
    c, d = position(l, True, axis)
    p = c.astype(F32) + d
    w = F32(360) / F32(NC - 1)
    ang = ((p * w - F32(180)) / F32(180)) * F32(np.pi)
    t = torch.from_numpy(np.ascontiguousarray(ang))
    vec = np.stack([torch.cos(t).numpy(), torch.sin(t).numpy()], -1).astype(F32)   # torch's cos / sin, as decode_bin evaluates them
    vec[c == NC - 1] = 0
    return vec if axis in (-1, l.ndim - 1) else np.moveaxis(vec, -1, axis)


def decode_latitude(logits, axis=-1):
    """Latitudes in degrees of the 180-bin head, class axis removed."""
    l = np.asarray(logits)
    NC = l.shape[axis]
    c, d = position(l, False, axis)
    p = c.astype(F32) + d
    w = F32(180) / F32(NC)
    return ((F32(-90) + p * w) + w * F32(0.5)).astype(F32)


def pf_postprocess(result, height, width, net_hw=(NET_H, NET_W)):
    """oracle.model.pf_postprocess at the working size net_hw (oracle_resize's where it is not 320 x 320)."""
    if tuple(net_hw) == (NET_H, NET_W):
        return om.pf_postprocess(result, height, width)
    return ro.pf_postprocess(result, height, width, net_hw)


def postprocess_gravity(result, height, width, net_hw=(NET_H, NET_W)):
    """oracle.model.postprocess_gravity with the sub-bin decode: result [NC, H, W] logits."""
    vec = torch.from_numpy(decode_gravity(np.asarray(result, F32), axis=0))
    scale = torch.tensor([[width / net_hw[1]], [height / net_hw[0]]]).unsqueeze(-1)
    return F.normalize(pf_postprocess(vec * scale, height, width, net_hw), dim=0)


def postprocess_latitude(result, height, width, net_hw=(NET_H, NET_W)):
    """oracle.model.postprocess_latitude with the sub-bin decode: result [NC, H, W] logits."""
    lat = torch.from_numpy(decode_latitude(np.asarray(result, F32), axis=0)).unsqueeze(0)
    return pf_postprocess(lat, height, width, net_hw)[0]
