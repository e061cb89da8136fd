"""CPU restatement of the scoring rules (perspectivefields_b200.metrics, PerspectiveFields.targets_from_fields / .losses,
DESIGN.md section 1), and the seeded inputs of the loss fixtures (tests/golden/losses.npz).

The encoders are restated in float32 torch in the reference's order of operations (utils/utils.py:94-146); the losses, the
targets' sine and the field errors are computed in float64."""
import math

import numpy as np
import torch

# (name, loss type, batch, H, W, seed) of the loss fixtures
LOSS_CASES = [
    ("reg_b1_320", "regression", 1, 320, 320, 11),
    ("reg_b3_320", "regression", 3, 320, 320, 12),
    ("reg_b1_384x512", "regression", 1, 384, 512, 13),
    ("reg_b3_384x512", "regression", 3, 384, 512, 14),
    ("cls_b1_320", "classification", 1, 320, 320, 21),
    ("cls_b3_320", "classification", 3, 320, 320, 22),
    ("cls_b1_384x512", "classification", 1, 384, 512, 23),
]
NUM_BIN, NUM_LAT = 73, 180
IGNORE_GRAVITY, IGNORE_LATITUDE = 72, -1      # config/defaults.yaml: GRAVITY_DECODER / LATITUDE_DECODER.IGNORE_VALUE


def label_checksum(labels):
    """Order-sensitive int64 checksum of a label tensor (the fixtures store it instead of the labels)."""
    a = np.asarray(labels, np.int64).reshape(-1)
    return int(np.sum(a * (np.arange(a.size, dtype=np.int64) % 1009 + 1)))


def random_up(g, n, h, w, invalid=True):
    """[n, h, w, 2] float32 unit vectors at random angles; with ``invalid`` a rectangle and a sprinkle of pixels per image are
    (0, 0), the reference's invalid ground truth."""
    ang = torch.rand((n, h, w), generator=g, dtype=torch.float64) * (2 * math.pi) - math.pi
    up = torch.stack([torch.cos(ang), torch.sin(ang)], -1).float()
    if invalid:
        for b in range(n):
            y0, x0 = int(torch.randint(0, h // 2, (1,), generator=g)), int(torch.randint(0, w // 2, (1,), generator=g))
            up[b, y0:y0 + h // 4, x0:x0 + w // 5] = 0
        up[torch.rand((n, h, w), generator=g) < 0.02] = 0
    return up


def random_lat_deg(g, n, h, w):
    """[n, h, w] float32 latitudes in degrees, a few of them exactly on class boundaries (integers)."""
    lat = (torch.rand((n, h, w), generator=g, dtype=torch.float64) * 179.8 - 89.9).float()
    on = torch.rand((n, h, w), generator=g) < 0.05
    lat[on] = torch.round(lat[on])
    return lat


def loss_inputs(loss_type, n, h, w, seed):
    """(pred_gravity, pred_latitude, up [n,h,w,2], lat degrees [n,h,w]) on the CPU for one fixture case.  Regression
    predictions are what the heads return (normalised vectors, latitudes clamped to [-1, 1]); classification ones are logits."""
    g = torch.Generator().manual_seed(seed)
    up = random_up(g, n, h, w)
    lat = random_lat_deg(g, n, h, w)
    if loss_type == "regression":
        v = torch.randn((n, 2, h, w), generator=g) + 2.0 * up.permute(0, 3, 1, 2)
        pg = v / v.norm(dim=1, keepdim=True).clamp_min(1e-12)
        pl = (torch.sin(lat.double() * (math.pi / 180)).float()[:, None] + 0.3 * torch.randn((n, 1, h, w), generator=g)).clamp(-1, 1)
    else:
        pg = 3.0 * torch.randn((n, NUM_BIN, h, w), generator=g)
        pl = 3.0 * torch.randn((n, NUM_LAT, h, w), generator=g)
    return pg, pl, up, lat


def special_vectors():
    """[2, 1, K] float32 vectors: the axes, bin centres, zero vectors and, found by search, vectors whose float32 angle pipeline
    lands exactly on a rounding boundary (k + 0.5 bins: ties to even)."""
    vs = [(1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), (0.0, -1.0), (0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (1e-30, 0.0), (-1.0, -0.0), (-1.0, 1e-30)]
    for k in range(NUM_BIN - 1):   # bin centres
        a = math.radians(k * 5.0 - 180.0)
        vs.append((math.cos(a), math.sin(a)))
    rng = np.random.default_rng(5)
    ties = 0
    for k in range(NUM_BIN - 1):
        a0 = math.radians(k * 5.0 + 2.5 - 180.0)
        for _ in range(4000):
            a = a0 + rng.normal() * 1e-6
            x, y = np.float32(math.cos(a)), np.float32(math.sin(a))
            q = float(_angle_over_bin(torch.tensor([x]), torch.tensor([y]), NUM_BIN)[0])
            if q == k + 0.5:
                vs.append((float(x), float(y)))
                ties += 1
                break
    v = torch.tensor(vs, dtype=torch.float32).t().reshape(2, 1, -1)
    return v, ties


def _angle_over_bin(x, y, num_bin):
    a = (torch.atan2(y, x) / np.pi * 180 + 180) % 360
    return torch.div(a, 360 / (num_bin - 1))


def encode_bin(v, num_bin):
    """[2, H, W] float32 -> int64 [H, W] (utils.py:94-111)."""
    lab = torch.round(_angle_over_bin(v[0], v[1], num_bin)).long()
    lab[lab == num_bin - 1] = 0
    lab[(v[0] == 0) & (v[1] == 0)] = num_bin - 1
    return lab


def latitude_boundaries(num_classes):
    return (np.float32(-90.0) + np.arange(1, num_classes, dtype=np.float32) * np.float32(180.0 / num_classes)).astype(np.float32)


def encode_bin_latitude(lat_deg, num_classes):
    """float32 degrees -> int64 labels (utils.py:133-146): the number of boundaries below the value (searchsorted 'left')."""
    a = np.asarray(lat_deg, np.float32)
    return torch.from_numpy(np.searchsorted(latitude_boundaries(num_classes), a, side="left").astype(np.int64))


def decode_bin(lab, num_bin):
    """Inverse of encode_bin (utils.py:114-130): bin centre angle, (0, 0) for bin num_bin - 1.  float64 [2, ...]."""
    a = (lab.double() * (360 / (num_bin - 1)) - 180) / 180 * math.pi
    v = torch.stack([torch.cos(a), torch.sin(a)])
    v[:, lab == num_bin - 1] = 0
    return v


def targets(up, lat, loss_type, lat_mode="deg"):
    """The targets rule: up [n,H,W,2], lat [n,H,W] -> (gt_gravity, gt_latitude)."""
    if loss_type == "regression":
        rad = lat.double() * (math.pi / 180) if lat_mode == "deg" else lat.double()
        return up.permute(0, 3, 1, 2).contiguous(), torch.sin(rad).float()[:, None]
    deg = lat if lat_mode == "deg" else lat * np.float32(180 / math.pi)
    gg = torch.stack([encode_bin(u.permute(2, 0, 1), NUM_BIN) for u in up])
    gl = torch.stack([encode_bin_latitude(d.numpy(), NUM_LAT) for d in deg])
    return gg, gl


def _msg(d, mask):
    """msgil_norm_loss (loss_fns.py:5-43) of d = pred - gt [n, c, H, W] float64 with bool mask, summed over the 4 scales."""
    tot = 0.0
    for s in range(4):
        st = 2 ** s
        ds, ms = d[:, :, ::st, ::st], mask[:, :, ::st, ::st].double()
        vm, hm = ms[:, :, :-2, :] * ms[:, :, 2:, :], ms[:, :, :, :-2] * ms[:, :, :, 2:]
        vg, hg = (ds[:, :, :-2, :] - ds[:, :, 2:, :]).abs() * vm, (ds[:, :, :, :-2] - ds[:, :, :, 2:]).abs() * hm
        tot += float((vg.sum() + hg.sum()) / (vm.sum() + hm.sum() + 1e-8))
    return tot


def losses(pg, pl, gg, gl, loss_type, wg=1.0, wl=1.0, ig=IGNORE_GRAVITY, il=IGNORE_LATITUDE):
    """The losses dict in float64 (persformer_heads.py:60-70)."""
    if loss_type == "regression":
        p, t = pg.double(), gg.double()
        m = t.norm(dim=1, keepdim=True) > 1e-5
        l2 = ((p - t) ** 2).sum(1, keepdim=True)[m]
        pl_, tl = pl.double(), gl.double()
        return {"gravity-msg-normal-loss": 0.1 * _msg(p - t, m.expand(-1, 2, -1, -1)) * wg,
                "gravity-l2-loss": (float(l2.mean()) if l2.numel() else float("nan")) * wg,
                "latitude-msg-normal-loss": 0.1 * _msg(pl_ - tl, torch.ones_like(tl, dtype=torch.bool)) * wl,
                "latitude-l2-loss": float(((pl_ - tl) ** 2).mean()) * wl}

    def ce(logits, lab, ignore):
        lp = torch.log_softmax(logits.double(), dim=1)
        keep = lab != ignore
        if not bool(keep.any()):
            return float("nan")
        lab_c = lab.clamp(0, logits.shape[1] - 1)
        v = -lp.gather(1, lab_c[:, None])[:, 0]
        bad = keep & ((lab < 0) | (lab >= logits.shape[1]))
        if bool(bad.any()):
            return float("nan")
        return float(v[keep].mean())

    return {"loss_gravity": ce(pg, gg, ig) * wg, "loss_latitude": ce(pl, gl, il) * wl}


def error_maps(pu, pl, gu, gl, lat_mode="deg", mask=None):
    """The field-error rule in float64: pu [2,H,W], pl [H,W] degrees, gu [H,W,2], gl [H,W] -> (up map, latitude map), NaN at
    invalid pixels."""
    pu, pl, gu, gl = (np.asarray(x, np.float64) for x in (pu, pl, gu, gl))
    if lat_mode == "rad":
        gl = gl * (180.0 / math.pi)
    px, py, gx, gy = pu[0], pu[1], gu[..., 0], gu[..., 1]
    m = np.ones(gl.shape, bool) if mask is None else np.asarray(mask, bool)
    with np.errstate(invalid="ignore"):
        vu = m & np.isfinite(gx) & np.isfinite(gy) & (np.sqrt(gx * gx + gy * gy) > 1e-5)
        pok = np.isfinite(px) & np.isfinite(py) & (np.sqrt(px * px + py * py) > 1e-5)
        eu = np.degrees(np.arctan2(np.abs(px * gy - py * gx), px * gx + py * gy))
        eu = np.where(pok, eu, 180.0)
        vl = m & np.isfinite(gl)
        el = np.where(np.isfinite(pl), np.abs(pl - gl), np.inf)
    return np.where(vu, eu, np.nan), np.where(vl, el, np.nan)


def stats(err_map, thresholds):
    """count, mean, median (np.median) and the fractions below each threshold of the non-NaN values of a map."""
    v = np.asarray(err_map, np.float64)
    v = v[~np.isnan(v)]
    if v.size == 0:
        return 0, float("nan"), float("nan"), [float("nan")] * len(thresholds)
    return int(v.size), float(v.mean()), float(np.median(v)), [float((v < t).mean()) for t in thresholds]
