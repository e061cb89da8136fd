"""CPU restatement of ``PanoCam.crop_equi`` and the crop of ``PanoCam(path).get_image`` (perspective2d/utils/panocam.py:121-249).
TEST INFRASTRUCTURE (oracle).

The reference wraps ``equilib.equi2pers`` (equilib 0.3.0), which is neither in the reference tree nor installable here, so the
crop's geometry and sampler are this project's rule (DESIGN.md section 1), restated below in float64 numpy in the order of
operations of csrc/equi.cuh.  ``equi2pers`` is a drop-in with the keyword arguments the reference passes: the golden generator
(tests/golden/make_golden_equi.py) installs it in the unmodified reference, which pins the wrapper's own arithmetic (fov_x, the
rot dict, the dtype casts, ToTensor / ToPILImage / cv2 steps) to this file.  The geometry is pinned through the ground truth the
reference pairs with the crop (``get_lat`` / ``get_up``, tests/test_oracle_equi_crop.py).  The sampler is the one of
tests/oracle_pano.py (parity unpinned).
"""
import math

import numpy as np

import oracle_pano

CALLS = []      # the arguments of every equi2pers call (the golden generator records what the reference's wrapper passes)


def wrapper_args(vfov, im_w, im_h, azimuth, elevation, roll, ar):
    """:216-225 -> (fov_x in degrees, rot dict in radians), the reference's own expressions."""
    fov_x = float(2 * np.arctan(np.tan(vfov * np.pi / 180.0 / 2) * ar) * 180 / np.pi)
    rot = {"roll": float(roll / 180 * np.pi), "pitch": -float(elevation / 180 * np.pi), "yaw": -float(azimuth / 180 * np.pi)}
    return fov_x, rot


def pixel_map(h, w, fov_x, rot, hp, wp):
    """The rule's geometry: (u, v) panorama pixel of every view pixel, plus (theta, phi), float64 [h, w] each."""
    f = w / (2 * math.tan(fov_x * math.pi / 180 / 2))
    roll, el, az = rot["roll"], -rot["pitch"], -rot["yaw"]
    cr, sr, ce, se, ca, sa = math.cos(roll), math.sin(roll), math.cos(el), math.sin(el), math.cos(az), math.sin(az)
    j, i = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    x, y = (j - w / 2.0) / f, (i - h / 2.0) / f                 # x right, y down, z = 1 forward
    xr, yr = x * cr - y * sr, x * sr + y * cr                   # roll
    ye, ze = yr * ce - se, yr * se + ce                         # elevation
    xa, za = xr * ca + ze * sa, -(xr * sa) + ze * ca            # azimuth
    n = np.sqrt((xa * xa + ye * ye) + za * za)
    theta = np.arctan2(xa, za)
    phi = -np.arcsin(ye / n)
    return (theta + np.pi) * (wp / (2 * np.pi)), (np.pi / 2 - phi) * (hp / np.pi), theta, phi


def sample(chw, u, v, mode):
    """chw: [C, Hp, Wp] (any real dtype) -> float64 [C, h, w]: oracle_pano's bilinear sampler, or the nearest pixel."""
    if mode == "bilinear":
        return oracle_pano.grid_sample_precast(chw, np.stack((v, u)))
    if mode == "nearest":
        _, hp, wp = chw.shape
        x = np.mod(np.floor(u + 0.5).astype(np.int64), wp)
        y = np.clip(np.floor(v + 0.5), 0, hp - 1).astype(np.int64)
        return chw.astype(np.float64)[:, y, x]
    raise ValueError(f"unknown mode {mode!r}")


def equi2pers(equi, rot, w_pers, h_pers, fov_x, skew=0.0, sampling_method="default", mode="bilinear"):
    """Drop-in for ``equilib.equi2pers`` as panocam.py:176-185 and :234-243 call it: torch [C, Hp, Wp] float32 -> torch float32
    [C, h_pers, w_pers] (the sample rounded to float32) on the input's device."""
    import torch
    CALLS.append({"fov_x": fov_x, "w": w_pers, "h": h_pers, "mode": mode, **rot})
    chw = equi.detach().cpu().numpy()
    u, v, _, _ = pixel_map(h_pers, w_pers, fov_x, rot, chw.shape[1], chw.shape[2])
    return torch.from_numpy(sample(chw, u, v, mode).astype(np.float32)).to(equi.device)


def to_output(s, dtype, unit=False):
    """float64 sample -> the crop's values: rounded to float32 (what the sampler returns), then cast to the panorama's dtype
    (crop_equi's np.asarray(.., dtype=equi_img.dtype): uint8 truncates); unit: times 255 in float32 and truncated to uint8
    (ToPILImage's mul(255).byte(), or get_image's np.asarray(x * 255, uint8) for BGR)."""
    s32 = np.asarray(s).astype(np.float32)
    if unit:
        return np.clip(s32 * np.float32(255), 0, 255).astype(np.uint8)
    if np.dtype(dtype) == np.uint8:
        return np.clip(s32, 0, 255).astype(np.uint8)
    return s32


def crop_equi_full(equi_img, vfov, im_w, im_h, azimuth, elevation, roll, ar, mode="bilinear", unit=False, swap_rb=False):
    """The crop and what the tests compare against: dict with im (the crop, [H, W, 3] or [H, W] in the output dtype), sample
    (float64 [H, W, C], the sampler's value before any cast), u, v, theta, phi (float64 [H, W]).
    unit=False: crop_equi (:226-249), the float32 sample cast back to the panorama's dtype (uint8: truncated).
    unit=True (uint8 only): get_image (:163-186), ToTensor's p / 255 in float32, sampled, times 255 in float32, truncated.
    swap_rb: channels in the order 2, 1, 0 (get_image's img_format="BGR")."""
    equi_img = np.asarray(equi_img)
    chw = equi_img.transpose(2, 0, 1) if equi_img.ndim == 3 else equi_img[None]
    if unit:
        chw = chw.astype(np.float32) / np.float32(255)
    fov_x, rot = wrapper_args(vfov, im_w, im_h, azimuth, elevation, roll, ar)
    u, v, theta, phi = pixel_map(int(im_h), int(im_w), fov_x, rot, chw.shape[1], chw.shape[2])
    s = sample(chw, u, v, mode)
    if swap_rb:
        s = s[::-1]
    im = to_output(s, equi_img.dtype, unit).transpose(1, 2, 0)
    if equi_img.ndim == 2:
        im = im[:, :, 0]
    return {"im": im, "sample": s.transpose(1, 2, 0), "u": u, "v": v, "theta": theta, "phi": phi}


def crop_equi(equi_img, vfov, im_w, im_h, azimuth, elevation, roll, ar, mode):
    """PanoCam.crop_equi's signature -> the crop."""
    return crop_equi_full(equi_img, vfov, im_w, im_h, azimuth, elevation, roll, ar, mode)["im"]
