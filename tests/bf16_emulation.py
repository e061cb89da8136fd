"""CPU emulation of the engine's opt-in bf16 precision mode (option "bf16", ``PerspectiveFields(..., precision="bf16")``).
TEST INFRASTRUCTURE: it sizes the end-to-end error of the mode against the fp32 oracle before any GPU run.

``with Bf16Emulation(): oracle.model.forward(...)`` rounds both operands of every product the engine runs on tensor cores to
bf16 (``t.bfloat16().float()``, round to nearest even: the hi plane of the engine's split) and keeps fp32 accumulation:

  * ``F.conv2d`` with ``groups == 1`` (patch embeds, spatial reduction, linear_c proc convs, RCU / fusion convs, conv_fuse_conv0 /
    conv1, the ParamNet downsampling convs, and the two 7x7 stems, which run on the engine as patch gather + GEMM);
  * ``F.linear`` (q, kv, proj, fc1, fc2, linear_c, ConvNeXt pwconv1 / pwconv2);
  * both attention matmuls, q k^T and softmax(.) v.

Left in fp32, as the engine runs them on CUDA cores: depthwise convolutions (``groups > 1``), the 1x1 prediction convs
(32 input channels), the ParamNet 4x4 stem (4 input channels, ``stem_conv_launch``) and the ParamNet head Linear
(768 -> <= 7 outputs, ``layers.cuh:param_tail_kernel``, which also runs the final LayerNorm).

The engine rounds at other points than the reference graph (the composed linear_c o proc conv, the phase-composed conv1 and
its fp32 border ring, the folded BatchNorm of the low-level encoder), so this measures the size of the error, not the engine's
bits.
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch.overrides import TorchFunctionMode

# Bounds of the end-to-end error of precision="bf16" against the fp32 oracle, for every variant and output (DESIGN.md section 3).
# rel: max|a - b| / max|b| per returned tensor ("pred_latitude_original": sine domain, see sine_rel_err); deg: ParamNet angles
# (roll, pitch, vfov / general_vfov) in degrees.  The emulation's largest errors on the two golden images are 0.035 and 0.18
# degrees; the bounds leave about 3x / 5x for the engine's other rounding points.  They are the tolerances of tests/test_gpu_bf16.py.
REL_BOUND = 0.1
DEG_BOUND = 1.0
ANGLE_KEYS = ("pred_roll", "pred_pitch", "pred_vfov", "pred_general_vfov")


def _bf16(t):
    return t.bfloat16().float()


def _tensor_core_conv(w, groups):
    if groups != 1:
        return False                                  # depthwise
    o, i, kh, kw = w.shape
    if kh == 1 and kw == 1 and i == 32:
        return False                                  # 1x1 prediction conv (CUDA-core tail)
    if i == 4:
        return False                                  # ParamNet 4x4 stem (CUDA-core direct convolution)
    return True


class Bf16Emulation(TorchFunctionMode):
    """Context manager: bf16-rounded operands for the tensor-core products of oracle.model (see module docstring)."""

    def __init__(self, stems=True):
        super().__init__()
        self.stems = stems   # False: keep the two 7x7 stems (3 input channels) in fp32, to size their share of the error

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = dict(kwargs or {})
        if func is F.conv2d:
            x, w = args[0], args[1]
            groups = kwargs.get("groups", args[6] if len(args) > 6 else 1)
            if _tensor_core_conv(w, groups) and (self.stems or w.shape[1] != 3):
                args = (_bf16(x), _bf16(w)) + tuple(args[2:])
        elif func is F.linear:
            x, w = args[0], args[1]
            if not (w.shape[1] == 768 and w.shape[0] <= 8):   # ParamNet head: CUDA-core tail
                args = (_bf16(x), _bf16(w)) + tuple(args[2:])
        elif func in (torch.matmul, torch.Tensor.matmul, torch.Tensor.__matmul__):   # (`a @ b` arrives as Tensor.matmul)
            args = (_bf16(args[0]), _bf16(args[1])) + tuple(args[2:])
        return func(*args, **kwargs)


def sine_rel_err(a, b):
    """rel err of a latitude field in degrees, measured on sin(latitude) (asin is not Lipschitz at +-90 degrees)."""
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    sa, sb = torch.sin(torch.deg2rad(a)), torch.sin(torch.deg2rad(b))
    return ((sa - sb).abs().max() / sb.abs().max().clamp_min(1e-30)).item()


def rel_err(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def error_table(out, ref, classification=False):
    """{output: worst error over the images} of ``out`` against ``ref`` (lists of result dicts).  Tensors: rel err (latitude in
    degrees: sine domain); ParamNet angles: degrees; the argmax-decoded *_original fields of the classification variant are
    skipped (discontinuous in the logits; the GPU test compares them on stable pixels)."""
    worst = {}
    for o, r in zip(out, ref):
        for k, v in r.items():
            if isinstance(v, str) or (classification and k.endswith("_original")):
                continue
            a, v = torch.as_tensor(o[k]).detach().cpu(), torch.as_tensor(v).detach().cpu()
            if k in ANGLE_KEYS:
                e = (a.double() - torch.as_tensor(v).double()).abs().max().item()
            elif k == "pred_latitude_original":
                e = sine_rel_err(a, v)
            elif torch.as_tensor(v).ndim == 0:
                continue                               # rel_cx / rel_cy / rel_focal: covered by the angles they derive from
            else:
                e = rel_err(a, v)
            worst[k] = max(worst.get(k, 0.0), e)
    return worst


def bound(key):
    return DEG_BOUND if key in ANGLE_KEYS else REL_BOUND


def emulate(sd, version, imgs, stems=True):
    """(fp32 oracle results, emulated bf16 results) of oracle.model.inference_batch on ``imgs``."""
    from oracle import model as om

    ref = om.inference_batch(sd, version, imgs)
    with Bf16Emulation(stems=stems):
        out = om.inference_batch(sd, version, imgs)
    return ref, out


if __name__ == "__main__":   # prints the DESIGN.md table: python tests/bf16_emulation.py
    import os
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from golden_util import golden_images
    from oracle import weights_gen as wg
    from oracle.variants import VARIANTS

    imgs = golden_images()
    for version in VARIANTS:
        sd = wg.synth_state_dict(version, 0)
        for stems in (True, False):
            ref, out = emulate(sd, version, imgs, stems)
            t = error_table(out, ref, VARIANTS[version]["gravity"] == "classification")
            print(version, "stems bf16" if stems else "stems fp32", {k: float(np.format_float_positional(v, 3)) for k, v in t.items()})
