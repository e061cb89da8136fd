"""CPU: host-side logic of the product package -- zoo/config surface, checkpoint schema and loader semantics,
weight repack algebra (composition + border-class bias, BN folding, hi/lo split), result assembly rules."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pf_test_util as U
from oracle import schema as oschema
from oracle import weights_gen as wg
from perspectivefields_b200 import checkpoint, variants, weights


def test_zoo_matches_reference_surface():
    assert list(variants.model_zoo) == ["Paramnet-360Cities-edina-centered", "Paramnet-360Cities-edina-uncentered",
                                        "PersNet-360Cities", "PersNet_Paramnet-GSV-uncentered", "PersNet_Paramnet-GSV-centered"]
    for k, v in variants.model_zoo.items():
        assert set(v) == {"weights", "config_file", "param", "description"}
        assert v["weights"].startswith("https://huggingface.co/spaces/jinlinyi/PerspectiveFields/resolve/main/models/")
        assert v["param"] == (variants.VARIANTS[k]["param_net"] is not None)


@pytest.mark.parametrize("version", list(variants.VARIANTS))
def test_schema_equals_oracle_schema(version):
    assert checkpoint.checkpoint_schema(version) == oschema.state_dict_schema(version)


def test_split_hi_lo_precision():
    w = torch.randn(1000, dtype=torch.float64)
    hi, lo = weights.split_hi_lo(w)
    assert hi.dtype == lo.dtype == torch.bfloat16
    assert ((hi.double() + lo.double() - w).abs() / w.abs()).max() < 2 ** -15


def test_repack_composition_and_bn_fold():
    ver = "Paramnet-360Cities-edina-uncentered"
    sd = wg.synth_state_dict(ver, 1)
    rp = weights.repack(sd, variants.VARIANTS[ver])
    # composed linear_c2 o linear_c2_proc of the latitude head, incl. border-class bias
    p = "persformer_heads.latitude_head."
    x = torch.randn(1, 128, 7, 9)
    t = F.linear(x.flatten(2).transpose(1, 2), sd[p + "linear_c2.proj.weight"], sd[p + "linear_c2.proj.bias"]).permute(0, 2, 1).reshape(1, -1, 7, 9)
    ref = F.conv2d(t, sd[p + "linear_c2_proc.weight"], sd[p + "linear_c2_proc.bias"], padding=1).double()
    W = (rp["head.proc2.whi"].double() + rp["head.proc2.wlo"].double())[256:].reshape(256, 3, 3, 128).permute(0, 3, 1, 2)
    got = F.conv2d(x.double(), W, None, padding=1)
    b = rp["head.proc2.b"].reshape(9, 512)[:, 256:].double()
    for y in range(7):
        for xx in range(9):
            cls = (0 if y == 0 else (2 if y == 6 else 1)) * 3 + (0 if xx == 0 else (2 if xx == 8 else 1))
            got[0, :, y, xx] += b[cls]
    assert U.rel_err(got, ref) < 2e-5
    # BN folded into the low-level encoder conv
    img = torch.randn(1, 3, 32, 32) * 50
    ref = F.relu(F.batch_norm(F.conv2d(img, sd["ll_enc.conv1.weight"], None, stride=2, padding=3), sd["ll_enc.bn1.running_mean"],
                              sd["ll_enc.bn1.running_var"], sd["ll_enc.bn1.weight"], sd["ll_enc.bn1.bias"], False, 0.1, 1e-5))
    wk = rp["llencg.whi"].double() + rp["llencg.wlo"].double()      # [64][160]: K = (ky, kx, c), 147 columns + 13 of padding
    assert wk.shape == (64, 160) and not wk[:, 147:].any()
    wf = wk[:, :147].reshape(64, 7, 7, 3).permute(0, 3, 1, 2)
    got = F.relu(F.conv2d(img.double(), wf, rp["llencg.b"].double(), stride=2, padding=3))
    assert U.rel_err(got, ref) < 1e-5
    # every GEMM layer has hi/lo/bias, K multiple of 32
    for k in rp:
        if k.endswith(".whi"):
            assert k[:-4] + ".wlo" in rp and k[:-4] + ".b" in rp


def test_model_surface_without_gpu():
    m, sd = U.make_model("PersNet_Paramnet-GSV-centered", seed=2, device=None)
    assert m.version == "PersNet_Paramnet-GSV-centered" and m.param_on is True and m.input_format == "BGR"
    assert m.cfg.MODEL.RECOVER_RPF is True and m.cfg.MODEL.RECOVER_PP is False and m.cfg.DATALOADER.RESIZE == [320, 320]
    assert (m.aug.new_h, m.aug.new_w, m.aug.interp) == (320, 320, 2)     # perspectivefields.py:155; PIL.Image.BILINEAR == 2
    got = m.state_dict()
    assert list(got) == [k for k, _ in oschema.state_dict_schema(m.version)]
    assert all(torch.equal(got[k], sd[k]) for k in sd)
    with pytest.raises(RuntimeError):
        m.train()
    assert m.eval() is m
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.inference(np.zeros((8, 8, 3), np.uint8))
    with pytest.raises(KeyError):
        type(m)("no-such-version")
    # strict=False tolerance + shape check, as torch does
    r = m.load_state_dict({"backbone.norm1.weight": torch.ones(64), "extra": torch.ones(1)}, strict=False)
    assert "extra" in r.unexpected_keys and len(r.missing_keys) == len(got) - 1
    with pytest.raises(RuntimeError, match="size mismatch"):
        m.load_state_dict({"backbone.norm1.weight": torch.ones(65)}, strict=False)


def test_compat_alias():
    import sys

    from perspectivefields_b200 import compat

    sys.modules.pop("perspective2d", None)
    sys.modules.pop("perspective2d.perspectivefields", None)
    pkg = compat.install()
    from perspective2d import PerspectiveFields  # noqa
    from perspective2d.perspectivefields import model_zoo  # noqa

    assert PerspectiveFields is pkg.PerspectiveFields and "PersNet-360Cities" in model_zoo
    sys.modules.pop("perspective2d", None)
    sys.modules.pop("perspective2d.perspectivefields", None)


def test_gelu_polynomial_in_the_kernels_matches_erf():
    """csrc/common.cuh:gelu_erf evaluates erf through a degree-8 polynomial for log2 erfc and one ex2.  The coefficients are
    read from the source and the same fp32 arithmetic is replayed here against scipy's erf in float64: the error must stay at
    the level of fp32 rounding (the libm erff route measures 4.5e-7 on the same grid)."""
    import math
    import os
    import re
    import numpy as np
    from scipy.special import erf
    src = open(os.path.join(os.path.dirname(__file__), "..", "perspectivefields_b200", "csrc", "common.cuh")).read()
    body = src[src.index("float gelu_erf(float x)"):]
    body = body[body.index("#else"):body.index("#endif")]
    zmax = float(re.search(r"fminf\(fabsf\(x\) \* [0-9.]+f, ([0-9.]+)f\)", body).group(1))
    lead = float(re.search(r"float q = (-?[0-9.e+-]+)f;", body).group(1))
    rest = [float(m) for m in re.findall(r"q = fmaf\(q, z, (-?[0-9.e+-]+)f\);", body)]
    assert len(rest) == 8
    f32 = np.float32
    x = np.linspace(-12, 12, 2_000_001).astype(f32)
    z = np.minimum(np.abs(x) * f32(0.70710678118654752440), f32(zmax))
    q = np.full_like(z, f32(lead))
    for c in rest:
        q = q * z + f32(c)
    assert abs(rest[-1] + 1.0) < 1e-7                     # the constant term carries the 1/2: ex2 returns erfc / 2
    h = np.exp2(q).astype(f32)
    t = (np.abs(x) * (f32(0.5) - h)).astype(f32)
    g = (x.astype(np.float64) * 0.5 + t.astype(np.float64)).astype(f32).astype(np.float64)     # fmaf(x, 0.5, t): one rounding
    xd = x.astype(np.float64)
    exact = 0.5 * xd * (1 + erf(xd / math.sqrt(2)))
    err = np.abs(g - exact)
    assert err.max() < 6e-7
    assert (err / np.maximum(np.abs(xd), 1)).max() < 2e-7


def test_up2_conv3_composition():
    """weights.py:_compose_up2_conv3: conv3x3(pad 1) o bilinear x2 equals four 3x3 phase convolutions on the low-res grid
    everywhere except the two outermost output rows / columns (those are recomputed by conv1_ring_kernel)."""
    import torch.nn.functional as F
    from perspectivefields_b200.weights import _compose_up2_conv3
    torch.manual_seed(0)
    x = torch.randn(2, 6, 9, 11, dtype=torch.float64)
    w = torch.randn(5, 6, 3, 3, dtype=torch.float64)
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False), w, padding=1)
    y = F.conv2d(x, _compose_up2_conv3(w), padding=1)              # [2, 4*5, 9, 11], row = (py*2+px)*5 + o
    y = y.view(2, 2, 2, 5, 9, 11).permute(0, 3, 4, 1, 5, 2).reshape(2, 5, 18, 22)
    assert (y - ref)[:, :, 2:-2, 2:-2].abs().max() < 1e-12
    assert (y - ref).abs().max() > 1e-3                            # the ring really differs: it needs the exact kernel


def test_fast_asin_and_atan2_polynomials_of_the_kernels():
    """csrc/prepost.cuh: fast_asinf (post-process: degrees = asin(sin latitude)) and fast_atan2_deg (camera_fields_kernel), emulated
    in float32 numpy with the coefficients parsed from the source, against float64 libm: <= 2e-7 rad and <= 1e-5 degrees."""
    import os
    import re

    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "perspectivefields_b200", "csrc", "prepost.cuh")).read()
    f = np.float32

    def coeffs(fn):
        body = src[src.index(fn):]
        body = body[:body.index("\n}\n")]
        first = re.search(r"float p = ([-0-9.e]+)f;", body).group(1)
        rest = re.findall(r"p = fmaf\(p, z, ([-0-9.e]+)f\);", body)
        return [f(first)] + [f(c) for c in rest]

    ca, ct = coeffs("float fast_asinf(float x)"), coeffs("float fast_atan2_deg(float y, float h)")
    assert len(ca) == 5 and len(ct) == 4
    x = np.concatenate([np.linspace(-1, 1, 2000001), [0.5, -0.5, 0.4999999, 0.5000001, 1.0, -1.0, 0.0]]).astype(f)
    a = np.abs(x)
    big = a > f(0.5)
    z = np.where(big, (f(1) - a) * f(0.5), a * a).astype(f)
    s_ = np.where(big, np.sqrt(z).astype(f), a).astype(f)
    p = ca[0]
    for c in ca[1:]:
        p = (p * z + c).astype(f)
    r = (s_ + (s_ * z).astype(f) * p).astype(f)
    r = np.where(big, (f(1.5707963267948966) - (r + r)).astype(f), r).astype(f)
    r = np.copysign(r, x)
    assert np.abs(r.astype(np.float64) - np.arcsin(x.astype(np.float64))).max() < 2e-7
    rs = np.random.RandomState(0)
    yw, h = rs.uniform(-3, 3, 1000000).astype(f), np.abs(rs.uniform(0.01, 3, 1000000)).astype(f)
    a = np.abs(yw)
    hi = a > f(2.414213562373095) * h
    mid = (~hi) & (a > f(0.4142135623730950) * h)
    num = np.where(hi, -h, np.where(mid, a - h, a)).astype(f)
    den = np.where(hi, a, np.where(mid, a + h, h)).astype(f)
    q = (num / den).astype(f)
    z = (q * q).astype(f)
    p = ct[0]
    for c in ct[1:]:
        p = (p * z + c).astype(f)
    pr = (q + (q * z).astype(f) * p).astype(f)
    deg = np.copysign((pr.astype(np.float64) * np.float64(f(57.29577951308232)) + np.where(hi, 90.0, np.where(mid, 45.0, 0.0))).astype(f), yw)   # fmaf: one rounding
    ref = np.degrees(np.arctan2(yw.astype(np.float64), h.astype(np.float64)))
    assert np.abs(deg.astype(np.float64) - ref).max() < 1e-5


# (BN, KB) the dispatcher picks for test_gpu_ops.TC_CASES on a 132-SM H100, in order (halo mode: 3x3 / s1 / p1, Cin % 64 == 0)
TC_PICKS = [("halo", 256, 32), ("halo", 256, 32), ("halo", 256, 32), ("gemm", 32, 64), ("gemm", 32, 32), ("halo", 256, 32),
            ("gemm", 32, 64), ("gemm", 32, 32), ("gemm", 32, 64), ("gemm", 32, 64), ("halo", 32, 64), ("halo", 64, 64),
            ("gemm", 32, 64), ("gemm", 32, 64), ("gemm", 160, 32), ("gemm", 192, 32), ("gemm", 160, 32), ("gemm", 224, 32),
            ("gemm", 64, 64)]


def test_tile_dispatch_of_the_op_cases():
    """pf_tma_pick_tile (the host-side dispatcher of the TMA engine, no device needed) on the op-test shapes: records which
    instantiation each of them exercises, so that a change of the cost model shows up here and in the case comments."""
    import ctypes

    from perspectivefields_b200 import _native
    from test_gpu_ops import TC_CASES

    _native.build()
    L = _native.lib()
    got = []
    for B, H, W, Cin, N, K, s, p, *_ in TC_CASES:
        halo = K == 3 and s == 1 and p == 1 and Cin % 64 == 0
        M = B * ((H + 2 * p - K) // s + 1) * ((W + 2 * p - K) // s + 1)
        bn, kb = ctypes.c_int(), ctypes.c_int()
        _native.check(L.pf_tma_pick_tile(int(halo), M, N, K * K * Cin, 132, ctypes.byref(bn), ctypes.byref(kb)))
        got.append(("halo" if halo else "gemm", bn.value, kb.value))
    assert got == TC_PICKS
    assert L.pf_tma_pick_tile(2, 1, 32, 32, 132, ctypes.byref(bn), ctypes.byref(kb)) < 0
