"""CPU: the opt-in bf16 precision mode's public surface and its error budget.

``PerspectiveFields(version, precision=...)`` validation, and the CPU emulation of the mode (tests/bf16_emulation.py: bf16-rounded
operands for every product the engine runs on tensor cores, fp32 elsewhere) against the fp32 oracle on the two golden images
(480 x 640 and 360 x 500) for all five variants: every output must stay within the bounds DESIGN.md section 3 states and the GPU
test applies to the engine."""
import pytest
import torch

import pf_test_util as U
from bf16_emulation import Bf16Emulation, bound, emulate, error_table
from golden_util import golden_images
from oracle import weights_gen as wg
from oracle.variants import VARIANTS


def test_precision_argument_is_validated_and_stored_as_an_engine_option():
    version = "Paramnet-360Cities-edina-centered"
    m, _ = U.make_model(version, device=None)
    assert "bf16" not in m._options
    m, _ = U.make_model(version, device=None, model_kwargs={"precision": "fp32"})
    assert "bf16" not in m._options
    m, _ = U.make_model(version, device=None, model_kwargs={"precision": "bf16"})
    assert m._options == {"bf16": 1}
    m, _ = U.make_model("PersNet-360Cities", device=None, model_kwargs={"precision": "bf16", "logits": False})
    assert m._options == {"decode_only": 1, "bf16": 1}
    from perspectivefields_b200 import PerspectiveFields
    for bad in ("fp16", "BF16", "tf32", None, 16):
        with pytest.raises(ValueError):
            PerspectiveFields(version, precision=bad)


def test_emulation_rounds_only_the_tensor_core_operands():
    """Depthwise convs, 1x1 prediction convs (32 inputs), the ParamNet 4x4 stem (4 inputs) and its 768 -> n head stay fp32."""
    import torch.nn.functional as F

    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 32, 6, 6, generator=g)
    exact = {
        "dw": (lambda: F.conv2d(x, torch.randn(32, 1, 3, 3, generator=g), None, padding=1, groups=32)),
        "pred": (lambda: F.conv2d(x, torch.randn(2, 32, 1, 1, generator=g))),
        "pn_stem": (lambda: F.conv2d(x[:, :4], torch.randn(96, 4, 4, 4, generator=g), stride=2)),
        "pn_head": (lambda: F.linear(torch.randn(2, 768, generator=g), torch.randn(5, 768, generator=g))),
    }
    rounded = {
        "conv3x3": (lambda: F.conv2d(x, torch.randn(8, 32, 3, 3, generator=g), None, padding=1)),
        "stem": (lambda: F.conv2d(x[:, :3], torch.randn(8, 3, 7, 7, generator=g), padding=3)),
        "linear": (lambda: F.linear(torch.randn(4, 64, generator=g), torch.randn(16, 64, generator=g))),
        "matmul": (lambda: torch.randn(4, 64, generator=g) @ torch.randn(64, 16, generator=g)),
    }
    for name, f in list(exact.items()) + list(rounded.items()):
        state = g.get_state()
        ref = f()
        g.set_state(state)
        with Bf16Emulation():
            emu = f()
        assert torch.equal(ref, emu) == (name in exact), name


@pytest.mark.parametrize("version", sorted(VARIANTS))
def test_emulated_bf16_error_is_within_the_documented_bounds(version):
    imgs = golden_images()
    assert imgs[0].shape != imgs[1].shape
    sd = wg.synth_state_dict(version, 0)
    ref, out = emulate(sd, version, imgs)
    table = error_table(out, ref, VARIANTS[version]["gravity"] == "classification")
    print(version, {k: round(v, 4) for k, v in table.items()})
    assert "pred_gravity" in table and "pred_latitude" in table
    for k, e in table.items():
        assert e < bound(k), (version, k, e, bound(k))
    # the emulation does round: the error is that of bf16, far above the fp32 path's 1e-3
    assert max(e for k, e in table.items() if bound(k) < 1) > 2e-3
