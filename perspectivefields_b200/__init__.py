"""perspectivefields_b200 -- H100-native (sm_90a CUDA) implementation of the PerspectiveFields inference path.

    from perspectivefields_b200 import PerspectiveFields
    model = PerspectiveFields("Paramnet-360Cities-edina-centered").eval().cuda()
    pred = model.inference(img_bgr)            # same dictionary as perspective2d.PerspectiveFields
    preds = model.inference_batch([img, ...])

``perspectivefields_b200.compat.install()`` additionally registers the package under the reference's import name
(``from perspective2d import PerspectiveFields``).
"""
from .perspectivefields import PerspectiveFields  # noqa: F401
from .variants import model_zoo  # noqa: F401

__all__ = ["PerspectiveFields", "model_zoo"]
