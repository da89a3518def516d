"""``model.e2fgvi_hq`` — resolution-agnostic variant (reference: model/e2fgvi_hq.py): run-time fold size and a
3x3 ``sc.bias_conv`` instead of the learned ``sc.bias`` map."""
from .discriminator import Discriminator  # noqa: F401
from .generator import BaseNetwork, Encoder, deconv  # noqa: F401
from .generator import InpaintGeneratorHQ as InpaintGenerator  # noqa: F401

__all__ = ["InpaintGenerator", "Encoder", "deconv", "BaseNetwork", "Discriminator"]
