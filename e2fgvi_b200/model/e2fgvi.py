"""``model.e2fgvi`` — fixed 432x240 variant (reference: model/e2fgvi.py).  ``Discriminator`` trains on the GPU
(forward and backward); the generator has no backward pass yet, so only the discriminator step of train.py runs here."""
from .discriminator import Discriminator  # noqa: F401
from .generator import BaseNetwork, Encoder, InpaintGenerator, deconv  # noqa: F401

__all__ = ["InpaintGenerator", "Encoder", "deconv", "BaseNetwork", "Discriminator"]
