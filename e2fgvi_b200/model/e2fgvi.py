"""``model.e2fgvi`` — fixed 432x240 variant (reference: model/e2fgvi.py).  ``Discriminator`` trains on the GPU
(forward and backward), and so does the generator's ``update_spynet`` through ``forward_bidirect_flow`` and
``FlowCompletionLoss`` (INTEGRATION "Flow completion").  The rest of the generator has no backward pass yet:
``InpaintGenerator.forward`` is inference-only."""
from .discriminator import Discriminator  # noqa: F401
from .generator import BaseNetwork, Encoder, InpaintGenerator, deconv  # noqa: F401

__all__ = ["InpaintGenerator", "Encoder", "deconv", "BaseNetwork", "Discriminator"]
