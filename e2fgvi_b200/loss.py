"""Losses of the reference's trainer (core/loss.py) that the discriminator step needs, and the flow completion loss
(model/modules/flow_comp.py)."""
import torch
import torch.nn as nn

from .model.modules.flow_comp import FlowCompletionLoss  # noqa: F401


class AdversarialLoss(nn.Module):
    """GAN loss of type ``nsgan`` (BCE), ``lsgan`` (MSE) or ``hinge`` (https://arxiv.org/abs/1711.10337).

    ``loss(outputs, is_real, is_disc=None)``.  Hinge: for the discriminator (``is_disc``) mean(relu(1 - outputs)) on
    real and mean(relu(1 + outputs)) on fake samples; for the generator -mean(outputs).  nsgan / lsgan compare the
    outputs with the real or fake label whatever ``is_disc`` is."""

    def __init__(self, type="nsgan", target_real_label=1.0, target_fake_label=0.0):
        super().__init__()
        if type not in ("nsgan", "lsgan", "hinge"):
            raise ValueError(f"AdversarialLoss: unknown type {type!r} (nsgan, lsgan or hinge)")
        self.type = type
        self.register_buffer("real_label", torch.tensor(target_real_label))
        self.register_buffer("fake_label", torch.tensor(target_fake_label))
        self.criterion = {"nsgan": nn.BCELoss, "lsgan": nn.MSELoss, "hinge": nn.ReLU}[type]()

    def __call__(self, outputs, is_real, is_disc=None):
        if self.type == "hinge":
            if not is_disc:
                return (-outputs).mean()
            return self.criterion(1 + (-outputs if is_real else outputs)).mean()
        labels = (self.real_label if is_real else self.fake_label).expand_as(outputs)
        return self.criterion(outputs, labels)
