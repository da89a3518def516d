"""Functional float64 restatement of the reference's Temporal PatchGAN discriminator (model/e2fgvi.py:271-344) and of
its spectral norm (model/modules/spectral_norm.py:40-96), on plain torch ops.  The CPU tests pin it to the goldens of
the unmodified reference; the GPU tests use it at sizes too large for goldens."""
import torch
import torch.nn.functional as F


def sn_weight(w_orig, u, v, train, eps=1e-12):
    """(weight_orig / sigma, u, v): one power iteration first in train mode, u and v constant for autograd."""
    wm = w_orig.reshape(w_orig.shape[0], -1)
    if train:
        with torch.no_grad():
            v = F.normalize(torch.mv(wm.t(), u), dim=0, eps=eps)
            u = F.normalize(torch.mv(wm, v), dim=0, eps=eps)
    sigma = torch.dot(u, torch.mv(wm, v))
    return w_orig / sigma, u, v


class _LeakyWithSlopes(torch.autograd.Function):
    """LeakyReLU(0.2) whose backward takes its slope from ``positive`` (1 where True, else 0.2) instead of the sign of
    its own input."""

    @staticmethod
    def forward(ctx, z, positive):
        ctx.save_for_backward(positive)
        return F.leaky_relu(z, 0.2)

    @staticmethod
    def backward(ctx, g):
        (positive,) = ctx.saved_tensors
        return g * torch.where(positive, 1.0, 0.2).to(g.dtype), None


def forward(params, xs, train=True, use_sigmoid=False, use_spectral_norm=True, slopes=None):
    """Discriminator forward of xs (B, T, C, H, W) with state-dict tensors ``params``.  In train mode the updated
    ``weight_u`` / ``weight_v`` are written back into ``params`` (detached), as the reference's hooks do.

    ``slopes``: optional list of five bool tensors (B, C, T, H, W), where the LeakyReLU after conv i counts as positive
    in the backward.  A pre-activation within rounding of 0 can change sign between an fp32 implementation and this
    one; passing that implementation's signs makes the two backward passes take the same slopes."""
    x = xs.transpose(1, 2)
    for i in range(6):
        p = f"conv.{2 * i}."
        if use_spectral_norm and i < 5:
            w, u, v = sn_weight(params[p + "weight_orig"], params[p + "weight_u"], params[p + "weight_v"], train)
            params[p + "weight_u"], params[p + "weight_v"] = u.detach(), v.detach()
            b = None
        else:
            w, b = params[p + "weight"], params[p + "bias"]
        x = F.conv3d(x, w, b, stride=(1, 2, 2), padding=1 if i == 0 else (1, 2, 2))
        if i < 5:
            x = F.leaky_relu(x, 0.2) if slopes is None else _LeakyWithSlopes.apply(x, slopes[i])
    if use_sigmoid:
        x = torch.sigmoid(x)
    return x.transpose(1, 2)


def hinge(out, is_real, is_disc):
    """core/loss.py's hinge AdversarialLoss."""
    if not is_disc:
        return (-out).mean()
    return torch.relu(1 + (-out if is_real else out)).mean()
