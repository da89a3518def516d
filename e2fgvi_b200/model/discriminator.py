"""Temporal PatchGAN discriminator (reference: model/e2fgvi.py:271-344, identical in e2fgvi_hq.py), trainable.

Six Conv3d layers, kernel (3, 5, 5), stride (1, 2, 2), channels in -> 32 -> 64 -> 128 -> 128 -> 128 -> 128, padding 1
for the first and (1, 2, 2) for the others, LeakyReLU(0.2) between them.  With spectral norm (the default) the first five
convs carry ``weight_orig`` / ``weight_u`` / ``weight_v`` and no bias, as the reference's ``spectral_norm`` hooks leave
them, so reference checkpoints load with ``strict=True``.

Every conv runs on the library's sm_90a kernels, forward and backward (``ops.dis_conv3d``, ``dis_conv3d_dgrad``,
``dis_conv3d_wgrad``).  The spectral norm's power iteration and ``weight_orig / sigma`` are a few mat-vecs and stay in
torch, so autograd takes the weight gradient on from the normalised weight to ``weight_orig``.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .generator import BaseNetwork

_CHANNELS = (32, 64, 128, 128, 128, 128)


class _DisConv(torch.autograd.Function):
    """One conv (+ LeakyReLU(0.2) when ``leaky``) on NDHWC activations.

    ``x`` is the fp32 activation and (x_hi, x_lo) its bf16 split, the operand the kernels read.  Outputs: the fp32
    result and its split.  The gradient a layer returns for its input already includes the derivative of the
    LeakyReLU that produced that input (``dact``): it is fused into the input-gradient kernel's epilogue, so the
    preceding layer's backward receives the gradient of its conv output directly.  The LeakyReLU keeps the sign of its
    input, so the saved output decides the derivative.
    """

    @staticmethod
    def forward(ctx, x, weight, bias, x_hi, x_lo, pad, leaky, dact):
        w_hi, w_lo = ops.dis_pack_weight(weight, x_hi.shape[-1])
        out, hi, lo = ops.dis_conv3d(x_hi, x_lo, w_hi, w_lo, None if bias is None else bias.detach().float().contiguous(),
                                     weight.shape[0], pad, leaky)
        ctx.save_for_backward(weight, x_hi, x_lo)
        ctx.pad, ctx.dact, ctx.has_bias = pad, dact, bias is not None
        ctx.mark_non_differentiable(hi, lo)
        return out, hi, lo

    @staticmethod
    def backward(ctx, g, _g_hi, _g_lo):
        weight, x_hi, x_lo = ctx.saved_tensors
        g = g.contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            # the layer above wrote the split of g along with g; a gradient autograd summed or copied has none
            g_hi, g_lo = getattr(g, "_e2f_split", None) or ops.split_bf16(g)
            b, t, h, w, cs = x_hi.shape
            wt_hi, wt_lo = ops.dis_pack_weight_t(weight, ctx.pad, cs)
            dx, dx_hi, dx_lo = ops.dis_conv3d_dgrad(g_hi, g_lo, wt_hi, wt_lo, x_hi if ctx.dact else None, h, w, cs,
                                                    ctx.pad, split=ctx.dact)
            if ctx.dact:
                dx._e2f_split = (dx_hi, dx_lo)
        want_db = ctx.has_bias and ctx.needs_input_grad[2]
        if ctx.needs_input_grad[1] or want_db:
            dw, db = ops.dis_conv3d_wgrad(g, x_hi, x_lo, weight.shape[1], ctx.pad, want_db)
            if not ctx.needs_input_grad[1]:
                dw = None
        return dx, dw, db, None, None, None, None, None


class _SNConv3d(nn.Module):
    """A bias-free Conv3d under the reference's spectral norm (model/modules/spectral_norm.py:40-96): parameters and
    buffers ``weight_orig``, ``weight_u``, ``weight_v``; one power iteration per call in training mode."""

    def __init__(self, cin, cout, eps=1e-12):
        super().__init__()
        self.eps = eps
        self.weight_orig = nn.Parameter(torch.empty(cout, cin, 3, 5, 5))
        nn.init.kaiming_uniform_(self.weight_orig, a=math.sqrt(5))        # nn.Conv3d's default
        self.register_buffer("weight_u", F.normalize(torch.randn(cout), dim=0, eps=eps))
        self.register_buffer("weight_v", F.normalize(torch.randn(cin * 75), dim=0, eps=eps))
        self.bias = None
        # plain attribute, as the reference's hook leaves it: aliases weight_orig until the first forward, then the
        # last normalised weight
        self.weight = self.weight_orig.data

    def normalized_weight(self):
        w_mat = self.weight_orig.reshape(self.weight_orig.shape[0], -1)
        u, v = self.weight_u, self.weight_v
        if self.training:
            with torch.no_grad():
                v = F.normalize(torch.mv(w_mat.t(), u), dim=0, eps=self.eps, out=v)
                u = F.normalize(torch.mv(w_mat, v), dim=0, eps=self.eps, out=u)
                u, v = u.clone(), v.clone()      # the buffers change again in the next call; autograd keeps these
        sigma = torch.dot(u, torch.mv(w_mat, v))
        self.weight = self.weight_orig / sigma
        return self.weight


class Discriminator(BaseNetwork):
    """Drop-in for the reference's ``Discriminator``: same constructor, state dict and forward.

    ``forward(xs)``: xs (B, T, C, H, W) fp32 on the GPU -> (B, T, 128, H', W'), sigmoid-ed if ``use_sigmoid``.
    Differentiable with respect to ``xs`` and every parameter; an input that does not require a gradient costs no
    first-layer input-gradient kernel, and parameters that do not require one cost no weight-gradient kernels.
    ``init_weights(init_type='normal', gain=0.02)`` and ``print_network()`` come from BaseNetwork; under spectral
    norm ``weight`` aliases ``weight_orig`` at construction, as the reference's hook leaves it, so the init reaches
    ``weight_orig``.  The ``nn.LeakyReLU`` entries of ``conv`` keep the reference's indices; the activations run
    fused into the conv kernels, so those modules are never called."""

    _graphs = None                                  # BaseNetwork.load_state_dict: no captured graphs here

    def __init__(self, in_channels=3, use_sigmoid=False, use_spectral_norm=True, init_weights=True):
        super().__init__()
        self.use_sigmoid = use_sigmoid
        self.use_spectral_norm = use_spectral_norm
        layers = []
        cin = in_channels
        for i, cout in enumerate(_CHANNELS):
            if i < 5 and use_spectral_norm:
                layers.append(_SNConv3d(cin, cout))
            else:
                layers.append(nn.Conv3d(cin, cout, (3, 5, 5), (1, 2, 2), padding=1 if i == 0 else (1, 2, 2)))
            if i < 5:
                layers.append(nn.LeakyReLU(0.2, inplace=True))
            cin = cout
        self.conv = nn.Sequential(*layers)
        if init_weights:
            self.init_weights()

    def _convs(self):
        return [self.conv[2 * i] for i in range(len(_CHANNELS))]

    def forward(self, xs):
        if not xs.is_cuda:
            raise RuntimeError("Discriminator runs on the e2fgvi_b200 CUDA kernels; move it and its input to the GPU")
        c = xs.shape[2]
        x = xs.float().permute(0, 1, 3, 4, 2)
        cs = -(-c // 8) * 8                         # the kernels read channels in multiples of 8
        x = F.pad(x, (0, cs - c)).contiguous()
        x_hi, x_lo = ops.split_bf16(x.detach())
        for i, m in enumerate(self._convs()):
            w = m.normalized_weight() if isinstance(m, _SNConv3d) else m.weight
            x, x_hi, x_lo = _DisConv.apply(x, w, m.bias, x_hi, x_lo, 1 if i == 0 else 2, i < 5, i > 0)
        if self.use_sigmoid:
            x = torch.sigmoid(x)
        return x.permute(0, 1, 4, 2, 3)
