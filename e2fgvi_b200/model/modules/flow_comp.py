"""Flow completion on the hot path: SPyNet, ``flow_warp`` and ``FlowCompletionLoss`` (reference:
model/modules/flow_comp.py:11-226,345-383).

``SPyNet.bidirect_flows`` has a backward pass (gradients into SPyNet's parameters, not into the frames): it is what
``InpaintGenerator.forward_bidirect_flow`` runs when gradients are needed.

State-dict layout (must stay byte-compatible with released checkpoints, SURVEY §8(b)):
``basic_module.{0..5}.basic_module.{0..4}.conv.{weight,bias}`` + buffers ``mean``/``std`` [1,3,1,1].
The ``.conv.`` level exists in the reference because it wraps each conv in ``mmcv.cnn.ConvModule``
(flow_comp.py:181-215); here a tiny holder module provides the same key path with no mmcv dependency.
The constructor never touches the network (the reference downloads pretrained weights, flow_comp.py:59-72;
E2FGVI checkpoints carry ``update_spynet.*`` anyway).
"""
import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops

# (cin, cout) of the five 7x7 convs of one pyramid level, ReLU after all but the last (flow_comp.py:181-215)
_LEVEL_CONVS = ((8, 32), (32, 64), (64, 32), (32, 16), (16, 2))
_NUM_LEVELS = 6


def flow_warp(x, flow, interpolation="bilinear", padding_mode="zeros", align_corners=True):
    """Same signature and error behaviour as the reference ``flow_warp`` (flow_comp.py:345-383); CUDA kernel."""
    return ops.flow_warp(x, flow, interpolation, padding_mode, align_corners)


class _ConvHolder(nn.Module):
    """Gives a conv the ``<idx>.conv.{weight,bias}`` key path of mmcv's ConvModule."""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size=7, stride=1, padding=3)


class SPyNetBasicModule(nn.Module):
    """One pyramid level: 5 x (7x7 conv), ReLU between (flow_comp.py:172-226)."""

    def __init__(self):
        super().__init__()
        self.basic_module = nn.Sequential(*[_ConvHolder(ci, co) for ci, co in _LEVEL_CONVS])

    def forward(self, tensor_input):
        """Five 7x7 convs on the wgmma implicit-GEMM kernel, ReLU fused (LeakyReLU with slope 0), the bf16 split
        operand handed from conv to conv.  Activations with <= 32 channels (the 8-channel input, the 32- and
        16-channel intermediates) travel in the row-gapped layout so their convs use window-packed K: 7 / 28 / 14 K
        chunks per tile instead of 49 taps zero-padded to 64 channels."""
        convs = [holder.conv for holder in self.basic_module]
        y = ops.pack_rows(tensor_input, lead=convs[0].padding[0])
        last = len(convs) - 1
        for i, conv in enumerate(convs):
            if i == last:
                return ops.conv3x3(y, conv.weight, conv.bias, negative_slope=1.0, out="f32")
            nxt = convs[i + 1]
            if ops.rows_channels(nxt.in_channels) == nxt.in_channels:      # 8 / 16 / 32 channels: row-gapped hand-off
                y = ops.conv3x3(y, conv.weight, conv.bias, negative_slope=0.0, out="rows", out_lead=nxt.padding[0])
            else:
                y = ops.conv3x3(y, conv.weight, conv.bias, negative_slope=0.0, out="split")


def _basic_module_rows(module, rows, residual, keep=None):
    """SPyNetBasicModule on a ready row-gapped operand; the last conv adds ``residual`` = flow_up (flow_comp.py:127:
    ``flow = flow_up + basic_module(...)``) in its epilogue and returns the new flow (P, hk, wk, 2) fp32.  ``keep`` (a
    list or None) receives the five convs' input operands, the ReLU outputs the backward pass needs."""
    convs = [holder.conv for holder in module.basic_module]
    y = rows
    last = len(convs) - 1
    if keep is not None:
        keep.append(y)
    if ops.KXN_CONVS:
        # 8 -> 32 and 32 -> 64 on the window-packed kernel (wide enough outputs), then 64 -> 32, 32 -> 16 and 16 -> 2 on
        # the kx-in-N kernel: with <= 32 output channels the plain implicit GEMM re-reads its A tile for every tap
        y = ops.conv3x3(y, convs[0].weight, convs[0].bias, negative_slope=0.0, out="rows", out_lead=convs[1].padding[0])
        if keep is not None:
            keep.append(y)
        y = ops.conv3x3(y, convs[1].weight, convs[1].bias, negative_slope=0.0, out="split")
        if keep is not None:
            keep.append(y)
        y = ops.conv_kxn(y, convs[2].weight, convs[2].bias, negative_slope=0.0, out="split")
        if keep is not None:
            keep.append(y)
        y = ops.conv_kxn(y, convs[3].weight, convs[3].bias, negative_slope=0.0, out="split")
        if keep is not None:
            keep.append(y)
        out = ops.conv_kxn(y, convs[4].weight, convs[4].bias, residual=residual.permute(0, 3, 1, 2))
        return out.permute(0, 2, 3, 1)                         # NHWC storage: a view, (P, hk, wk, 2) contiguous
    for i, conv in enumerate(convs):
        if i == last:
            out = ops.conv3x3(y, conv.weight, conv.bias, negative_slope=1.0, out="f32", residual=residual.permute(0, 3, 1, 2))
            return out.permute(0, 2, 3, 1)                     # NHWC storage: a view, (P, hk, wk, 2) contiguous
        nxt = convs[i + 1]
        if ops.rows_channels(nxt.in_channels) == nxt.in_channels:
            y = ops.conv3x3(y, conv.weight, conv.bias, negative_slope=0.0, out="rows", out_lead=nxt.padding[0])
        else:
            y = ops.conv3x3(y, conv.weight, conv.bias, negative_slope=0.0, out="split")
        if keep is not None:
            keep.append(y)


# Layout of each input gradient that the next (shallower) input gradient reads as its dy: row-gapped (window-packed K)
# for <= 32 channels, dense for the 64-channel one.
_DGRAD_OUT = {4: "rows", 3: "rows", 2: "split", 1: "rows"}


def _level_backward(module, keep, dflow, need, conv_lo, want_input):
    """Backward of one pyramid level, conv 5 down to conv 1.  dflow (P, hk, wk, 2): gradient of the level's output flow
    (also the residual's); keep: the forward's operands; need[i] = (weight, bias) needs grad for conv i.  Input
    gradients run down to conv ``conv_lo``; ``want_input`` also returns the gradient of the level's 8-channel input.
    Returns ({(i, 'weight' | 'bias'): grad}, d_in or None)."""
    convs = [holder.conv for holder in module.basic_module]
    grads = {}
    dy32 = dflow
    dy = ops.pack_rows(dflow.permute(0, 3, 1, 2), lead=3, cin=8)      # 8: a stride-1 row-gapped operand needs >= 8 channels
    for i in range(4, -1, -1):
        nw, nb = need[i]
        if nw or nb:
            dw, db = ops.conv2d_wgrad(dy32, keep[i], convs[i].in_channels, with_bias=nb)
            if nw:
                grads[(i, "weight")] = dw
            if nb:
                grads[(i, "bias")] = db
        if i > conv_lo:
            dy32, dy = ops.conv2d_dgrad(dy, convs[i].weight, act=keep[i], out=_DGRAD_OUT[i])
        elif i == 0 and want_input:
            d_in, _ = ops.conv2d_dgrad(dy, convs[0].weight)
            return grads, d_in
        else:
            break
    return grads, None


class _BidirectFlows(torch.autograd.Function):
    """``SPyNet.bidirect_flows`` with a backward pass into SPyNet's 60 parameters.  The forward is the inference
    sequence (the same kernels and operands), keeping the operands for the backward; the backward walks the levels from
    fine to coarse and stops below the coarsest level with a parameter that needs a gradient.  The parameters are saved
    with ``save_for_backward``, so that changing one in place between forward and backward (an ``optimizer.step()``)
    raises autograd's usual error instead of giving the gradient of the new weights.  The backward frees the kept
    operands: a second backward (``retain_graph=True``) raises."""

    @staticmethod
    def forward(ctx, spynet, frames, num_local_frames, unit, *params):
        levels = []
        fwd, bwd = spynet._bidirect_flows(frames, num_local_frames, unit, levels)
        ctx.spynet, ctx.levels = spynet, levels
        ctx.save_for_backward(*params)
        return fwd, bwd

    @staticmethod
    def backward(ctx, d_forward, d_backward):
        spynet, levels = ctx.spynet, ctx.levels
        if levels is None:
            raise RuntimeError("SPyNet.bidirect_flows: the backward frees the operands it keeps, so the flows cannot be "
                               "backpropagated a second time (retain_graph=True is not supported); run the forward again")
        ctx.saved_tensors                       # raises if a parameter was modified in place since the forward
        needs = ctx.needs_input_grad[4:]
        n_conv = len(_LEVEL_CONVS)
        need = [[(needs[2 * (lv * n_conv + i)], needs[2 * (lv * n_conv + i) + 1]) for i in range(n_conv)]
                for lv in range(_NUM_LEVELS)]
        active = [lv for lv in range(_NUM_LEVELS) if any(a or b for a, b in need[lv])]
        grads = [None] * (2 * _NUM_LEVELS * n_conv)
        if not active:
            return (None, None, None, None) + tuple(grads)
        lowest = active[0]
        pyr = levels[0][0]
        dflow = ops.spynet_final_backward(d_forward, d_backward, pyr)
        for lv in range(_NUM_LEVELS - 1, lowest - 1, -1):
            _, keep, flow_up = levels[lv]
            if lv > lowest:
                conv_lo, want_input = 0, True
            else:
                conv_lo, want_input = min(i for i in range(n_conv) if any(need[lv][i])), False
            g, d_in = _level_backward(spynet.basic_module[lv], keep, dflow, need[lv], conv_lo, want_input)
            for (i, kind), v in g.items():
                grads[2 * (lv * n_conv + i) + (kind == "bias")] = v
            if want_input:
                dflow = ops.spynet_level_input_backward(d_in, dflow, pyr, _NUM_LEVELS - 1 - lv, flow_up)
        ctx.levels = None
        return (None, None, None, None) + tuple(grads)


class SPyNet(nn.Module):
    """6-level coarse-to-fine flow estimator (flow_comp.py:49-169). ``forward(ref, supp) -> flow (n,2,h,w)``."""

    def __init__(self, use_pretrain=False, pretrained=None):
        super().__init__()
        del use_pretrain, pretrained  # accepted for signature compatibility; never fetched
        self.basic_module = nn.ModuleList([SPyNetBasicModule() for _ in range(_NUM_LEVELS)])
        self.register_buffer("mean", torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
        self.register_buffer("std", torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))

    def compute_flow(self, ref, supp):
        """ref/supp (n,3,h,w) with h,w multiples of 32 (flow_comp.py:84-134)."""
        n, _, h, w = ref.shape
        pyr_ref = [(ref - self.mean) / self.std]
        pyr_supp = [(supp - self.mean) / self.std]
        for _ in range(_NUM_LEVELS - 1):
            pyr_ref.append(F.avg_pool2d(pyr_ref[-1], kernel_size=2, stride=2, count_include_pad=False))
            pyr_supp.append(F.avg_pool2d(pyr_supp[-1], kernel_size=2, stride=2, count_include_pad=False))
        flow = ref.new_zeros(n, 2, h >> (_NUM_LEVELS - 1), w >> (_NUM_LEVELS - 1))
        for level in range(_NUM_LEVELS):
            r, s = pyr_ref[_NUM_LEVELS - 1 - level], pyr_supp[_NUM_LEVELS - 1 - level]
            if level == 0:
                flow_up = flow
            else:
                flow_up = F.interpolate(flow, scale_factor=2, mode="bilinear", align_corners=True) * 2.0
            warped = flow_warp(s, flow_up.permute(0, 2, 3, 1), padding_mode="border")
            flow = flow_up + self.basic_module[level](torch.cat([r, warped, flow_up], 1))
        return flow

    def bidirect_flows(self, masked_frames, num_local_frames, unit=False):
        """Both flow directions of ``InpaintGenerator.forward_bidirect_flow`` (e2fgvi.py:210-234) straight from the
        masked frames (b,t,3,H,W) in [-1,1] (in [0, 1] with ``unit``): 1 pyramid launch, per level 1 input launch + five
        7x7 convs, 1 final launch.  Returns (flows_forward, flows_backward), each (b, l_t-1, 2, H/4, W/4).

        With grad mode on and some SPyNet parameter requiring grad, the flows carry a ``grad_fn`` whose backward gives
        those parameters their gradients (not the frames': frames that require grad raise ``ValueError``)."""
        params = self._flow_params()
        if torch.is_grad_enabled() and any(p.requires_grad for p in params):
            if masked_frames.requires_grad:
                raise ValueError("SPyNet.bidirect_flows: the gradient with respect to the frames is not implemented "
                                 "(detach them; the flows' gradient reaches SPyNet's parameters)")
            return _BidirectFlows.apply(self, masked_frames, num_local_frames, unit, *params)
        return self._bidirect_flows(masked_frames, num_local_frames, unit)

    def _flow_params(self):
        return [t for level in self.basic_module for holder in level.basic_module for t in (holder.conv.weight, holder.conv.bias)]

    def _bidirect_flows(self, masked_frames, num_local_frames, unit=False, keep=None):
        """The launch sequence of ``bidirect_flows``; ``keep`` (a list or None) receives per level (pyramid, the five
        convs' input operands, flow_up)."""
        pyr = ops.spynet_pyramid(masked_frames, num_local_frames, self.mean, self.std, unit=unit)
        flow = None
        for level in range(_NUM_LEVELS):
            rows, flow_up = ops.spynet_level_input(pyr, _NUM_LEVELS - 1 - level, flow,
                                                   lead=self.basic_module[level].basic_module[0].conv.padding[0])
            ops_kept = [] if keep is not None else None
            flow = _basic_module_rows(self.basic_module[level], rows, flow_up, ops_kept)
            if keep is not None:
                keep.append((pyr, ops_kept, flow_up))
        return ops.spynet_final(flow, pyr)

    def forward(self, ref, supp):
        h, w = ref.shape[2:4]
        w_up = w if w % 32 == 0 else 32 * (w // 32 + 1)
        h_up = h if h % 32 == 0 else 32 * (h // 32 + 1)
        ref = F.interpolate(ref, size=(h_up, w_up), mode="bilinear", align_corners=False)
        supp = F.interpolate(supp, size=(h_up, w_up), mode="bilinear", align_corners=False)
        flow = F.interpolate(self.compute_flow(ref, supp), size=(h, w), mode="bilinear", align_corners=False)
        # rescale u by w/w_up and v by h/h_up (flow_comp.py:164-167)
        return torch.stack((flow[:, 0] * (float(w) / float(w_up)), flow[:, 1] * (float(h) / float(h_up))), dim=1)


def _load_spynet_weights(module, pretrained):
    """mmcv ``load_checkpoint(module, pretrained, strict=True)`` for a local file or a state dict: the ``state_dict``
    entry if there is one, ``module.`` prefixes stripped.  Never touches the network."""
    if isinstance(pretrained, str):
        if "://" in pretrained:
            raise ValueError(f"FlowCompletionLoss: pretrained={pretrained!r} is a URL; pass a local path or a state dict")
        ckpt = torch.load(pretrained, map_location="cpu", weights_only=True)
    elif isinstance(pretrained, dict):
        ckpt = pretrained
    else:
        raise TypeError(f"FlowCompletionLoss: pretrained must be a path, a state dict or None, got {type(pretrained)}")
    sd = ckpt["state_dict"] if "state_dict" in ckpt else ckpt
    sd = {(k[7:] if k.startswith("module.") else k): v for k, v in sd.items()}
    module.load_state_dict(sd, strict=True)


class FlowCompletionLoss(nn.Module):
    """Flow completion loss (flow_comp.py:11-46): L1 between the predicted flows and those of a frozen SPyNet
    (``fix_spynet``) on the ground-truth frames, per direction, summed.

    ``loss(pred_flows, gt_local_frames)``: pred_flows = (forward, backward), each (b, l_t-1, 2, h/4, w/4);
    gt_local_frames (b, l_t, 3, h, w) in [0, 1].  The ground-truth flows run under ``no_grad`` on the fused path.
    ``pretrained``: SPyNet weights as a local path or a state dict, loaded as mmcv's ``load_checkpoint`` does (the
    reference downloads them); without it the ground-truth flows come from an untrained network (a warning says so)."""

    def __init__(self, pretrained=None):
        super().__init__()
        self.fix_spynet = SPyNet()
        if pretrained is None:
            warnings.warn("FlowCompletionLoss: no SPyNet weights given (pretrained=None): the ground-truth flows come from "
                          "an untrained network", RuntimeWarning, stacklevel=2)
        else:
            _load_spynet_weights(self.fix_spynet, pretrained)
        for p in self.fix_spynet.parameters():
            p.requires_grad = False
        self.l1_criterion = nn.L1Loss()

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        ops.invalidate_weight_caches()
        return out

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        ops.invalidate_weight_caches()
        return out

    def forward(self, pred_flows, gt_local_frames):
        b, l_t, c, h, w = gt_local_frames.size()
        with torch.no_grad():
            gt_flows_forward, gt_flows_backward = self.fix_spynet.bidirect_flows(gt_local_frames, l_t, unit=True)
        forward_flow_loss = self.l1_criterion(pred_flows[0].view(-1, 2, h // 4, w // 4),
                                              gt_flows_forward.view(-1, 2, h // 4, w // 4))
        backward_flow_loss = self.l1_criterion(pred_flows[1].view(-1, 2, h // 4, w // 4),
                                               gt_flows_backward.view(-1, 2, h // 4, w // 4))
        return forward_flow_loss + backward_flow_loss
