"""Flow-guided feature propagation (reference: model/modules/feat_prop.py:13-149).

``SecondOrderDeformableAlignment`` keeps the reference's parameter names (``weight``, ``bias``,
``conv_offset.{0,2,4,6}``) and attributes (stride/padding/dilation/groups/deform_groups) but its DCN is the
fused sm_90a kernel (``ops.deform_align_fused``): 10*tanh + flow add + sigmoid + bilinear sampling + im2col +
wgmma GEMM + bias in one launch, no column buffer.  ``BidirectionalPropagation`` restates the recurrence,
including the two reference quirks that trained weights depend on (SURVEY §7): the flow index is ``i-1`` for BOTH
sweep directions (feat_prop.py:94-103) and the caller passes (forward, backward) flows into
(flows_backward, flows_forward) (e2fgvi.py:249-250).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from .flow_comp import flow_warp


class SecondOrderDeformableAlignment(nn.Module):
    """Second-order deformable alignment: offset head (4 convs) + modulated deformable 3x3 conv, 16 groups."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, dilation=1, groups=1,
                 deform_groups=16, max_residue_magnitude=10):
        super().__init__()
        if kernel_size != 3:
            raise ValueError("E2FGVI uses a 3x3 deformable kernel")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = (3, 3)
        self.stride, self.padding, self.dilation = (stride,) * 2, (padding,) * 2, (dilation,) * 2
        self.groups, self.deform_groups = groups, deform_groups
        self.max_residue_magnitude = max_residue_magnitude
        # same init family as mmcv's ModulatedDeformConv2d (uniform +-1/sqrt(fan_in), zero bias)
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, 3, 3))
        self.bias = nn.Parameter(torch.zeros(out_channels))
        bound = 1.0 / math.sqrt(in_channels * 9)
        nn.init.uniform_(self.weight, -bound, bound)
        co = out_channels
        self.conv_offset = nn.Sequential(
            nn.Conv2d(3 * co + 4, co, 3, 1, 1), nn.LeakyReLU(0.1, inplace=True),
            nn.Conv2d(co, co, 3, 1, 1), nn.LeakyReLU(0.1, inplace=True),
            nn.Conv2d(co, co, 3, 1, 1), nn.LeakyReLU(0.1, inplace=True),
            nn.Conv2d(co, 27 * deform_groups, 3, 1, 1))
        self.fused = True  # False: torch epilogue + ops.modulated_deform_conv2d (the reference's operator split)
        self.init_offset()

    def packed_weight(self):
        """fp16 [Cout, 9*Cin] operand of the DCN GEMM, re-packed whenever the parameter changes or moves."""
        # ops.pack_dcn_weight is looked up when the operand is built, so a replacement of it takes effect
        return ops._derived_one(self.weight, ("dcn", self.deform_groups), lambda w, g: ops.pack_dcn_weight(w, g),
                                self.deform_groups)

    def init_offset(self):
        """Zero the last offset conv (feat_prop.py:32-33)."""
        nn.init.zeros_(self.conv_offset[-1].weight)
        nn.init.zeros_(self.conv_offset[-1].bias)

    def offset_head(self, cond_sources, flow_1, flow_2):
        """conv_offset on cat[cond..., flow_1, flow_2] (feat_prop.py:36-37) without building the cat: each tensor is
        one TMA source of the first conv; LeakyReLU(0.1) is fused into the conv epilogues.  Returns the raw
        27*dg-channel head, fp32, channels_last."""
        co = self.conv_offset
        flows = torch.cat([flow_1, flow_2], dim=1)
        y = ops.conv3x3(list(cond_sources) + [flows], co[0].weight, co[0].bias, negative_slope=0.1, out="split")
        y = ops.conv3x3([y], co[2].weight, co[2].bias, negative_slope=0.1, out="split")
        y = ops.conv3x3([y], co[4].weight, co[4].bias, negative_slope=0.1, out="split")
        return ops.conv3x3([y], co[6].weight, co[6].bias)

    def offset_head_frames(self, cond_sources, flows):
        """``offset_head`` for sources that may be frame slices of (b,t,h,w,c) buffers (``ops.conv_frames``)."""
        co = self.conv_offset
        y = ops.conv_frames(list(cond_sources) + [flows], co[0].weight, co[0].bias, negative_slope=0.1, out="split")
        y = ops.conv_frames([y], co[2].weight, co[2].bias, negative_slope=0.1, out="split")
        y = ops.conv_frames([y], co[4].weight, co[4].bias, negative_slope=0.1, out="split")
        return ops.conv_frames([y], co[6].weight, co[6].bias)

    def align_split(self, x, cond_sources, flow_1, flow_2, flows):
        """Fused alignment returning ``(fp32 tensor, SplitNHWC)``: the DCN epilogue also writes the bf16 operand pair of
        the backbone conv that follows (feat_prop.py:131-136)."""
        head = self.offset_head_frames(cond_sources, flows)
        return ops.deform_align_fused(x, head, flow_1, flow_2, self.packed_weight(), self.bias, self.deform_groups,
                                      self.max_residue_magnitude, out_split=True)

    def align(self, x, cond_sources, flow_1, flow_2):
        head = self.offset_head(cond_sources, flow_1, flow_2)
        if self.fused:
            return ops.deform_align_fused(x, head, flow_1, flow_2, self.packed_weight(), self.bias, self.deform_groups,
                                          self.max_residue_magnitude)
        # operator-level path, identical maths to feat_prop.py:41-58
        o1, o2, mask = torch.chunk(head, 3, dim=1)
        offset = self.max_residue_magnitude * torch.tanh(torch.cat((o1, o2), dim=1))
        off1, off2 = torch.chunk(offset, 2, dim=1)
        off1 = off1 + flow_1.flip(1).repeat(1, off1.size(1) // 2, 1, 1)
        off2 = off2 + flow_2.flip(1).repeat(1, off2.size(1) // 2, 1, 1)
        return ops.modulated_deform_conv2d(x, torch.cat([off1, off2], dim=1), torch.sigmoid(mask), self.weight,
                                           self.bias, self.stride, self.padding, self.dilation, self.groups,
                                           self.deform_groups)

    def forward(self, x, extra_feat, flow_1, flow_2):
        """Reference boundary (feat_prop.py:35): extra_feat is the already concatenated condition tensor."""
        return self.align(x, [extra_feat], flow_1, flow_2)


class BidirectionalPropagation(nn.Module):
    """Backward then forward recurrent sweep with second-order alignment, 1x1 fusion and residual."""

    DIRECTIONS = ("backward_", "forward_")

    def __init__(self, channel):
        super().__init__()
        self.channel = channel
        self.deform_align = nn.ModuleDict()
        self.backbone = nn.ModuleDict()
        for i, name in enumerate(self.DIRECTIONS):
            self.deform_align[name] = SecondOrderDeformableAlignment(2 * channel, channel, 3, padding=1,
                                                                    deform_groups=16)
            self.backbone[name] = nn.Sequential(
                nn.Conv2d((2 + i) * channel, channel, 3, 1, 1), nn.LeakyReLU(0.1, inplace=True),
                nn.Conv2d(channel, channel, 3, 1, 1))
        self.fusion = nn.Conv2d(2 * channel, channel, 1, 1, 0)
        # False: forward() runs the operator-by-operator sequence of feat_prop.py:106-126, as it does for channel counts
        # that are not a multiple of 16
        self.fused_prologue = True

    def propagate_frames(self, x32, x_hi, x_lo, flows_backward, flows_forward, into=None):
        """The fast path: every per-frame tensor is a FRAME SLICE of a (b,t,h,w,c) buffer, read and written in place.

        x32 / x_hi / x_lo: (b,t,h,w,c) fp32 features and their bf16 (hi, lo) split (dense inner (h,w,c); the t axis may
        be a prefix slice of a longer buffer).  ``into`` = (o32, ohi, olo) buffers of the same shape that receive the
        fused result frame by frame — passing the inputs themselves updates them IN PLACE (each pixel's residual is
        read by the thread that overwrites it; the sweeps are complete before the first fusion launch).  No
        ``x[:, i].contiguous()`` gathers, no per-step split passes, no token-buffer copies, no stack / cat:
        per step = prologue, 4 offset-head convs, DCN (+ split epilogue), 2 backbone convs."""
        b, t, h, w, c = x32.shape
        cur = [ops.SplitNHWC(x_hi[:, i], x_lo[:, i], (b, c, h, w)) for i in range(t)]
        zero = torch.zeros((b, h, w, c), dtype=x_hi.dtype, device=x32.device)
        zero_sp = ops.SplitNHWC(zero, zero, (b, c, h, w))
        # per-direction results live in (t, b, h, w, c) buffers: frame idx is the dense slice buf[idx], and for a single
        # clip (b == 1) all frames are one contiguous batch, so the 1x1 fusion runs as ONE launch instead of t
        bufs = {}
        for name in self.DIRECTIONS:
            bufs[name] = (torch.empty((t, b, h, w, c), dtype=torch.float32, device=x32.device),
                          torch.empty((t, b, h, w, c), dtype=x_hi.dtype, device=x32.device),
                          torch.empty((t, b, h, w, c), dtype=x_lo.dtype, device=x32.device))
        swept_sp = {}
        for name in self.DIRECTIONS:
            backward = name == "backward_"
            order = list(range(t - 1, -1, -1)) if backward else list(range(t))
            flows = flows_backward if backward else flows_forward
            align, backbone = self.deform_align[name], self.backbone[name]
            r32, rhi, rlo = bufs[name]
            hist32 = []
            for i, idx in enumerate(order):
                prop32, prop_sp = None, zero_sp
                if i > 0:
                    xg, cond_n1, cond_n2, flows_op, flow_n1, flow_n2 = ops.prop_prologue(
                        hist32[-1], hist32[-2] if i > 1 else None, flows[:, i - 1], flows[:, i - 2] if i > 1 else None)
                    prop32, prop_sp = align.align_split(xg, [cond_n1, cur[idx], cond_n2], flow_n1, flow_n2, flows_op)
                parts = [cur[idx], prop_sp] if backward else [cur[idx], swept_sp["backward_"][idx], prop_sp]
                y = ops.conv_frames(parts, backbone[0].weight, backbone[0].bias, negative_slope=0.1, out="split")
                new32, _ = ops.conv_frames([y], backbone[2].weight, backbone[2].bias, residual=prop32, out="both",
                                           into=(r32[idx], rhi[idx], rlo[idx]))
                hist32.append(new32)
            swept_sp[name] = [ops.SplitNHWC(rhi[i], rlo[i], (b, c, h, w)) for i in range(t)]
        if into is None:
            into = (torch.empty_like(x32), torch.empty_like(x_hi), torch.empty_like(x_lo))
        o32, ohi, olo = into
        # 1x1 fusion conv over cat(backward, forward) as two sources, "+ x" fused (feat_prop.py:143-149)
        if b == 1:
            srcs = [ops.SplitNHWC(bufs[n_][1].view(t, h, w, c), bufs[n_][2].view(t, h, w, c), (t, c, h, w)) for n_ in self.DIRECTIONS]
            ops.conv_frames(srcs, self.fusion.weight, self.fusion.bias, residual=x32[0].permute(0, 3, 1, 2), out="both",
                            into=(o32[0], ohi[0], olo[0]))
        else:
            for i in range(t):
                ops.conv_frames([swept_sp["backward_"][i], swept_sp["forward_"][i]], self.fusion.weight, self.fusion.bias,
                                residual=x32[:, i].permute(0, 3, 1, 2), out="both", into=(o32[:, i], ohi[:, i], olo[:, i]))
        return o32, ohi, olo

    def forward(self, x, flows_backward, flows_forward):
        """x (b,t,c,h,w); flows_* (b,t-1,2,h,w) -> (b,t,c,h,w)."""
        b, t, c, h, w = x.shape
        if self.fused_prologue and c % 16 == 0:
            x32 = x.permute(0, 1, 3, 4, 2).contiguous().float()          # no-op for (b,t,h,w,c) storage
            x_hi, x_lo = ops.split_bf16(x32)
            o32, _, _ = self.propagate_frames(x32, x_hi, x_lo, flows_backward, flows_forward)
            return o32.permute(0, 1, 4, 2, 3)
        frames = [x[:, i].contiguous(memory_format=torch.channels_last) for i in range(t)]
        # every frame is a source of two convs per direction: split it into the bf16 operand pair once
        frame_ops = [ops.split_nhwc(f) for f in frames]
        swept = {}
        for name in self.DIRECTIONS:
            backward = name == "backward_"
            order = list(range(t - 1, -1, -1)) if backward else list(range(t))
            flows = flows_backward if backward else flows_forward
            align, backbone = self.deform_align[name], self.backbone[name]
            prop = torch.zeros_like(frames[0])
            hist = []
            for i, idx in enumerate(order):
                cur = frame_ops[idx]
                if i > 0:
                    flow_n1 = flows[:, i - 1]
                    grid_n1 = flow_n1.permute(0, 2, 3, 1)
                    cond_n1 = flow_warp(prop, grid_n1)
                    if i > 1:
                        feat_n2 = hist[-2]
                        flow_n2 = flow_n1 + flow_warp(flows[:, i - 2], grid_n1)
                        cond_n2 = flow_warp(feat_n2, flow_n2.permute(0, 2, 3, 1))
                    else:
                        feat_n2 = torch.zeros_like(prop)
                        flow_n2 = torch.zeros_like(flow_n1)
                        cond_n2 = torch.zeros_like(cond_n1)
                    prop = align.align(ops.dcn_pack_input(prop, feat_n2), [cond_n1, cur, cond_n2], flow_n1, flow_n2)
                parts = [cur, prop] if backward else [cur, swept["backward_"][idx], prop]
                # feat_prop + backbone(cat(parts)): conv+LeakyReLU(0.1), then conv with the residual add fused
                y = ops.conv3x3(parts, backbone[0].weight, backbone[0].bias, negative_slope=0.1, out="split")
                prop = ops.conv3x3([y], backbone[2].weight, backbone[2].bias, residual=prop)
                hist.append(prop)
            swept[name] = hist[::-1] if backward else hist
        # 1x1 fusion conv == a Linear over pixels; "+ x" is its fused residual (feat_prop.py:143-149)
        # cat(backward, forward) of every frame, written straight into the (b,t,h,w,2c) token buffer (no per-frame cat
        # followed by a stack)
        tokens = torch.empty((b, t, h, w, 2 * c), dtype=x.dtype, device=x.device)
        for i in range(t):
            tokens[:, i, :, :, :c].copy_(swept["backward_"][i].permute(0, 2, 3, 1))
            tokens[:, i, :, :, c:].copy_(swept["forward_"][i].permute(0, 2, 3, 1))
        out = ops.linear(tokens, self.fusion.weight, self.fusion.bias, residual=x.permute(0, 1, 3, 4, 2))
        return out.permute(0, 1, 4, 2, 3)
