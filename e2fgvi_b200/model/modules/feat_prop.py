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
from .._kept import KeptLaunches, tracked
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

    def transposed_weight(self):
        """bf16 split of W16^T, the weight operand of the backward's dA = dY . W16, cached like ``packed_weight``."""
        return ops._derived_one(self.weight, ("dcn_t", self.deform_groups),
                                lambda w, g: ops.dcn_transposed_split(w, g), self.deform_groups)

    def _flows_dgrad_weight(self):
        """conv_offset.0's weight with 4 zero input channels after the flows' 4: its flows source is read as 8
        channels (the split pads it), and the input-gradient kernel takes 8-channel sources."""
        return ops._derived_one(self.conv_offset[0].weight, ("dcn_head_flows8",),
                                lambda w: F.pad(w.detach().float(), (0, 0, 0, 0, 0, 4)))

    def _params(self):
        co = self.conv_offset
        return [self.weight, self.bias] + [t for k in (0, 2, 4, 6) for t in (co[k].weight, co[k].bias)]

    def _forward_keep(self, x, extra_feat, flow_1, flow_2, keep):
        """``align(x, [extra_feat], flow_1, flow_2)``'s launches, keeping the operands of the backward: the fp16 x,
        the head convs' split inputs (the LeakyReLU outputs also in fp32, for the activation's derivative), the raw head
        and the flows.  The same kernels compute the same bits; the head convs also store their fp32 outputs."""
        co = self.conv_offset
        if x.dtype != torch.float16 or not ops._is_cl(x):
            x = x.to(dtype=torch.float16, memory_format=torch.channels_last)
        srcs = [ops.split_nhwc(extra_feat), ops.split_nhwc(torch.cat([flow_1, flow_2], dim=1))]
        y1_32, y1 = ops.conv3x3(srcs, co[0].weight, co[0].bias, negative_slope=0.1, out="both")
        y2_32, y2 = ops.conv3x3([y1], co[2].weight, co[2].bias, negative_slope=0.1, out="both")
        y3_32, y3 = ops.conv3x3([y2], co[4].weight, co[4].bias, negative_slope=0.1, out="both")
        head = ops.conv3x3([y3], co[6].weight, co[6].bias)
        keep.update(x=x, head=head, flow_1=flow_1, flow_2=flow_2, srcs=[srcs, [y1], [y2], [y3]],
                    acts=[None, y1_32, y2_32, y3_32])
        return ops.deform_align_fused(x, head, flow_1, flow_2, self.packed_weight(), self.bias, self.deform_groups,
                                      self.max_residue_magnitude)

    def forward(self, x, extra_feat, flow_1, flow_2):
        """Reference boundary (feat_prop.py:35): extra_feat is the already concatenated condition tensor.  Under grad
        mode, with the fused kernel, and when x, extra_feat, a flow or a parameter requires grad, the result carries a
        ``grad_fn`` into all of them (``_align_backward``); it is bit-identical to the untracked call."""
        params = self._params()
        if self.fused and tracked((x, extra_feat, flow_1, flow_2), params):
            return KeptLaunches.apply("SecondOrderDeformableAlignment", _align_run, _align_back, self, x, extra_feat,
                                      flow_1, flow_2, *params)
        return self.align(x, [extra_feat], flow_1, flow_2)


def _align_run(keep, mod, x, extra_feat, flow_1, flow_2, *params):
    """The tracked launches of ``SecondOrderDeformableAlignment.forward`` (``_forward_keep``); saves the 10
    parameters."""
    keep["mod"] = mod
    return mod._forward_keep(x, extra_feat, flow_1, flow_2, keep), params


def _align_back(keep, saved, needs, grad):
    """``_align_backward`` for ``_align_run``."""
    return (None, *_align_backward(keep["mod"], keep, grad, needs[1:5], needs[5:]))


def _align_backward(mod, keep, grad, need_in, need):
    """Gradients of ``SecondOrderDeformableAlignment.forward``.  need_in = (x, extra_feat, flow_1, flow_2) need a
    gradient; need = the 10 parameters of ``_params()``.  The DCN backward (``ops.deform_align_backward``) gives dx, dW,
    db and d head with the offsets' share of d flow; the walk down the offset head (convs 6, 4, 2, 0) then runs each
    conv's weight gradient where needed and its input gradient times LeakyReLU(0.1)'s derivative, and stops at the
    lowest conv that needs something.  conv 0's flows input gradient adds the offsets' share (its residual).
    Returns (dx, d extra_feat, d flow_1, d flow_2, *parameter gradients)."""
    nx, ne, nf1, nf2 = need_in
    nf = nf1 or nf2
    head_need = [(need[2 + 2 * i], need[3 + 2 * i]) for i in range(4)]
    active = [i for i in range(4) if any(head_need[i])]
    lowest = 0 if (ne or nf) else (active[0] if active else 4)
    need_head = lowest < 4
    dx, dhead, dflow, dw, db = ops.deform_align_backward(
        keep["x"], keep["head"], keep["flow_1"], keep["flow_2"], mod.packed_weight(), grad, mod.deform_groups,
        mod.max_residue_magnitude, need_x=nx, need_head=need_head, need_flow=nf, need_weight=need[0],
        need_bias=need[1], wt_split=mod.transposed_weight() if (nx or need_head) else None)
    grads = [dw, db] + [None] * 8
    dextra = dflow1 = dflow2 = None
    if need_head:
        co = mod.conv_offset
        convs = [co[0], co[2], co[4], co[6]]
        srcs, acts = keep["srcs"], keep["acts"]
        g32 = dhead.permute(0, 2, 3, 1)                       # NHWC, a view
        gsp = ops.SplitNHWC(*ops.split_bf16(g32), dhead.shape)
        extra_c = srcs[0][0].shape[1]
        chans = [extra_c, 4]
        for i in range(3, lowest - 1, -1):
            nw_i, nb_i = head_need[i]
            if nw_i or nb_i:
                dw_i, db_i = ops.conv3x3_wgrad(g32, srcs[i], with_bias=nb_i, cin=extra_c + 4 if i == 0 else None)
                grads[2 + 2 * i] = dw_i if nw_i else None
                grads[3 + 2 * i] = db_i
            if i > lowest:
                d = ops.conv_dgrad(gsp, convs[i].weight)
                g32, gsp = ops.leaky_relu_backward(d, acts[i].permute(0, 2, 3, 1), 0.1, out="both")
        if ne:
            dextra = ops.conv_dgrad(gsp, convs[0].weight, src_channels=chans, source=0).permute(0, 3, 1, 2)
        if nf:
            d8 = ops.conv_dgrad(gsp, mod._flows_dgrad_weight(), src_channels=[extra_c, 8], source=1, residual=dflow)
            dflow1 = d8[..., 0:2].permute(0, 3, 1, 2) if nf1 else None
            dflow2 = d8[..., 2:4].permute(0, 3, 1, 2) if nf2 else None
    return (dx, dextra, dflow1, dflow2, *grads)


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

    def _params(self):
        """The 30 parameters in the order of the tracked call: per direction the alignment's 10 and the backbone's 4,
        then the fusion's weight and bias."""
        ps = []
        for name in self.DIRECTIONS:
            bb = self.backbone[name]
            ps += self.deform_align[name]._params() + [bb[0].weight, bb[0].bias, bb[2].weight, bb[2].bias]
        return ps + [self.fusion.weight, self.fusion.bias]

    def _propagate_keep(self, x32, x_hi, x_lo, flows_backward, flows_forward, keep):
        """``propagate_frames``' launches for (b,t,h,w,c) x, keeping the operands of the backward: per step the
        prologue's outputs, the grouped fp16 DCN input, the offset head's split inputs and fp32 LeakyReLU outputs, the
        raw head, the backbone conv 0's output (fp32 and split) and the aligned features' split; per direction the
        results' (t,b,h,w,c) fp32 and split buffers.  The head convs and backbone conv 0 store their fp32 output too
        (out="both"); the same kernels compute the same bits, so the result is ``propagate_frames``' to the bit."""
        b, t, h, w, c = x32.shape
        cur = [ops.SplitNHWC(x_hi[:, i], x_lo[:, i], (b, c, h, w)) for i in range(t)]
        zero = torch.zeros((b, h, w, c), dtype=x_hi.dtype, device=x32.device)
        zero_sp = ops.SplitNHWC(zero, zero, (b, c, h, w))
        bufs, steps = {}, {}
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
            co = align.conv_offset
            r32, rhi, rlo = bufs[name]
            hist32, steps[name] = [], []
            for i, idx in enumerate(order):
                st = {"idx": idx}
                prop32, prop_sp = None, zero_sp
                if i > 0:
                    xg, cond_n1, cond_n2, flows_op, flow_n1, flow_n2 = ops.prop_prologue(
                        hist32[-1], hist32[-2] if i > 1 else None, flows[:, i - 1], flows[:, i - 2] if i > 1 else None)
                    y1_32, y1 = ops.conv_frames([cond_n1, cur[idx], cond_n2, flows_op], co[0].weight, co[0].bias,
                                                negative_slope=0.1, out="both")
                    y2_32, y2 = ops.conv_frames([y1], co[2].weight, co[2].bias, negative_slope=0.1, out="both")
                    y3_32, y3 = ops.conv_frames([y2], co[4].weight, co[4].bias, negative_slope=0.1, out="both")
                    head = ops.conv_frames([y3], co[6].weight, co[6].bias)
                    prop32, prop_sp = ops.deform_align_fused(xg, head, flow_n1, flow_n2, align.packed_weight(),
                                                             align.bias, align.deform_groups,
                                                             align.max_residue_magnitude, out_split=True)
                    st.update(xg=xg.data, head=head, flow_n1=flow_n1, flow_n2=flow_n2, conds=(cond_n1, cond_n2),
                              flows_op=flows_op, head_srcs=[[y1], [y2], [y3]], acts=[None, y1_32, y2_32, y3_32])
                parts = [cur[idx], prop_sp] if backward else [cur[idx], swept_sp["backward_"][idx], prop_sp]
                y32, y = ops.conv_frames(parts, backbone[0].weight, backbone[0].bias, negative_slope=0.1, out="both")
                new32, _ = ops.conv_frames([y], backbone[2].weight, backbone[2].bias, residual=prop32, out="both",
                                           into=(r32[idx], rhi[idx], rlo[idx]))
                st.update(parts=parts, y32=y32, y=y)
                hist32.append(new32)
                steps[name].append(st)
            swept_sp[name] = [ops.SplitNHWC(rhi[i], rlo[i], (b, c, h, w)) for i in range(t)]
        o32, ohi, olo = torch.empty_like(x32), torch.empty_like(x_hi), torch.empty_like(x_lo)
        if b == 1:
            srcs = [ops.SplitNHWC(bufs[n_][1].view(t, h, w, c), bufs[n_][2].view(t, h, w, c), (t, c, h, w)) for n_ in self.DIRECTIONS]
            ops.conv_frames(srcs, self.fusion.weight, self.fusion.bias, residual=x32[0].permute(0, 3, 1, 2), out="both",
                            into=(o32[0], ohi[0], olo[0]))
        else:
            for i in range(t):
                ops.conv_frames([swept_sp["backward_"][i], swept_sp["forward_"][i]], self.fusion.weight, self.fusion.bias,
                                residual=x32[:, i].permute(0, 3, 1, 2), out="both", into=(o32[:, i], ohi[:, i], olo[:, i]))
        keep.update(bufs=bufs, steps=steps, x_split=(x_hi, x_lo), shape=(b, t, h, w, c))
        return o32

    def forward(self, x, flows_backward, flows_forward):
        """x (b,t,c,h,w); flows_* (b,t-1,2,h,w) -> (b,t,c,h,w).  Under grad mode, on the fused path, and when x, a flow or
        a parameter requires grad, the result carries a ``grad_fn`` into all of them (``_prop_backward``); it is
        bit-identical to the untracked call."""
        b, t, c, h, w = x.shape
        if self.fused_prologue and c % 16 == 0:
            params = self._params()
            if tracked((x, flows_backward, flows_forward), params):
                return KeptLaunches.apply("BidirectionalPropagation", _prop_run, _prop_back, self, x, flows_backward,
                                          flows_forward, *params)
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


def _prop_run(keep, mod, x, flows_backward, flows_forward, *params):
    """The tracked launches of ``BidirectionalPropagation.forward`` (``_propagate_keep``); saves the 30 parameters."""
    x32 = x.permute(0, 1, 3, 4, 2).contiguous().float()
    x_hi, x_lo = ops.split_bf16(x32)
    keep.update(mod=mod, flows={"backward_": flows_backward, "forward_": flows_forward})
    o32 = mod._propagate_keep(x32, x_hi, x_lo, flows_backward, flows_forward, keep)
    return o32.permute(0, 1, 4, 2, 3), params


def _prop_back(keep, saved, needs, grad):
    """``_prop_backward`` for ``_prop_run``."""
    return (None, *_prop_backward(keep["mod"], keep, grad, needs[1:4], needs[4:]))


def _dense(sources):
    """One dense ``SplitNHWC`` of split operands (batch-strided frame slices allowed), channel-concatenated: the weight
    gradient reads dense sources, at most two of them."""
    if len(sources) == 1 and sources[0].hi.is_contiguous():
        return sources[0]
    n, _, h, w = sources[0].shape
    hi = torch.cat([s.hi for s in sources], -1) if len(sources) > 1 else sources[0].hi.contiguous()
    lo = torch.cat([s.lo for s in sources], -1) if len(sources) > 1 else sources[0].lo.contiguous()
    return ops.SplitNHWC(hi, lo, (n, hi.shape[-1], h, w))


def _accumulate(grads, first, parts):
    """Adds each step's parameter gradients to the sum of the steps walked before it (None: nothing to add)."""
    for j, v in enumerate(parts):
        if v is not None:
            grads[first + j] = v if grads[first + j] is None else grads[first + j].add_(v)


def _prop_backward(mod, keep, grad, need_in, need):
    """Gradients of the tracked ``BidirectionalPropagation.forward``.  need_in = (x, flows_backward, flows_forward) need a
    gradient; need = the 30 parameters of ``_params()``.  Returns (dx, d flows_backward, d flows_forward, *parameter
    gradients).

    The walk: the fusion, then the forward_ sweep last frame first, then the backward_ sweep in the reverse of its order.
    A step's result gradient G is, in this order: the fusion's share, the next step's (cond_n1 warp scatter + first half
    of its DCN dx), the step after's (cond_n2 warp scatter + second half of that DCN dx) and, for backward_ results, the
    forward_ backbone's read.  Per step: backbone conv 2 (its residual passes G to the aligned features), LeakyReLU(0.1)'s
    derivative and backbone conv 0, the alignment (``_align_backward`` on the step's kept operands) and the prologue's
    adjoint (``ops.flow_warp_backward``).  Steps whose result needs no gradient are skipped, frozen convs launch no weight
    gradient, and inputs that need none get no scatter."""
    nx, nfb, nff = need_in
    b, t, h, w, c = keep["shape"]
    bufs, steps = keep["bufs"], keep["steps"]
    names = mod.DIRECTIONS
    nflows = {"backward_": nfb, "forward_": nff}
    pn = {name: need[14 * k: 14 * k + 14] for k, name in enumerate(names)}     # [0:10] alignment, [10:14] backbone
    al_need = {n_: any(pn[n_][:10]) for n_ in names}
    bb_need = {n_: any(pn[n_][10:]) for n_ in names}
    # below[name][i]: the result of step i needs a gradient (something it reaches does)
    below = {}
    for name in names:
        below[name] = []
        for i in range(t):
            v = nx or bb_need[name] or (i >= 1 and (al_need[name] or nflows[name] or below[name][i - 1])) or \
                (i >= 2 and below[name][i - 2])
            if name == "forward_":
                v = v or below["backward_"][t - 1 - i]
            below[name].append(v)
    any_below = any(any(v) for v in below.values())
    grads = [None] * 30
    rows = t * b * h * w
    go = dcat = None
    if nx or need[28] or need[29] or any_below:
        go = grad.permute(1, 0, 3, 4, 2).contiguous().float()            # (t, b, h, w, c): the results' row order
    if need[28] or need[29]:
        gsp = ops.SplitMat(*ops.split_bf16(go.view(rows, c)))
        halves = []
        for k, name in enumerate(names):
            _, rhi, rlo = bufs[name]
            dw_k, db_k = ops.linear_wgrad(gsp, ops.SplitMat(rhi.view(rows, c), rlo.view(rows, c)),
                                          with_bias=need[29] and k == 0)
            halves.append(dw_k)
            if k == 0:
                grads[29] = db_k
            if not need[28]:
                break
        if need[28]:
            grads[28] = torch.cat(halves, 1).view(c, 2 * c, 1, 1)
    if any_below:
        dcat = ops.linear(go, mod.fusion.weight, transpose=True)           # (t, b, h, w, 2c)
    # the fusion's "+ x" passes the gradient on; a copy, since go may be the incoming gradient itself (b == 1), which
    # autograd may also hand to other branches
    dxs = go.clone() if nx else None
    dflows = {n_: torch.zeros((b, t - 1, 2, h, w), dtype=torch.float32, device=grad.device) if nflows[n_] else None
              for n_ in names}
    pend = {n_: [{} for _ in range(t)] for n_ in names}
    for k, name in reversed(list(enumerate(names))):
        off = 14 * k
        r32 = bufs[name][0]
        flows = keep["flows"][name]
        nf = nflows[name]
        align, bb = mod.deform_align[name], mod.backbone[name]
        pb = pn[name][10:]
        for i in range(t - 1, -1, -1):
            if not below[name][i]:
                continue
            st = steps[name][i]
            idx = st["idx"]
            g = dcat[idx, ..., k * c:(k + 1) * c].contiguous()
            for key in ("n1", "n2", "bb"):
                if key in pend[name][i]:
                    g.add_(pend[name][i].pop(key))
            if pb[2] or pb[3]:
                dw2, db2 = ops.conv3x3_wgrad(g, [st["y"]], with_bias=pb[3])
                _accumulate(grads, off + 12, [dw2 if pb[2] else None, db2])
            parts = st["parts"]
            need_rb = name == "forward_" and below["backward_"][t - 1 - idx]
            need_prop = i >= 1 and (al_need[name] or nf or nx or below[name][i - 1] or (i >= 2 and below[name][i - 2]))
            if not (pb[0] or pb[1] or nx or need_rb or need_prop):
                continue
            d = ops.conv_dgrad(ops.SplitNHWC(*ops.split_bf16(g), (b, c, h, w)), bb[2].weight)
            g0, g0_sp = ops.leaky_relu_backward(d, st["y32"].permute(0, 2, 3, 1), 0.1, out="both")
            if pb[0] or pb[1]:
                srcs = [_dense([s]) for s in parts] if len(parts) == 2 else [_dense(parts)]
                dw0, db0 = ops.conv3x3_wgrad(g0, srcs, with_bias=pb[1])
                _accumulate(grads, off + 10, [dw0 if pb[0] else None, db0])
            chans = [c] * len(parts)
            if nx:
                dxs[idx].add_(ops.conv_dgrad(g0_sp, bb[0].weight, src_channels=chans, source=0))
            if need_rb:
                pend["backward_"][t - 1 - idx]["bb"] = ops.conv_dgrad(g0_sp, bb[0].weight, src_channels=chans, source=1)
            if not need_prop:
                continue
            da = ops.conv_dgrad(g0_sp, bb[0].weight, src_channels=chans, source=len(parts) - 1, residual=g)
            # the alignment, on a keep dict of the step's operands
            need_r1, need_r2 = below[name][i - 1], i >= 2 and below[name][i - 2]
            n_dx = need_r1 or need_r2
            n_extra = n_dx or nx or nf
            cond_n1, cond_n2 = st["conds"]
            akeep = dict(x=st["xg"].permute(0, 2, 3, 1, 4).reshape(b, h, w, 2 * c).permute(0, 3, 1, 2),
                         head=st["head"], flow_1=st["flow_n1"], flow_2=st["flow_n2"],
                         srcs=[[_dense([cond_n1, parts[0], cond_n2]), st["flows_op"]]] + st["head_srcs"], acts=st["acts"])
            ddx, dextra, dfl1, dfl2, *ag = _align_backward(align, akeep, da.permute(0, 3, 1, 2),
                                                           (n_dx, n_extra, nf, nf and i >= 2), pn[name][:10])
            _accumulate(grads, off, ag)
            if nx:
                dxs[idx].add_(dextra[:, c:2 * c].permute(0, 2, 3, 1))
            # the prologue's adjoint
            f1n, f2n = st["flow_n1"].permute(0, 2, 3, 1), st["flow_n2"].permute(0, 2, 3, 1)
            dflow_n2 = None
            if i >= 2 and (need_r2 or nf):
                r2 = r32[steps[name][i - 2]["idx"]].permute(0, 3, 1, 2)
                c2, dflow_n2 = ops.flow_warp_backward(
                    r2, f2n, dextra[:, 2 * c:], need_x=need_r2, need_flow=nf,
                    residual=ddx[:, c:] if need_r2 else None, flow_residual=dfl2.permute(0, 2, 3, 1) if nf else None)
                if need_r2:
                    pend[name][i - 2]["n2"] = c2.permute(0, 2, 3, 1)
            dflow_n1 = None
            if need_r1 or nf:
                r1 = r32[steps[name][i - 1]["idx"]].permute(0, 3, 1, 2)
                fres = None
                if nf:
                    fres = dfl1.permute(0, 2, 3, 1)
                    if dflow_n2 is not None:
                        fres = fres + dflow_n2
                c1, dflow_n1 = ops.flow_warp_backward(r1, f1n, dextra[:, :c], need_x=need_r1, need_flow=nf,
                                                      residual=ddx[:, :c] if need_r1 else None, flow_residual=fres)
                if need_r1:
                    pend[name][i - 1]["n1"] = c1.permute(0, 2, 3, 1)
            if nf:
                if dflow_n2 is not None:
                    dprev, dflow_n1 = ops.flow_warp_backward(flows[:, i - 2], f1n, dflow_n2.permute(0, 3, 1, 2),
                                                             flow_residual=dflow_n1)
                    dflows[name][:, i - 2].add_(dprev)
                dflows[name][:, i - 1].add_(dflow_n1.permute(0, 3, 1, 2))
    dx = None if dxs is None else dxs.permute(1, 0, 4, 2, 3)
    return (dx, dflows["backward_"], dflows["forward_"], *grads)
