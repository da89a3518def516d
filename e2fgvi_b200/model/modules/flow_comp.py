"""Flow completion on the hot path: SPyNet and ``flow_warp`` (reference: model/modules/flow_comp.py:49-226,345-383).

State-dict layout (must stay byte-compatible with released checkpoints, SURVEY §8(b)):
``basic_module.{0..5}.basic_module.{0..4}.conv.{weight,bias}`` + buffers ``mean``/``std`` [1,3,1,1].
The ``.conv.`` level exists in the reference because it wraps each conv in ``mmcv.cnn.ConvModule``
(flow_comp.py:181-215); here a tiny holder module provides the same key path with no mmcv dependency.
The constructor never touches the network (the reference downloads pretrained weights, flow_comp.py:59-72;
E2FGVI checkpoints carry ``update_spynet.*`` anyway).
"""
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


def _basic_module_rows(module, rows, residual):
    """SPyNetBasicModule on a ready row-gapped operand; the last conv adds ``residual`` = flow_up (flow_comp.py:127:
    ``flow = flow_up + basic_module(...)``) in its epilogue and returns the new flow (P, hk, wk, 2) fp32."""
    convs = [holder.conv for holder in module.basic_module]
    y = rows
    last = len(convs) - 1
    if ops.KXN_CONVS:
        # 8 -> 32 and 32 -> 64 on the window-packed kernel (wide enough outputs), then 64 -> 32, 32 -> 16 and 16 -> 2 on
        # the kx-in-N kernel: with <= 32 output channels the plain implicit GEMM re-reads its A tile for every tap
        y = ops.conv3x3(y, convs[0].weight, convs[0].bias, negative_slope=0.0, out="rows", out_lead=convs[1].padding[0])
        y = ops.conv3x3(y, convs[1].weight, convs[1].bias, negative_slope=0.0, out="split")
        y = ops.conv_kxn(y, convs[2].weight, convs[2].bias, negative_slope=0.0, out="split")
        y = ops.conv_kxn(y, convs[3].weight, convs[3].bias, negative_slope=0.0, out="split")
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

    def bidirect_flows(self, masked_frames, num_local_frames):
        """Both flow directions of ``InpaintGenerator.forward_bidirect_flow`` (e2fgvi.py:210-234) straight from the
        masked frames (b,t,3,H,W) in [-1,1]: 1 pyramid launch, per level 1 input launch + five 7x7 convs, 1 final
        launch.  Returns (flows_forward, flows_backward), each (b, l_t-1, 2, H/4, W/4)."""
        pyr = ops.spynet_pyramid(masked_frames, num_local_frames, self.mean, self.std)
        flow = None
        for level in range(_NUM_LEVELS):
            rows, flow_up = ops.spynet_level_input(pyr, _NUM_LEVELS - 1 - level, flow,
                                                   lead=self.basic_module[level].basic_module[0].conv.padding[0])
            flow = _basic_module_rows(self.basic_module[level], rows, flow_up)
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
