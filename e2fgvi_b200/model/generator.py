"""InpaintGenerator — the drop-in boundary (reference: model/e2fgvi.py:71-263, model/e2fgvi_hq.py).

Contract kept (SURVEY §8(b)): ``InpaintGenerator()`` takes no required args, ``load_state_dict`` of a reference
checkpoint is strict-compatible (243 entries base / 244 HQ), and
``forward(masked_frames[b,t,3,H,W], num_local_frames) -> (pred[b*t,3,H,W], (flows_fwd, flows_bwd))``, inference-only.
``forward_bidirect_flow`` has a backward pass into ``update_spynet`` (the flow-completion loss of train.py).
The constructor never downloads SPyNet weights.
"""
import contextlib

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ._kept import KeptLaunches, tracked
from .modules.flow_comp import SPyNet
from .modules.feat_prop import BidirectionalPropagation, SecondOrderDeformableAlignment
from .modules.tfocal_transformer import SoftComp, SoftSplit, TemporalFocalTransformerBlock

# Encoder convs: (cin, cout, stride, groups); LeakyReLU(0.2) after each (e2fgvi.py:75-94).
# From the 6th conv on, the input is the 256-ch tensor x0 (input of conv 5) concatenated group-wise with the
# previous output (e2fgvi.py:96-109).
_ENC = ((3, 64, 2, 1), (64, 64, 1, 1), (64, 128, 2, 1), (128, 256, 1, 1), (256, 384, 1, 1),
        (640, 512, 1, 2), (768, 384, 1, 4), (640, 256, 1, 8), (512, 128, 1, 1))


@contextlib.contextmanager
def library_precision(mode):
    """TF32 switch of torch's LIBRARY ops around forward.  No cuDNN / cuBLAS kernel is left on the path (every conv and
    Linear runs on the bf16x3 wgmma kernels, DCN / attention on fp16 operands with fp32 accumulation), so this only
    matters for library ops a caller wraps around the model; "strict" (default) keeps them at full fp32 like the
    reference's CPU path — TF32 costs 3-7e-3 over ~60 layers on O(1) activations (DESIGN.md §2) — "tf32" restores
    PyTorch's own default."""
    if mode not in ("strict", "tf32"):
        raise ValueError("precision must be 'strict' or 'tf32'")
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = (mode == "tf32")
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


class BaseNetwork(nn.Module):
    def print_network(self):
        n = sum(p.numel() for p in self.parameters())
        print(f"Network [{type(self).__name__}] was created. Total number of parameters: {n / 1e6:.1f} million.")

    def init_weights(self, init_type="normal", gain=0.02):
        """N(0, gain) on every Conv*/Linear weight, zero bias (e2fgvi.py:29-68, 'normal' branch only)."""
        if init_type != "normal":
            raise NotImplementedError("only the reference default init_type='normal' is provided")
        for m in self.modules():
            cls = type(m).__name__
            if hasattr(m, "weight") and ("Conv" in cls or "Linear" in cls) and isinstance(m.weight, torch.Tensor):
                nn.init.normal_(m.weight.data, 0.0, gain)
                if getattr(m, "bias", None) is not None:
                    nn.init.constant_(m.bias.data, 0.0)
        ops.invalidate_weight_caches()      # `.data` updates do not bump Parameter versions

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        ops.invalidate_weight_caches()
        if self._graphs is not None:
            self._graphs = {}                               # captured graphs hold the old derived operands
        return out


class Encoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.group = [1, 2, 4, 8, 1]
        layers = []
        for cin, cout, stride, groups in _ENC:
            layers += [nn.Conv2d(cin, cout, 3, stride, 1, groups=groups), nn.LeakyReLU(0.2, inplace=True)]
        self.layers = nn.ModuleList(layers)

    def forward(self, x, last_out="f32"):
        """All nine convs run on the wgmma implicit-GEMM kernel (stride 2 via TMA element strides) with LeakyReLU
        fused and the bf16 split operand handed from epilogue to the next conv; the group-wise concatenation of
        e2fgvi.py:103-108 is expressed as two TMA sources, never materialised.  ``last_out="both"`` also returns the
        bf16 (hi, lo) split of the features (operand of the propagation convs and of SoftSplit).

        Trainable: with grad mode on, the default ``last_out`` and some encoder parameter requiring grad, the features
        carry a ``grad_fn`` whose backward gives the parameters that require grad their gradients
        (``_encoder_backward``); the features are bit-identical to the untracked call.  Frames that require grad raise
        ``ValueError`` (no gradient into the frames).  Other ``last_out`` values stay untracked."""
        if last_out == "f32":
            params = [t for conv in self.layers[::2] for t in (conv.weight, conv.bias)]
            if tracked((), params):
                if x.requires_grad:
                    raise ValueError("Encoder: the gradient with respect to the frames is not implemented (detach them; "
                                     "the features' gradient reaches the encoder's parameters)")
                return KeptLaunches.apply("Encoder", _encoder_run, _encoder_backward, self, x, *params)
        return self._forward(x, last_out)

    def _forward(self, x, last_out="f32", keep=None):
        """The launch sequence of ``forward``; ``keep`` (a list or None) receives each conv's input operands (the stem's
        row-gapped frames, then [SplitNHWC] or [x0, SplitNHWC] for the two-source convs): the LeakyReLU outputs the
        backward reads."""
        out = x
        x0 = None
        last = len(_ENC) - 1
        for k, (_, _, stride, _) in enumerate(_ENC):
            conv = self.layers[2 * k]
            mode = last_out if k == last else "split"
            if k == 0:
                # 3-channel stem: row-gapped 4-channel layout, window-packed K (3 K chunks per tile instead of 9
                # taps zero-padded from 3 to 64 channels)
                out = ops.pack_rows(out, lead=conv.padding[0])
            if k == 4:
                x0 = out
            if keep is not None:
                keep.append([x0, out] if k > 4 else [out])
            if k > 4 and conv.out_channels // conv.groups <= 32 and mode == "split":
                # groups of 32 output channels (e2fgvi.py:97): the kx-in-N kernel, one tile per (pixels, group)
                out = ops.conv_kxn([x0, out], conv.weight, conv.bias, negative_slope=0.2, out=mode, groups=conv.groups)
            elif k > 4:
                out = ops.conv3x3([x0, out], conv.weight, conv.bias, groups=self.group[k - 4], negative_slope=0.2,
                                  out=mode)
            else:
                out = ops.conv3x3([out], conv.weight, conv.bias, negative_slope=0.2, out=mode, stride=stride)
        return out


def _encoder_run(keep, enc, frames, *params):
    """``Encoder.forward``'s tracked launches: ``_forward`` keeping each conv's input operands; saves the frames, the
    features and the 18 parameters."""
    keep["enc"], keep["inputs"] = enc, []
    feat = enc._forward(frames, "f32", keep["inputs"])
    return feat, (frames, feat, *params)


def _encoder_backward(keep, saved, needs, grad):
    """Gradients of the encoder's parameters from ``grad`` = d loss / d features (N, 128, h, w).  Convs 8 -> 0:
    LeakyReLU's derivative at each conv's output is fused into the input gradient that produces that output's
    gradient; x0 (conv 3's output, read by convs 4-8) collects the contributions of convs 8, 7, 6, 5 through the
    residual epilogue, and conv 4's input gradient adds its own and applies the derivative:
    (acc4 + (acc5 + (acc6 + (acc7 + acc8)))) * LeakyReLU'(x0).  The walk stops at the lowest conv with a trainable
    parameter.  Returns (None, None, dW0, db0, dW1, ...) (None where not needed)."""
    enc, inputs = keep["enc"], keep["inputs"]
    frames, feat = saved[:2]
    need = list(zip(needs[2::2], needs[3::2]))         # (weight, bias) of conv k need a gradient
    grads = [None] * (2 * len(_ENC))
    active = [k for k in range(len(_ENC)) if any(need[k])]
    if not active:
        return (None, None, *grads)
    lowest = active[0]
    convs = [enc.layers[2 * k] for k in range(len(_ENC))]
    g = grad.permute(0, 2, 3, 1)                 # NHWC, a view for channels_last gradients
    dy32, dy = ops.leaky_relu_backward(g, feat.permute(0, 2, 3, 1), 0.2, out="both")
    dx0 = None
    x0_c = _ENC[4][0]
    for k in range(len(_ENC) - 1, lowest - 1, -1):
        cin, cout, stride, groups = _ENC[k]
        conv = convs[k]
        nw, nb = need[k]
        if nw or nb:
            srcs = [ops.pack_rows(frames, lead=1, cin=8)] if k == 0 else inputs[k]   # 8-channel copy of the frames
            dw, db = ops.conv3x3_wgrad(dy32, srcs, groups=groups, stride=stride, with_bias=nb,
                                       cin=cin // groups)
            grads[2 * k] = dw if nw else None
            grads[2 * k + 1] = db
        if k == lowest:
            break
        if k > 4:
            chans = [x0_c, cin - x0_c]
            if lowest <= 3:
                dx0 = ops.conv_dgrad(dy, conv.weight, groups=groups, src_channels=chans, source=0, residual=dx0)
            dy32, dy = ops.conv_dgrad(dy, conv.weight, groups=groups, src_channels=chans, source=1, act=inputs[k][1],
                                      out="both")
        else:
            src = inputs[k][0]
            dy32, dy = ops.conv_dgrad(dy, conv.weight, stride=stride, in_size=src.shape[2:], act=src,
                                      residual=dx0 if k == 4 else None, out="both")
    return (None, None, *grads)


class deconv(nn.Module):
    """x2 bilinear upsample (align_corners=True) + conv (e2fgvi.py:112-130)."""

    def __init__(self, input_channel, output_channel, kernel_size=3, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(input_channel, output_channel, kernel_size=kernel_size, stride=1, padding=padding)

    def forward(self, x):
        """Stand-alone call (the generator's ``_decode`` fuses the following LeakyReLU and keeps the bf16 split between
        layers): the same two kernels — x2 bilinear upsample written as the conv's split operand, then the conv."""
        return ops.conv3x3([ops.upsample2x_split(x)], self.conv.weight, self.conv.bias)


class InpaintGenerator(BaseNetwork):
    HQ = False

    def __init__(self, init_weights=True):
        super().__init__()
        channel, hidden = 256, 512
        self.encoder = Encoder()
        self.decoder = nn.Sequential(
            deconv(channel // 2, 128, kernel_size=3, padding=1), nn.LeakyReLU(0.2, inplace=True),
            nn.Conv2d(128, 64, kernel_size=3, stride=1, padding=1), nn.LeakyReLU(0.2, inplace=True),
            deconv(64, 64, kernel_size=3, padding=1), nn.LeakyReLU(0.2, inplace=True),
            nn.Conv2d(64, 3, kernel_size=3, stride=1, padding=1))
        self.feat_prop_module = BidirectionalPropagation(channel // 2)

        kernel_size, padding, stride, output_size = (7, 7), (3, 3), (3, 3), (60, 108)
        t2t_params = {"kernel_size": kernel_size, "stride": stride, "padding": padding}
        if not self.HQ:
            t2t_params["output_size"] = output_size
        self.ss = SoftSplit(channel // 2, hidden, kernel_size, stride, padding, t2t_param=t2t_params)
        self.sc = SoftComp(channel // 2, hidden, None if self.HQ else output_size, kernel_size, stride, padding,
                           hq=self.HQ)
        n_vecs = 1
        for i, d in enumerate(kernel_size):
            n_vecs *= int((output_size[i] + 2 * padding[i] - (d - 1) - 1) / stride[i] + 1)
        depths = 8
        self.transformer = nn.Sequential(*[
            TemporalFocalTransformerBlock(dim=hidden, num_heads=4, window_size=(5, 9), focal_level=2,
                                          focal_window=(5, 9), n_vecs=n_vecs, t2t_params=t2t_params,
                                          pool_method="fc", hq=self.HQ) for _ in range(depths)])
        if init_weights:
            self.init_weights()
            for m in self.modules():
                if isinstance(m, SecondOrderDeformableAlignment):
                    m.init_offset()
        # built after init_weights, like the reference (e2fgvi.py:208): keeps its own default init
        self.update_spynet = SPyNet()

    def forward_bidirect_flow(self, masked_local_frames):
        """1/4 bilinear downsample then SPyNet in both directions (e2fgvi.py:210-234); both directions run as
        one batched SPyNet call (every op inside is batch-independent).  masked_local_frames (b, l_t, 3, h, w) in [0, 1].

        Trainable: with grad mode on and some ``update_spynet`` parameter requiring grad, CUDA frames go through the
        fused SPyNet path with a backward pass (``SPyNet.bidirect_flows``), and the flows carry a ``grad_fn`` into
        ``update_spynet``: the flow-completion step of train.py (see INTEGRATION "Flow completion").  The flows equal
        ``forward(masked_frames, l_t)[1]`` bit for bit when masked_local_frames = (masked_frames[:, :l_t] + 1) / 2.
        Frames that require grad raise ``ValueError`` there (no gradient into the frames)."""
        b, l_t, c, h, w = masked_local_frames.size()
        if masked_local_frames.is_cuda and l_t > 1 and tracked((), self.update_spynet.parameters()):
            return self.update_spynet.bidirect_flows(masked_local_frames, l_t, unit=True)
        small = F.interpolate(masked_local_frames.reshape(-1, c, h, w), scale_factor=1 / 4, mode="bilinear",
                              align_corners=True, recompute_scale_factor=True)
        small = small.view(b, l_t, c, h // 4, w // 4)
        a = small[:, :-1].reshape(-1, c, h // 4, w // 4)
        z = small[:, 1:].reshape(-1, c, h // 4, w // 4)
        n = a.size(0)
        both = self.update_spynet(torch.cat([a, z]), torch.cat([z, a]))
        fwd = both[:n].reshape(b, l_t - 1, 2, h // 4, w // 4)
        bwd = both[n:].reshape(b, l_t - 1, 2, h // 4, w // 4)
        return fwd, bwd

    precision = "strict"
    # SPyNet on a side stream next to the encoder (see _forward).  The benchmark's per-kernel profiling pass sets this to
    # False: kernels that run concurrently on two streams inflate each other's event-timed launches.
    overlap_flow = True
    _side_streams = None

    def _side_stream(self, device):
        if self._side_streams is None:
            self._side_streams = {}
        key = device.index if device.index is not None else torch.cuda.current_device()
        if key not in self._side_streams:
            self._side_streams[key] = torch.cuda.Stream(device=device)
        return self._side_streams[key]

    _warned_grad = False

    def forward(self, masked_frames, num_local_frames):
        """INFERENCE ONLY, CUDA ONLY: outputs carry no grad_fn, the flows included, and there is no CPU path.  To train
        ``update_spynet`` on the flow-completion loss, call ``forward_bidirect_flow`` (it has a backward pass).  The
        flows of this call stay untracked on purpose: with the trainer's ``gen_loss = gan + flow + hole + valid``, flows
        that alone tracked gradients would make ``gen_loss.backward()`` silently leave out every image-loss path into
        ``update_spynet``."""
        # (CPU tensors fail loudly inside the first kernel wrapper: ops._need_cuda, "there is no CPU fallback")
        if torch.is_grad_enabled() and not InpaintGenerator._warned_grad and any(p.requires_grad for p in self.parameters()):
            import warnings
            InpaintGenerator._warned_grad = True
            warnings.warn("e2fgvi_b200.InpaintGenerator.forward is inference-only: its outputs do not track gradients "
                          "(call it under torch.no_grad())", RuntimeWarning, stacklevel=2)
        if self._graphs is not None and masked_frames.is_cuda and not torch.cuda.is_current_stream_capturing():
            return self._forward_graphed(masked_frames, num_local_frames)
        return self._forward_eager(masked_frames, num_local_frames)

    def _forward_eager(self, masked_frames, num_local_frames):
        with library_precision(self.precision):
            return self._forward(masked_frames, num_local_frames)

    # ---- CUDA-graph replay behind the SAME call (model(x, l_t)): a single 432x240 clip is ~195 kernel launches for ~6 ms
    # of GPU work, so launching from Python costs more than the GPU time.  Opt-in, because replay returns tensors
    # produced by a captured allocation pool and requires the weights not to change between calls.
    _graphs = None
    _graph_limit = 4

    def enable_cuda_graphs(self, enabled=True, max_shapes=4):
        """``model.enable_cuda_graphs()``: every subsequent ``model(x, l_t)`` with a CUDA input replays a CUDA graph
        captured on the first call with that (shape, l_t) (up to ``max_shapes`` distinct shapes are kept, least recently
        used dropped).  Outputs are fresh tensors (copies of the graph's static outputs).  Weights must stay constant
        (inference); call ``enable_cuda_graphs(False)`` or ``load_state_dict`` to drop the captures."""
        self._graphs = {} if enabled else None
        self._graph_limit = int(max_shapes)
        return self

    def _forward_graphed(self, masked_frames, num_local_frames):
        from ..graph import GraphedGenerator
        key = (tuple(masked_frames.shape), int(num_local_frames), masked_frames.device.index, masked_frames.dtype)
        g = self._graphs.pop(key, None)
        if g is None:
            if len(self._graphs) >= self._graph_limit:
                self._graphs.pop(next(iter(self._graphs)))
            g = GraphedGenerator(self, masked_frames, num_local_frames)
        self._graphs[key] = g                               # most recently used last
        pred, flows = g(masked_frames)
        return pred.clone(), tuple(f.clone() for f in flows)

    def _forward(self, masked_frames, num_local_frames):
        l_t = num_local_frames
        b, t, ori_c, ori_h, ori_w = masked_frames.size()
        side = None
        if masked_frames.is_cuda and l_t > 1:
            # fused glue: (x + 1) / 2, the 1/4 downsample, the pyramids, per-level upsample + warp + cat (38 launches).
            # SPyNet only depends on the input frames, like the encoder: it runs on a side stream (a parallel branch of
            # a captured CUDA graph) so that its latency-bound coarse pyramid levels (8-32 CTAs for ~20 us each) fill in
            # next to the encoder's convs instead of preceding them on the single-clip critical path
            if self.overlap_flow:
                main = torch.cuda.current_stream()
                side = self._side_stream(masked_frames.device)
                side.wait_stream(main)
                with torch.cuda.stream(side), torch.no_grad():
                    pred_flows = self.update_spynet.bidirect_flows(masked_frames, l_t)
            else:
                with torch.no_grad():
                    pred_flows = self.update_spynet.bidirect_flows(masked_frames, l_t)
        else:
            with torch.no_grad():
                pred_flows = self.forward_bidirect_flow((masked_frames[:, :l_t] + 1) / 2)

        # encoder output: fp32 (b*t,c,h,w) in NHWC storage + its bf16 (hi, lo) split, both viewed as (b,t,h,w,c)
        enc32, enc_sp = self.encoder(masked_frames.reshape(b * t, ori_c, ori_h, ori_w), last_out="both")
        if side is not None:
            torch.cuda.current_stream().wait_stream(side)
            for f in pred_flows:                       # produced on the side stream, consumed (and freed) on this one
                f.record_stream(torch.cuda.current_stream())
        _, c, h, w = enc32.size()
        x32 = enc32.permute(0, 2, 3, 1).view(b, t, h, w, c)
        x_hi, x_lo = enc_sp.hi.view(b, t, h, w, c), enc_sp.lo.view(b, t, h, w, c)
        # NB: (forward, backward) flows go to (flows_backward, flows_forward) exactly as e2fgvi.py:249-250 does.
        # The local frames are propagated IN PLACE inside the (b,t,h,w,c) feature buffers (frame slices are read and
        # written by batch-strided convs): the cat(local_feat, enc_feat[:, l_t:]) of e2fgvi.py:252 is the buffer itself
        self.feat_prop_module.propagate_frames(x32[:, :l_t], x_hi[:, :l_t], x_lo[:, :l_t], pred_flows[0], pred_flows[1],
                                               into=(x32[:, :l_t], x_hi[:, :l_t], x_lo[:, :l_t]))
        enc_feat = enc32                                                # logical (b*t,c,h,w), NHWC storage

        fold_size = (h, w)
        tokens = self.ss(enc_sp, b, fold_size if self.HQ else None)
        # the blocks' untracked launches: a tracked block would keep its backward operands inside an inference call
        for blk in self.transformer:
            tokens = blk._forward(tokens, fold_size if self.HQ else None)
        # enc_feat + trans_feat (e2fgvi.py:263) is fused into SoftComp's fold / conv epilogue
        enc_feat = self.sc._forward(tokens, t, fold_size if self.HQ else None, residual=enc_feat)

        # tanh and the NCHW layout of the prediction are fused into the last decoder conv's epilogue
        return self._decode(enc_feat), pred_flows

    def decode(self, feat):
        """``tanh(self.decoder(feat))``, the decoder step of e2fgvi.py:262: feat (N, 128, h, w) -> prediction (N, 3, 4h, 4w)
        fp32, on ``_decode``'s kernel sequence.  With grad mode on and ``feat`` or some decoder parameter requiring
        grad, the prediction carries a ``grad_fn`` into both (``_decode_backward``); its values are the same bits."""
        params = self._decoder_params()
        if tracked([feat], params):
            return KeptLaunches.apply("decode", _decode_run, _decode_backward, self, feat, *params)
        return self._decode(feat)

    def _decoder_params(self):
        d = self.decoder
        return [t for conv in (d[0].conv, d[2], d[4].conv, d[6]) for t in (conv.weight, conv.bias)]

    def _decode(self, x, keep=None):
        """tanh(self.decoder(x)) (e2fgvi.py:143-150, :262) with the convs on the wgmma kernel, LeakyReLU(0.2) fused, and
        tanh + the NCHW store fused into the output conv.  ``keep`` (a list or None) receives the convs' operands: the
        upsampled input, the first conv's output, the second's (fp32), its upsample and the third's output."""
        d = self.decoder
        u0 = ops.upsample2x_split(x)
        y1 = ops.conv3x3([u0], d[0].conv.weight, d[0].conv.bias, negative_slope=0.2, out="split")
        y2 = ops.conv3x3([y1], d[2].weight, d[2].bias, negative_slope=0.2)
        u1 = ops.upsample2x_split(y2)
        y3 = ops.conv3x3([u1], d[4].conv.weight, d[4].conv.bias, negative_slope=0.2, out="split")
        if keep is not None:
            keep += [u0, y1, y2, u1, y3]
        return ops.conv3x3_tanh_nchw(y3, d[6].weight, d[6].bias)


def _decode_run(keep, gen, feat, *params):
    """``decode``'s tracked launches: ``_decode`` keeping its operands; saves the prediction and the 8 parameters."""
    keep["gen"], keep["ops"] = gen, []
    pred = gen._decode(feat, keep["ops"])
    return pred, (pred, *params)


def _decode_backward(keep, saved, needs, grad):
    """Gradients of ``decode`` into the features and the decoder convs (decoder[0].conv, [2], [4].conv, [6]).  tanh's
    derivative feeds the output conv's gradients; each input gradient fuses LeakyReLU's derivative at the activation it
    reaches (after the upsample adjoint for the deconvs).  Returns (None, d feat (N, 128, h, w), dW0, db0, ...), None
    where not needed."""
    d = keep["gen"].decoder
    pred = saved[0]
    want_feat = needs[1]
    need = list(zip(needs[2::2], needs[3::2]))         # (weight, bias) of decoder conv i need a gradient
    convs = (d[0].conv, d[2], d[4].conv, d[6])
    u0, y1, y2, u1, y3 = keep["ops"]
    srcs = (u0, y1, u1, y3)
    grads = [None] * 8
    active = [i for i in range(4) if any(need[i])]
    lowest = 0 if want_feat else (active[0] if active else 4)
    if lowest == 4:
        return (None, None, *grads)
    dy32, dy = ops.tanh_backward_rows(grad, pred, lead=1)
    cout = convs[3].out_channels
    dfeat = None
    for i in range(3, lowest - 1, -1):
        nw, nb = need[i]
        if nw or nb:
            dw, db = ops.conv3x3_wgrad(dy32[..., :cout] if i == 3 else dy32, [srcs[i]], with_bias=nb)
            grads[2 * i] = dw if nw else None
            grads[2 * i + 1] = db
        if i == 3 and lowest < 3:
            dy32, dy = ops.conv_dgrad(dy, convs[3].weight, act=y3, out="both")
        elif i == 2 and lowest < 2:
            dy32, dy = ops.upsample2x_backward(ops.conv_dgrad(dy, convs[2].weight), act=y2, out="both")
        elif i == 1 and lowest < 1:
            dy32, dy = ops.conv_dgrad(dy, convs[1].weight, act=y1, out="both")
        elif i == 0 and want_feat:
            dfeat = ops.upsample2x_backward(ops.conv_dgrad(dy, convs[0].weight)).permute(0, 3, 1, 2)
    return (None, dfeat, *grads)


class InpaintGeneratorHQ(InpaintGenerator):
    HQ = True
