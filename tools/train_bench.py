"""Time one training stage of the library against the float32 autograd of a torch restatement.

    python tools/train_bench.py STAGE [stage shape options] [--iters N] [--warmup N] [--profile] [--out DIR]

STAGE is one of dis, flow, encdec, ffn, attn, block, align, prop; ``train_bench.py STAGE --help`` describes its steps
and lists its shape options.  Each step runs on this library's kernels, then on the torch reference with TF32 off and
on (both ``torch.backends.cuda.matmul.allow_tf32`` and ``torch.backends.cudnn.allow_tf32``; "on" is PyTorch's default
for cuDNN plus TF32 matmuls).  A time is the median of --iters steps after --warmup, CUDA events around each step, with
the gradients reset outside the events; a run that does not fit in memory is reported as "out of memory".  The card,
its power limit and an SM clock sampled right after the library's steps come from the same run, and
``torch.cuda.max_memory_allocated`` of each library step is reported.  TFLOP/s are algorithmic, from the work the
stage counts from its shapes.  --profile instead takes the per-kernel split of each library step with torch.profiler,
in a run of its own (tracing slows the host).  One JSON line goes to stdout, and to DIR/train_bench_STAGE.json
(DIR/train_bench_STAGE_profile.json under --profile) with --out.
"""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BW = 3.35e12                                      # H100 SXM data-sheet HBM3 bandwidth, bytes/s
SIZE = (60, 108)                                       # feature size of a 240x432 frame
T2T = dict(kernel_size=(7, 7), stride=(3, 3), padding=(3, 3))


# ---- measurement, shared by every stage ----

def _smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def card():
    """The device's name and its power limit in W, read in the process that takes the timings."""
    return torch.cuda.get_device_name(0), _smi("power.limit")


def sm_clock():
    return _smi("clocks.sm")


def reset(grads):
    for t in grads:
        t.grad = None


def time_step(fn, grads, warmup, iters):
    """Median ms of fn over iters calls after warmup calls, or "out of memory"."""
    times = []
    try:
        for i in range(warmup + iters):
            reset(grads)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
    except torch.cuda.OutOfMemoryError:
        reset(grads)
        torch.cuda.empty_cache()
        return "out of memory"
    return statistics.median(times)


@contextlib.contextmanager
def tf32(on):
    """TF32 matmuls and TF32 cuDNN convolutions both on or both off; the previous flags come back on exit."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = on
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def profile_split(fn, grads, warmup):
    """Device ms and launches of each kernel over one call of fn after warmup calls, the heaviest first."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warmup):
        reset(grads)
        fn()
    reset(grads)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {ev.key: {"ms": ev.device_time_total / 1e3, "launches": ev.count}
             for ev in prof.key_averages() if ev.device_time_total > 0}
    return dict(sorted(split.items(), key=lambda kv: -kv[1]["ms"]))


def sort_share(split):
    """The radix sorts' (CUB's) part of a profiled step."""
    total = sum(v["ms"] for v in split.values())
    sort_ms = sum(v["ms"] for k, v in split.items() if "cub::" in k or "Onesweep" in k or "RadixSort" in k)
    return {"sort_ms": sort_ms, "sort_share": sort_ms / total if total else None}


# ---- the stages: build(args, dev) returns (shape fields, {step: (library callable, torch reference callable)},
# ---- the tensors whose gradients are reset, {step: algorithmic FLOPs}, a profile annotation or None) ----

CH = [3, 32, 64, 128, 128, 128, 128]


def torch_discriminator():
    """The reference's layer stack on nn.Conv3d, spectral norm through torch.nn.utils (same state-dict layout)."""
    layers = []
    for i in range(6):
        conv = nn.Conv3d(CH[i], CH[i + 1], (3, 5, 5), (1, 2, 2), padding=1 if i == 0 else (1, 2, 2), bias=i == 5)
        layers.append(nn.utils.spectral_norm(conv) if i < 5 else conv)
        if i < 5:
            layers.append(nn.LeakyReLU(0.2, inplace=True))
    seq = nn.Sequential(*layers)

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv = seq

        def forward(self, xs):
            return self.conv(xs.transpose(1, 2)).transpose(1, 2)
    return Net()


def conv_macs(b, t, h, w):
    """MACs of each discriminator layer's forward conv (= its input gradient's = its weight gradient's)."""
    out = []
    for i in range(6):
        pad = 1 if i == 0 else 2
        h, w = (h + 2 * pad - 5) // 2 + 1, (w + 2 * pad - 5) // 2 + 1
        out.append(b * t * h * w * CH[i + 1] * CH[i] * 75)
    return out


def dis_flops(b, t, h, w):
    """(dis step, gen step) FLOPs.  dis step: two forwards; per backward every weight gradient and the input gradients
    of layers 1..5.  gen step: forward + every input gradient."""
    macs = conv_macs(b, t, h, w)
    return 2 * (2 * sum(macs) + 2 * sum(macs) + 2 * sum(macs[1:])), 2 * sum(macs) + 2 * sum(macs)


def build_dis(a, dev):
    """The Temporal PatchGAN discriminator at the training shape (configs/train_e2fgvi.json: 8 clips of 5 + 3 frames at
240x432 per GPU) against a torch restatement on cuDNN.

* dis step: netD(real), netD(fake), hinge dis_loss, dis_loss.backward() (inputs need no gradient);
* gen step: netD(comp) with a frozen discriminator, hinge gan_loss, d gan_loss / d comp.

TFLOP/s are algorithmic: 2 * MACs of the convolutions the step needs, counted from the shapes."""
    from e2fgvi_b200.loss import AdversarialLoss
    from e2fgvi_b200.model.e2fgvi import Discriminator
    from e2fgvi_b200.synth import synth_dis_state_dict
    shape = (a.batch, a.frames, 3, a.height, a.width)
    g = torch.Generator(device=dev).manual_seed(0)
    real = torch.rand(shape, device=dev, generator=g) * 2 - 1
    fake = torch.rand(shape, device=dev, generator=g) * 2 - 1
    adv = AdversarialLoss("hinge")
    sd = synth_dis_state_dict(0)
    dis_flop, gen_flop = dis_flops(a.batch, a.frames, a.height, a.width)

    def steps(net):
        net.load_state_dict(sd, strict=True)
        net.to(dev).train()
        params = list(net.parameters())

        def dis_step():
            loss = (adv(net(real), True, True) + adv(net(fake), False, True)) / 2
            loss.backward()

        def gen_step():
            for p in params:
                p.requires_grad_(False)
            comp = fake.clone().requires_grad_(True)
            torch.autograd.grad(adv(net(comp), True, False), [comp])
            for p in params:
                p.requires_grad_(True)
        return params, dis_step, gen_step

    ours, ref = steps(Discriminator()), steps(torch_discriminator())
    return ({"shape": list(shape)}, {"dis": (ours[1], ref[1]), "gen": (ours[2], ref[2])}, ours[0] + ref[0],
            {"dis": dis_flop, "gen": gen_flop}, None)


def flow_flop(pairs, hu, wu):
    """2 * MACs of the 7x7 convs: the update and ground-truth forwards, every weight gradient, and the input gradients
    of every conv except the coarsest level's first."""
    from e2fgvi_b200.model.modules.flow_comp import _LEVEL_CONVS
    per_px = sum(ci * co * 49 for ci, co in _LEVEL_CONVS)
    first = _LEVEL_CONVS[0][0] * _LEVEL_CONVS[0][1] * 49
    fwd = sum(pairs * (hu >> k) * (wu >> k) * per_px for k in range(6))
    dgrad = fwd - pairs * (hu >> 5) * (wu >> 5) * first
    return 2 * (2 * fwd + fwd + dgrad)


def build_flow(a, dev):
    """The flow-completion step of train.py at the training shape (configs/train_e2fgvi.json: 8 clips of 5 + 3 frames
at 240x432, 64 (ref, supp) pairs at 64x128 per step) against a torch restatement on cuDNN.

Step: pred = netG.forward_bidirect_flow(masked local frames in [0, 1]) (tracks gradients into update_spynet),
loss = FlowCompletionLoss(pred, ground-truth local frames) (the ground-truth SPyNet under no_grad), loss.backward().
torch runs oracle/restate_flow.py in float32 (F.conv2d, F.grid_sample, autograd).  TFLOP/s are algorithmic: 2 * MACs
of the 7x7 convolutions the step needs, counted from the shapes."""
    from e2fgvi_b200.loss import FlowCompletionLoss
    from e2fgvi_b200.model.generator import InpaintGenerator
    from e2fgvi_b200.model.modules.flow_comp import SPyNet
    from e2fgvi_b200.synth import synth_spynet_state_dict
    from oracle import restate_flow

    class Holder(nn.Module):
        """What InpaintGenerator.forward_bidirect_flow needs of the generator: its update_spynet."""

        def __init__(self):
            super().__init__()
            self.update_spynet = SPyNet()

    g = torch.Generator(device=dev).manual_seed(0)
    shape = (a.batch, a.local, 3, a.height, a.width)
    gt = torch.rand(shape, device=dev, generator=g)
    masked = gt.clone()
    masked[..., a.height // 4: a.height // 2, a.width // 3: a.width // 2] = 0
    upd, fix = synth_spynet_state_dict(0), synth_spynet_state_dict(100)
    h, w = a.height // 4, a.width // 4
    hu, wu = -(-h // 32) * 32, -(-w // 32) * 32
    pairs = 2 * a.batch * (a.local - 1)

    net = Holder().to(dev)
    net.update_spynet.load_state_dict(upd)
    loss_fn = FlowCompletionLoss(pretrained=fix).to(dev)

    def ours():
        pred = InpaintGenerator.forward_bidirect_flow(net, masked)
        loss_fn(pred, gt).backward()

    params = restate_flow.params_from_state_dict(upd, "", dtype=torch.float32, device=dev, requires_grad=True)
    gt_params = restate_flow.params_from_state_dict(fix, "", dtype=torch.float32, device=dev)
    mean, std = upd["mean"].to(dev), upd["std"].to(dev)

    def reference():
        pred = restate_flow.forward_bidirect_flow(params, mean, std, masked)
        restate_flow.flow_completion_loss(gt_params, mean, std, pred, gt).backward()

    grads = list(net.parameters()) + [t for row in params for pair in row for t in pair]
    return ({"shape": list(shape), "pairs": pairs, "working_size": [hu, wu]}, {"flow": (ours, reference)}, grads,
            {"flow": flow_flop(pairs, hu, wu)}, None)


# (cin, cout, stride, groups) of the encoder convs (e2fgvi.py:75-94) and (cin, cout, upsample before) of the decoder's
ENC = ((3, 64, 2, 1), (64, 64, 1, 1), (64, 128, 2, 1), (128, 256, 1, 1), (256, 384, 1, 1),
       (640, 512, 1, 2), (768, 384, 1, 4), (640, 256, 1, 8), (512, 128, 1, 1))
DEC = ((128, 128, True), (128, 64, False), (64, 64, True), (64, 3, False))


def encdec_flops(h, w):
    """(forward, backward) algorithmic FLOPs of one frame: 2 * MACs of each 3x3 conv; the backward is the weight
    gradient of every conv plus the input gradient of every conv but the stem (nothing trains the frames)."""
    fwd = bwd = 0
    for k, (cin, cout, s, g) in enumerate(ENC):
        h, w = (h - 1) // s + 1, (w - 1) // s + 1
        f = 2 * h * w * cout * (cin // g) * 9
        fwd += f
        bwd += f * (2 if k else 1)
    for cin, cout, up in DEC:
        if up:
            h, w = 2 * h, 2 * w
        f = 2 * h * w * cout * cin * 9
        fwd += f
        bwd += 2 * f
    return fwd, bwd


def build_encdec(a, dev):
    """One encoder + decoder training step at the training shape: ``pred = netG.decode(netG.encoder(x))``, L1 against
a target, ``backward()``, against oracle/restate.encoder / decoder on cuDNN float32.  --frames is frames per clip
(5 local + 3 reference in train.py)."""
    from e2fgvi_b200.model.generator import InpaintGenerator
    from oracle import restate
    n = a.clips * a.frames
    fwd, bwd = encdec_flops(a.height, a.width)
    torch.manual_seed(0)
    gen = InpaintGenerator().to(dev)
    x = torch.rand(n, 3, a.height, a.width, device=dev) * 2 - 1
    target = torch.rand(n, 3, a.height, a.width, device=dev) * 2 - 1
    params = [p for k, p in gen.named_parameters() if k.startswith(("encoder.", "decoder."))]
    sd = {k: p for k, p in gen.named_parameters() if k.startswith(("encoder.", "decoder."))}

    def ours():
        F.l1_loss(gen.decode(gen.encoder(x)), target).backward()

    def cudnn():
        F.l1_loss(torch.tanh(restate.decoder(sd, restate.encoder(sd, x))), target).backward()

    return ({"frames": n, "size": [a.height, a.width], "fwd_gflop_per_frame": fwd / 1e9,
             "bwd_gflop_per_frame": bwd / 1e9}, {"encdec": (ours, cudnn)}, params, {"encdec": n * (fwd + bwd)}, None)


FFN_C, HIDDEN, FFN = 128, 512, 1960


def ffn_flops(tokens):
    """(forward, backward) algorithmic FLOPs: 2 * MACs of the four Linears; the backward is every weight gradient plus
    every input gradient but SoftSplit's (the features need no gradient here)."""
    ss = sc = 2 * tokens * FFN_C * 49 * HIDDEN
    ffn = 2 * 2 * tokens * HIDDEN * FFN
    return ss + sc + ffn, 2 * (sc + ffn) + ss


def build_ffn(a, dev):
    """One step of the transformer's dense token path at the training shape: ``sc(ffn(ss(feat)), residual=feat)``, L1
against a target, ``backward()`` into the three modules' parameters, against an fp32 torch restatement (F.unfold /
F.linear / F.fold).  --height and --width are the feature size (240 / 4, 432 / 4)."""
    from e2fgvi_b200.model.modules.tfocal_transformer import FusionFeedForward, SoftComp, SoftSplit
    n = a.clips * a.frames
    size = (a.height, a.width)
    fh, fw = (a.height - 1) // 3 + 1, (a.width - 1) // 3 + 1
    tokens = n * fh * fw
    fwd, bwd = ffn_flops(tokens)
    torch.manual_seed(0)
    ss = SoftSplit(FFN_C, HIDDEN, **T2T).to(dev)
    sc = SoftComp(FFN_C, HIDDEN, size).to(dev)
    ffn = FusionFeedForward(HIDDEN, t2t_params=dict(T2T, output_size=size)).to(dev)
    params = list(ss.parameters()) + list(sc.parameters()) + list(ffn.parameters())
    feat = torch.randn(n, FFN_C, *size, device=dev).contiguous(memory_format=torch.channels_last)
    target = torch.randn(n, FFN_C, *size, device=dev)
    ones = F.fold(torch.ones(1, FFN, fh * fw, device=dev), size, **T2T)      # the feed-forward's 40-channel fold

    def ours():
        tok = ss(feat, a.clips, size)
        x = tok.reshape(a.clips, -1, HIDDEN)
        y = ffn(x, size, residual=x)
        F.l1_loss(sc(y.reshape(tok.shape), a.frames, size, residual=feat), target).backward()

    def torch_fp32():
        tok = F.linear(F.unfold(feat, **T2T).transpose(1, 2), ss.embedding.weight, ss.embedding.bias)
        h = F.linear(tok, ffn.conv1[0].weight, ffn.conv1[0].bias)
        u = F.unfold(F.fold(h.transpose(1, 2), size, **T2T) / ones, **T2T).transpose(1, 2)
        y = F.linear(F.gelu(u), ffn.conv2[1].weight, ffn.conv2[1].bias) + tok
        cols = F.linear(y, sc.embedding.weight, sc.embedding.bias)
        F.l1_loss(F.fold(cols.transpose(1, 2), size, **T2T) + sc.bias + feat, target).backward()

    return ({"tokens": tokens, "size": list(size), "clips": a.clips, "frames": a.frames, "fwd_tflop": fwd / 1e12,
             "bwd_tflop": bwd / 1e12}, {"ffn": (ours, torch_fp32)}, params, {"ffn": fwd + bwd}, None)


ATTN_C, HEADS, WIN, EXP, FOC = 512, 4, (5, 9), (2, 4), (5, 9)


def attn_flops(b, t, h, w):
    """(forward, backward) algorithmic FLOPs: the two Linears (backward: weight and input gradients) and the attention
    products over the reference's key count (duplicated ring tokens merged): the forward is 2 products (S = QK^T,
    PV), the backward 5 (S, dP = dO V^T, dV = P^T dO, dQ = dS K, dK = dS^T Q)."""
    from e2fgvi_b200.ops import attention_flops
    tok, pool = b * t * h * w, b * t * (h // WIN[0]) * (w // WIN[1])
    lin = 2 * (tok + pool) * ATTN_C * 3 * ATTN_C + 2 * tok * ATTN_C * ATTN_C
    att = attention_flops(b, t, h, w, ATTN_C, WIN, EXP, FOC)
    return lin + att, 2 * lin + 2.5 * att


def build_attn(a, dev):
    """One training step of the focal window attention at the training shape: ``WindowAttention.attend(x, pooled)``, L1
against a target, ``backward()`` into qkv, proj, x and pooled, against an fp32 torch restatement (F.linear and the
reference's literal key list, oracle/restate.py).  --height and --width are the token grid's."""
    from e2fgvi_b200.model.modules.tfocal_transformer import WindowAttention, rolled_valid_indices
    from oracle import restate
    b, t, h, w = a.clips, a.frames, a.height, a.width
    fwd, bwd = attn_flops(b, t, h, w)
    torch.manual_seed(0)
    mod = WindowAttention(ATTN_C, EXP, WIN, FOC, 2, HEADS, True, "fc").to(dev)
    x = torch.randn(b, t, h, w, ATTN_C, device=dev, requires_grad=True)
    pooled = torch.randn(b, h // WIN[0], w // WIN[1], t, ATTN_C, device=dev, requires_grad=True)
    target = torch.randn(b, t, h, w, ATTN_C, device=dev)
    valid = rolled_valid_indices(WIN, EXP).to(dev)
    params = list(mod.parameters()) + [x, pooled]

    def ours():
        F.l1_loss(mod.attend(x, pooled), target).backward()

    def torch_fp32():
        qkv = F.linear(x, mod.qkv.weight, mod.qkv.bias)
        qkv_p = F.linear(pooled.permute(0, 3, 1, 2, 4), mod.qkv.weight, mod.qkv.bias)
        with dev:                                      # the restatement builds its pooled mask on the default device
            att = restate.focal_window_attention(qkv, qkv_p, HEADS, WIN, EXP, FOC, mod.scale, valid)
        F.l1_loss(F.linear(att, mod.proj.weight, mod.proj.bias), target).backward()

    return ({"clips": b, "frames": t, "grid": [h, w], "fwd_tflop": fwd / 1e12, "bwd_tflop": bwd / 1e12},
            {"attn": (ours, torch_fp32)}, params, {"attn": fwd + bwd}, None)


BLOCK_C = 512


def block_bytes(b, t, h=20, w=36):
    """Algorithmic bytes of the two LayerNorm backward kernels:
      layernorm_backward_kernel      x, dy, the residual g read, dx1 written fp32 and as the bf16 pair: 5 x rows x 2 KB;
      layernorm_pool_backward_kernel x, [dxn; dpooled], dx1 read, dx written: 4 x rows x 2 KB + pooled rows x 2 KB."""
    rows, pooled = b * t * h * w, b * t * (h // 5) * (w // 9)
    return {"layernorm_backward_kernel": 5 * rows * BLOCK_C * 4,
            "layernorm_pool_backward_kernel": 4 * rows * BLOCK_C * 4 + pooled * BLOCK_C * 4}


def build_block(a, dev):
    """Training steps of the temporal focal transformer at the training shape (8 clips x 8 frames, 60x108 features,
20x36 tokens): one ``TemporalFocalTransformerBlock`` (forward, L1 against a target, ``backward()`` into every parameter
and the tokens) and the eight-block trunk ``sc(transformer(ss(feat)), t, residual=feat)`` (forward, L1, backward into
every trunk parameter and feat), against the fp32 torch autograd of the restatement (oracle/restate.py).  --profile
also gives the LayerNorm backward kernels' achieved bytes/s against the data-sheet 3.35 TB/s."""
    from e2fgvi_b200.model.modules.tfocal_transformer import SoftComp, SoftSplit, TemporalFocalTransformerBlock
    from oracle import restate
    b, t = a.clips, a.frames
    nbytes = block_bytes(b, t)
    torch.manual_seed(0)
    t2t = dict(T2T, output_size=SIZE)
    ss = SoftSplit(128, BLOCK_C, **T2T, t2t_param=t2t).to(dev)
    sc = SoftComp(128, BLOCK_C, SIZE).to(dev)
    blocks = torch.nn.Sequential(*[TemporalFocalTransformerBlock(BLOCK_C, 4, (5, 9), focal_level=2,
                                                                 focal_window=(5, 9), t2t_params=t2t,
                                                                 pool_method="fc")
                                   for _ in range(8)]).to(dev)
    blk = blocks[0]
    x = torch.randn(b, t, 20, 36, BLOCK_C, device=dev, requires_grad=True)
    target = torch.randn(b, t, 20, 36, BLOCK_C, device=dev)
    feat = torch.randn(b * t, 128, *SIZE, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_()
    feat_target = torch.randn(b * t, 128, *SIZE, device=dev)
    sd = {f"transformer.{i}.{k}": v for i, m in enumerate(blocks) for k, v in
          list(m.named_parameters()) + list(m.named_buffers())}
    params = list(blocks.parameters()) + list(ss.parameters()) + list(sc.parameters()) + [x, feat]

    def block_ours():
        F.l1_loss(blk(x), target).backward()

    def block_torch():
        with dev:                                      # the restatement builds its pooled mask on the default device
            F.l1_loss(restate.transformer_block(sd, "transformer.0", x, SIZE), target).backward()

    def trunk_ours():
        F.l1_loss(sc(blocks(ss(feat, b)), t, residual=feat), feat_target).backward()

    def trunk_torch():
        with dev:
            tok = F.linear(F.unfold(feat, **T2T).transpose(1, 2), ss.embedding.weight, ss.embedding.bias)
            tok = tok.reshape(b, t, 20, 36, BLOCK_C)
            for i in range(8):
                tok = restate.transformer_block(sd, f"transformer.{i}", tok, SIZE)
            cols = F.linear(tok.reshape(b * t, -1, BLOCK_C), sc.embedding.weight, sc.embedding.bias)
            img = F.fold(cols.transpose(1, 2), SIZE, **T2T) + sc.bias
            F.l1_loss(img + feat, feat_target).backward()

    def annotate(split):
        out = {}
        for k, nb in nbytes.items():
            hits = [v for name, v in split.items() if k in name]
            if hits:
                us = 1e3 * sum(v["ms"] for v in hits) / sum(v["launches"] for v in hits)
                out[k] = {"us": us, "gb": nb / 1e9, "tb_per_s": nb / (us * 1e-6) / 1e12,
                          "share_of_3.35": nb / (us * 1e-6) / PEAK_BW}
        return out

    return ({"clips": b, "frames": t, "features": list(SIZE), "tokens": [20, 36], "layernorm_bytes": nbytes},
            {"block": (block_ours, block_torch), "trunk": (trunk_ours, trunk_torch)}, params, {}, annotate)


def build_align(a, dev):
    """A training step of one deformable alignment at the training shape (8 clips' frames, 60x108 features, 256 -> 128
channels, 16 deform groups): ``SecondOrderDeformableAlignment.forward`` + L1 against a target + ``backward()`` into x,
extra_feat, both flows and every parameter, against the fp32 torch autograd of the restatement
(oracle/restate.deform_align).  --n is the frames in one call (the training batch's clips).  --profile also gives the
radix sort's share of the step."""
    from e2fgvi_b200.model.modules.feat_prop import SecondOrderDeformableAlignment
    from oracle import restate
    torch.manual_seed(0)
    n, (h, w) = a.n, SIZE
    mod = SecondOrderDeformableAlignment(256, 128, 3, padding=1, deform_groups=16).to(dev)
    torch.nn.init.normal_(mod.conv_offset[-1].weight, std=0.01)       # non-trivial offsets
    x = torch.randn(n, 256, h, w, device=dev, requires_grad=True)
    extra = torch.randn(n, 384, h, w, device=dev, requires_grad=True)
    f1 = (3 * torch.randn(n, 2, h, w, device=dev)).requires_grad_()
    f2 = (3 * torch.randn(n, 2, h, w, device=dev)).requires_grad_()
    target = torch.randn(n, 128, h, w, device=dev)
    sd = {f"m.{k}": v for k, v in mod.named_parameters()}
    params = list(mod.parameters()) + [x, extra, f1, f2]

    def ours():
        F.l1_loss(mod(x, extra, f1, f2), target).backward()

    def torch_ref():
        with dev:                                      # the restatement builds its index tensors on the default device
            F.l1_loss(restate.deform_align(sd, "m", x, extra, f1, f2), target).backward()

    return ({"n": n, "features": list(SIZE), "cin": 256, "cout": 128, "deform_groups": 16},
            {"align": (ours, torch_ref)}, params, {}, sort_share)


def build_prop(a, dev):
    """A training step of the feature propagation at the trainer's shape (8 clips of 5 local frames, 128 channels at
60x108): ``BidirectionalPropagation.forward`` + L1 against a target + ``backward()`` into x, both flow tensors and every
parameter, against the fp32 torch autograd of the restatement (oracle/restate.bidirectional_propagation).  --b is the
clips (the training batch), --t the local frames per clip.  --profile also gives the radix sorts' share of the step."""
    from e2fgvi_b200.model.modules.feat_prop import BidirectionalPropagation
    from oracle import restate
    torch.manual_seed(0)
    b, t, (h, w) = a.b, a.t, SIZE
    mod = BidirectionalPropagation(128).to(dev)
    for name in mod.DIRECTIONS:                                         # non-trivial offsets
        torch.nn.init.normal_(mod.deform_align[name].conv_offset[-1].weight, std=0.01)
    x = torch.randn(b, t, 128, h, w, device=dev, requires_grad=True)
    fb = (2 * torch.randn(b, t - 1, 2, h, w, device=dev)).requires_grad_()
    ff = (2 * torch.randn(b, t - 1, 2, h, w, device=dev)).requires_grad_()
    target = torch.randn(b, t, 128, h, w, device=dev)
    sd = {f"m.{k}": v for k, v in mod.named_parameters()}
    params = list(mod.parameters()) + [x, fb, ff]

    def ours():
        F.l1_loss(mod(x, fb, ff), target).backward()

    def torch_ref():
        with dev:                                      # the restatement builds its index tensors on the default device
            F.l1_loss(restate.bidirectional_propagation(sd, "m", x, fb, ff), target).backward()

    return ({"b": b, "t": t, "features": list(SIZE), "channels": 128}, {"prop": (ours, torch_ref)}, params, {},
            sort_share)


# stage: (build, shape options and their defaults, --iters, --warmup)
STAGES = {
    "dis": (build_dis, dict(batch=8, frames=8, height=240, width=432), 20, 5),
    "flow": (build_flow, dict(batch=8, local=5, height=240, width=432), 20, 5),
    "encdec": (build_encdec, dict(clips=8, frames=8, height=240, width=432), 20, 5),
    "ffn": (build_ffn, dict(clips=8, frames=8, height=60, width=108), 20, 5),
    "attn": (build_attn, dict(clips=8, frames=8, height=20, width=36), 10, 3),
    "block": (build_block, dict(clips=8, frames=8), 10, 3),
    "align": (build_align, dict(n=8), 10, 3),
    "prop": (build_prop, dict(b=8, t=5), 10, 3),
}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="stage", required=True, metavar="STAGE")
    for stage, (build, shape, iters, warmup) in STAGES.items():
        p = sub.add_parser(stage, description=build.__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
        for k, v in shape.items():
            p.add_argument(f"--{k}", type=int, default=v)
        p.add_argument("--iters", type=int, default=iters)
        p.add_argument("--warmup", type=int, default=warmup)
        p.add_argument("--profile", action="store_true", help="per-kernel split of the library's steps instead")
        p.add_argument("--out", default=None, help="directory for the JSON result")
    return ap.parse_args(argv)


def run(a, dev):
    fields, steps, grads, flop, annotate = STAGES[a.stage][0](a, dev)
    name, power = card()
    result = {"stage": a.stage, "card": name, "power_limit_w": power, **fields, "steps": {}}
    if a.profile:
        for step, (ours, _) in steps.items():
            split = profile_split(ours, grads, a.warmup)
            result["steps"][step] = {"profile_total_ms": sum(v["ms"] for v in split.values()), "profile_ms": split,
                                     **(annotate(split) if annotate else {})}
        return result
    for step, (ours, _) in steps.items():
        torch.cuda.reset_peak_memory_stats()
        result["steps"][step] = {"ours_ms": time_step(ours, grads, a.warmup, a.iters),
                                 "ours_max_memory_gb": torch.cuda.max_memory_allocated() / 1e9}
    result["sm_clock_mhz"] = sm_clock()
    for on in (False, True):
        with tf32(on):
            for step, (_, ref) in steps.items():
                result["steps"][step][f"torch_{'tf32' if on else 'fp32'}_ms"] = time_step(ref, grads, a.warmup,
                                                                                         a.iters)
    for step, work in flop.items():
        res = result["steps"][step]
        res["gflop"] = work / 1e9
        for k in ("ours", "torch_fp32", "torch_tf32"):
            if not isinstance(res[k + "_ms"], str):
                res[k + "_tflops"] = work / res[k + "_ms"] / 1e9
    return result


def main(argv=None):
    a = parse_args(argv)
    if not torch.cuda.is_available():
        print(f"train_bench {a.stage}: no CUDA device; nothing was timed", file=sys.stderr)
        return 2
    from e2fgvi_b200 import ops
    try:
        result = run(a, torch.device("cuda:0"))
    finally:
        ops.invalidate_weight_caches()
    print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f"train_bench_{a.stage}" + ("_profile" if a.profile else "") + ".json"),
                  "w") as f:
            json.dump(result, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
