"""Goldens of the generator's training gradients: the unmodified reference run on the CPU with
``synth.synth_state_dict(..., "stress", seed)`` weights, in three precisions.

``python -m oracle.gen_golden_train`` writes ``tests/golden/train_<case>.npz`` and ``tests/golden/train_layout.json``.

Cases (``CASES``):

* ``gen_base``: the base model, b=1, t=2 at 240x432 (its bias map fixes 60x108 features).  With enc = encoder(masked),
  pred = tanh(decoder(enc + sc(transformer(ss(enc, b)), t))): ``InpaintGenerator.forward`` (e2fgvi.py:245-263) with
  the propagation replaced by the identity.  The loss is the trainer's hole + valid L1 terms (core/trainer.py:346-360,
  weights 1 and 1 from configs/train_e2fgvi.json) plus 0.01 x the generator-side hinge loss of a frozen reference
  ``Discriminator`` in eval mode on comp = target * (1 - m) + m * pred (trainer.py:309, :333-337).
* ``gen_hq``: the same chain on the HQ model (``[tokens, output_size]`` calls, ``sc.bias_conv``), b=2, t=3 at 120x216:
  10x18 tokens, so every ring of the focal attention wraps; hole + valid only.
* ``align``: ``feat_prop_module.deform_align.backward_`` alone, n=2 at 60x108 and n=3 at 13x19, flows of a few
  pixels; the loss is the sum of both parts' mean L1 against fixed targets; gradients into x, extra_feat, flow_1,
  flow_2 of each part and the module's 10 parameters.

The inputs are regenerated, not stored: ``clip`` and ``align_inputs`` draw them in float32 from CPU generators (the
precisions below read the same values).  The L1 targets are kept away from the predictions (|target| >= 1.25 against
a tanh output; |target| >= 6 against alignment outputs that stay within +-4, checked here): at an L1's kink a 1e-7
difference in a prediction flips the sign of that element's gradient, and a few such flips move every parameter's
gradient by about 1e-3 relative, more than any arithmetic difference the goldens are meant to expose.

Three runs per case:

* ``G64``: the reference in float64, the golden;
* ``G32``: the reference in float32 on the CPU.  Its distance from G64 is the cost of fp32 arithmetic (LeakyReLU
  decisions near 0 included), a yardstick;
* ``G16``: float64 with the library's operand policy imposed from outside, no reference source touched.  Every
  ``nn.Conv2d``, ``nn.Linear`` and ``nn.Conv3d`` but the window pooling's computes its output as the kernels do, from
  bf16 (hi, lo) splits of its input and weight with the lo x lo product dropped (about 16 significand bits: the offset
  head's offsets, and so the alignment's bilinear slopes, move about 100 times more than in fp32); every block's
  ``attn.qkv`` output, the attention's probabilities and its output (``attn.proj``'s input) are rounded to fp16; in the
  alignment x is rounded to fp16 and ``weight`` is loaded rounded to fp16 (INTEGRATION.md: gradients "at the kernels'
  fp16 qkv", "x and ``weight`` read through fp16").  The roundings pass the gradient through unchanged, as the kernels'
  backward does.  Its distance from G64 is the cost of that policy, the second yardstick.  (The window pooling runs
  in fp32 registers next to the LayerNorm; the DCN's fp16 samples move only its output, which no gradient of these
  losses reads.)

Stored per case, for every parameter that receives a gradient (``p:<name>``) and every input gradient
(``in:<name>``): ``P64/<n>``, ``P32/<n>``, ``P16/<n>``, the gradient's projections on 8 fixed unit vectors
(``gen_golden_dis.projections(<n>, numel, seed)``); ``max/<n>``, G64's max-abs value; for tensors of at most 4096
elements ``full/<n>``, G64's gradient (float32), and ``dev/<n>``, the largest element-wise distance of G32 or G16 from
G64.  Also ``loss64`` / ``loss32`` / ``loss16``, ``out64``, a strided subsample of G64's prediction (float32), and
``params``, the names of the parameters that received a gradient.

Importing this module does not touch the reference; only ``run_case`` and ``layout`` do.
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from e2fgvi_b200.synth import synth_dis_state_dict, synth_state_dict  # noqa: E402
from oracle import reference_loader  # noqa: E402
from oracle.gen_golden_dis import projections  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = {
    "gen_base": dict(kind="gen", hq=False, b=1, t=2, h=240, w=432, gan=True, seed=0),
    "gen_hq": dict(kind="gen", hq=True, b=2, t=3, h=120, w=216, gan=False, seed=1),
    "align": dict(kind="align", parts=((2, 60, 108), (3, 13, 19)), seed=2),
}
ALIGN = "feat_prop_module.deform_align.backward_"
HOLE_WEIGHT, VALID_WEIGHT, ADVERSARIAL_WEIGHT = 1.0, 1.0, 0.01       # configs/train_e2fgvi.json
FULL = 4096            # gradients of at most this many elements are stored whole
OUT_STRIDE = 8         # the prediction's subsample: every 8th row and column


# ------------------------------------------------------------------------------------------------------ inputs
def clip(name):
    """(masked, masks, targets) of a generator case, float32: masked = frames * (1 - masks) with frames in [-1, 1]
    (a smooth moving pattern plus noise), masks (b, t, 1, h, w) in {0, 1} (a rectangle per frame), and L1 targets
    of magnitude 1.25 to 1.75 with random signs."""
    c = CASES[name]
    b, t, h, w, seed = c["b"], c["t"], c["h"], c["w"], c["seed"]
    g = torch.Generator().manual_seed(3000 + seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, h), torch.linspace(0, 1, w), indexing="ij")
    frames = torch.empty(b, t, 3, h, w)
    for bi in range(b):
        for j in range(t):
            for ch in range(3):
                ph = 0.7 * ch + 0.9 * bi + 0.15 * j
                frames[bi, j, ch] = 0.8 * torch.sin(9 * xx + 5 * yy + ph) * torch.cos(6 * yy - 3 * xx + 2 * ph)
    frames = (frames + 0.2 * torch.rand(frames.shape, generator=g) - 0.1).clamp(-1, 1)
    masks = torch.zeros(b, t, 1, h, w)
    for bi in range(b):
        for j in range(t):
            y0, x0 = h // 4 + 3 * j + 5 * bi, w // 3 + 5 * j
            masks[bi, j, :, y0: y0 + h // 3, x0: x0 + w // 4] = 1
    sign = torch.where(torch.rand(frames.shape, generator=g) < 0.5, -1.0, 1.0)
    targets = sign * (1.25 + 0.5 * torch.rand(frames.shape, generator=g))
    return frames * (1 - masks), masks, targets


def align_inputs(name):
    """Per part of an alignment case, (x (n, 256, h, w), extra_feat (n, 384, h, w), flow_1, flow_2 (n, 2, h, w),
    target (n, 128, h, w)), float32: unit-variance features, flows of about 2 pixels and targets of magnitude 6 to 7
    with random signs."""
    c = CASES[name]
    out = []
    for k, (n, h, w) in enumerate(c["parts"]):
        g = torch.Generator().manual_seed(4000 + 10 * c["seed"] + k)
        x = torch.randn(n, 256, h, w, generator=g)
        extra = torch.randn(n, 384, h, w, generator=g)
        f1, f2 = (2 * torch.randn(n, 2, h, w, generator=g) for _ in range(2))
        sign = torch.where(torch.rand(n, 128, h, w, generator=g) < 0.5, -1.0, 1.0)
        target = sign * (6 + torch.rand(n, 128, h, w, generator=g))
        out.append((x, extra, f1, f2, target))
    return out


def weights(name, model):
    """The case's generator state dict for ``model`` (the reference's or the library's: the same keys give the same
    values) and, for ``gen_base``, the discriminator's."""
    c = CASES[name]
    return synth_state_dict(model, "stress", c["seed"]), synth_dis_state_dict(c["seed"])


def generator_loss(pred, masks, targets, dis_out=None):
    """The trainer's generator loss (core/trainer.py:333-360): hole + valid L1 terms and, with ``dis_out`` = netD(comp),
    the adversarial weight x the generator-side hinge loss.  pred (b, t, 3, h, w)."""
    hole = F.l1_loss(pred * masks, targets * masks) / torch.mean(masks) * HOLE_WEIGHT
    valid = F.l1_loss(pred * (1 - masks), targets * (1 - masks)) / torch.mean(1 - masks) * VALID_WEIGHT
    loss = hole + valid
    if dis_out is not None:
        loss = loss + (-dis_out).mean() * ADVERSARIAL_WEIGHT
    return loss


def composite(pred, masks, targets):
    """comp_imgs of trainer.py:309."""
    return targets * (1 - masks) + masks * pred


def align_loss(outs, targets):
    return sum(F.l1_loss(o, tg) for o, tg in zip(outs, targets))


# ------------------------------------------------------------------------------------------------------ reference
def _round_fp16(t):
    """t read through fp16, with the gradient passed through unchanged."""
    return t + (t.half().to(t.dtype) - t).detach()


def _split(t):
    """The bf16 (hi, lo) pair the kernels read for an fp32 operand t, as t's dtype."""
    hi = t.to(torch.bfloat16).to(t.dtype)
    return hi, (t - hi).to(torch.bfloat16).to(t.dtype)


def _three_term(m, inputs, out):
    """Forward hook: the module's output from split operands, hi.hi + hi.lo + lo.hi (bias added once), with the
    gradient of the exact output."""
    x = inputs[0]
    (xh, xl), (wh, wl) = _split(x.detach()), _split(m.weight.detach())
    if isinstance(m, nn.Linear):
        f = F.linear
    else:
        def f(a, b):
            return m._conv_forward(a, b, None)
    y = f(xh, wh) + f(xh, wl) + f(xl, wh)
    if m.bias is not None:
        y = y + (m.bias.view(-1, *([1] * (y.dim() - 2))) if not isinstance(m, nn.Linear) else m.bias).detach()
    return out + (y - out).detach()


def _operand_policy(net, pool=()):
    """G16's hooks on ``net``'s convs and Linears (but the modules in ``pool``) and its attention."""
    skip = {id(m) for m in pool}
    for m in net.modules():
        if isinstance(m, (nn.Conv2d, nn.Linear, nn.Conv3d)) and id(m) not in skip:
            m.register_forward_hook(_three_term)
    for m in net.modules():
        if hasattr(m, "qkv") and hasattr(m, "proj") and hasattr(m, "softmax"):
            m.qkv.register_forward_hook(lambda mod, i, o: _round_fp16(o))
            m.softmax.register_forward_hook(lambda mod, i, o: _round_fp16(o))
            m.proj.register_forward_pre_hook(lambda mod, args: (_round_fp16(args[0]),) + tuple(args[1:]))


def _reference(hq):
    return reference_loader.import_reference("model.e2fgvi_hq" if hq else "model.e2fgvi")


def _run_gen(name, prec):
    c = CASES[name]
    b, t, h, w, hq = c["b"], c["t"], c["h"], c["w"], c["hq"]
    ref = _reference(hq)
    net = ref.InpaintGenerator()
    sd, dsd = weights(name, net)
    net.load_state_dict(sd, strict=True)
    dt = torch.float32 if prec == "32" else torch.float64
    net = net.to(dt).train()
    if prec == "16":
        _operand_policy(net, [blk.pool_layers[0] for blk in net.transformer])
    masked, masks, targets = (v.to(dt) for v in clip(name))
    enc = net.encoder(masked.view(b * t, 3, h, w))
    _, ch, fh, fw = enc.shape
    if hq:
        tok = net.ss(enc, b, (fh, fw))
        tok = net.transformer([tok, (fh, fw)])[0]
        feat = net.sc(tok, t, (fh, fw))
    else:
        tok = net.transformer(net.ss(enc, b))
        feat = net.sc(tok, t)
    pred = torch.tanh(net.decoder(enc + feat)).view(b, t, 3, h, w)
    dis_out = None
    if c["gan"]:
        dis = ref.Discriminator().to(dt)
        dis.load_state_dict({k: v.to(dt) for k, v in dsd.items()}, strict=True)
        dis.eval().requires_grad_(False)
        if prec == "16":
            _operand_policy(dis)
        dis_out = dis(composite(pred, masks, targets))
    loss = generator_loss(pred, masks, targets, dis_out)
    loss.backward()
    grads = {"p:" + k: p.grad.double() for k, p in net.named_parameters() if p.grad is not None}
    return loss.item(), pred.detach().double()[..., ::OUT_STRIDE, ::OUT_STRIDE], grads


def _run_align(name, prec):
    ref = _reference(False)
    net = ref.InpaintGenerator()
    sd, _ = weights(name, net)
    net.load_state_dict(sd, strict=True)
    mod = net.feat_prop_module.deform_align["backward_"]
    dt = torch.float32 if prec == "32" else torch.float64
    mod = mod.to(dt)
    if prec == "16":
        with torch.no_grad():
            mod.weight.copy_(mod.weight.half().to(dt))
        mod.register_forward_pre_hook(lambda m, args: (_round_fp16(args[0]),) + tuple(args[1:]))
        _operand_policy(mod.conv_offset)
    leaves, outs, targets = {}, [], []
    for k, part in enumerate(align_inputs(name)):
        x, extra, f1, f2, target = (v.to(dt) for v in part)
        for nm, v in (("x", x), ("extra_feat", extra), ("flow_1", f1), ("flow_2", f2)):
            leaves[f"in:{nm}.{k}"] = v.requires_grad_(True)
        outs.append(mod(x, extra, f1, f2))
        targets.append(target)
    margin = min((o.detach() - tg).abs().min().item() for o, tg in zip(outs, targets))
    assert margin > 1.0, f"an alignment output comes within {margin} of its L1 target"
    loss = align_loss(outs, targets)
    loss.backward()
    grads = {"p:" + ALIGN + "." + k: p.grad.double() for k, p in mod.named_parameters() if p.grad is not None}
    grads.update({k: v.grad.double() for k, v in leaves.items()})
    return loss.item(), outs[0].detach().double()[..., ::OUT_STRIDE, ::OUT_STRIDE], grads


def run_case(name):
    c = CASES[name]
    run = _run_gen if c["kind"] == "gen" else _run_align
    runs = {prec: run(name, prec) for prec in ("64", "32", "16")}
    g64 = runs["64"][2]
    res = {"out64": runs["64"][1].float().numpy(),
           "params": np.array(sorted(k[2:] for k in g64 if k.startswith("p:")))}
    for prec, (loss, _, grads) in runs.items():
        res["loss" + prec] = np.float64(loss)
        assert grads.keys() == g64.keys(), prec
    for k, d in g64.items():
        P = projections(k, d.numel(), c["seed"])
        for prec, (_, _, grads) in runs.items():
            res[f"P{prec}/{k}"] = (P @ grads[k].reshape(-1)).numpy()
        del P
        res["max/" + k] = np.float64(d.abs().max().item())
        if d.numel() <= FULL:
            res["full/" + k] = d.float().numpy()
            res["dev/" + k] = np.float64(max((runs[p][2][k] - d).abs().max().item() for p in ("32", "16")))
    np.savez_compressed(os.path.join(GOLDEN, f"train_{name}.npz"), **res)
    return res


def layout():
    """The reference's parameter names and shapes of the trained parts: the trunk (encoder, ss, transformer, sc,
    decoder) of both models and the alignment module."""
    out = {}
    trunk = ("encoder.", "ss.", "transformer.", "sc.", "decoder.")
    for key, hq in (("base", False), ("hq", True)):
        net = _reference(hq).InpaintGenerator()
        out[key] = [[k, list(p.shape)] for k, p in net.named_parameters() if k.startswith(trunk)]
        if not hq:
            out["align"] = [[k, list(p.shape)] for k, p in net.named_parameters() if k.startswith(ALIGN + ".")]
    with open(os.path.join(GOLDEN, "train_layout.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    torch.manual_seed(0)
    layout()
    for name in sys.argv[1:] or CASES:
        run_case(name)
        print("wrote", name)
