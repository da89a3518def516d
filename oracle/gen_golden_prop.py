"""Goldens of the feature propagation's training gradients: the unmodified reference's ``BidirectionalPropagation``
(``feat_prop_module`` of the base ``InpaintGenerator``) run on the CPU with ``synth.synth_state_dict(..., "stress",
seed)`` weights, in the three precisions of ``oracle/gen_golden_train.py``, whose helpers this module uses.

``python -m oracle.gen_golden_prop`` writes ``tests/golden/train_prop.npz``.

Two parts, each its own forward, loss and backward (``PARTS``):

* ``large``: b = 1, t = 5 at 60x108 (the trainer's local frames at the base model's feature size);
* ``small``: b = 2, t = 3 at 13x19.

Inputs (``prop_inputs``), float32 from CPU generators: x (b, t, 128, h, w) of unit variance, both flow tensors
(b, t-1, 2, h, w) of about 2 pixels, and L1 targets of magnitude ``TARGET`` to ``TARGET`` + 1 with random signs, which
the outputs stay well away from (checked here), so that no element's gradient sign rests on a 1e-7 difference.  The
loss is the mean L1; gradients go into x, both flow tensors and the module's 30 parameters.

G64 is the golden; G32 (float32) and G16 (float64 under the library's operand policy: bf16 split operands with three
products in every conv, the DCNs' x and ``weight`` read through fp16) are the yardsticks.  Stored per part, under the
prefix ``<part>/``, with the key scheme of ``gen_golden_train.run_case``: ``P64/<n>``, ``P32/<n>``, ``P16/<n>``,
``max/<n>``, ``full/<n>`` and ``dev/<n>`` for tensors of at most 4096 elements, ``loss64`` / ``loss32`` / ``loss16``,
``out64`` (a strided subsample of G64's output) and ``params``.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from e2fgvi_b200.synth import synth_state_dict  # noqa: E402
from oracle.gen_golden_dis import projections  # noqa: E402
from oracle.gen_golden_train import FULL, GOLDEN, OUT_STRIDE, _operand_policy, _reference, _round_fp16  # noqa: E402

PROP = "feat_prop_module"
PARTS = {"large": dict(b=1, t=5, h=60, w=108, seed=5), "small": dict(b=2, t=3, h=13, w=19, seed=6)}
TARGET = 30.0
SEED = 5               # weights: synth_state_dict(..., "stress", SEED); projections: gen_golden_dis.projections(.., SEED)


def prop_inputs(part):
    """(x, flows_backward, flows_forward, target), float32."""
    p = PARTS[part]
    b, t, h, w = p["b"], p["t"], p["h"], p["w"]
    g = torch.Generator().manual_seed(5000 + p["seed"])
    x = torch.randn(b, t, 128, h, w, generator=g)
    fb, ff = (2 * torch.randn(b, t - 1, 2, h, w, generator=g) for _ in range(2))
    sign = torch.where(torch.rand(b, t, 128, h, w, generator=g) < 0.5, -1.0, 1.0)
    return x, fb, ff, sign * (TARGET + torch.rand(b, t, 128, h, w, generator=g))


def prop_weights(model):
    """The propagation's parameters of ``synth_state_dict(model, "stress", SEED)`` (the reference's or the library's
    generator: the same keys give the same values), keys without the ``feat_prop_module.`` prefix."""
    sd = synth_state_dict(model, "stress", SEED)
    return {k[len(PROP) + 1:]: v for k, v in sd.items() if k.startswith(PROP + ".")}


def prop_loss(out, target):
    return F.l1_loss(out, target)


def _run(part, prec):
    net = _reference(False).InpaintGenerator()
    mod = net.feat_prop_module
    mod.load_state_dict(prop_weights(net), strict=True)
    dt = torch.float32 if prec == "32" else torch.float64
    mod = mod.to(dt)
    if prec == "16":
        aligns = list(mod.deform_align.values())
        for a in aligns:
            with torch.no_grad():
                a.weight.copy_(a.weight.half().to(dt))
            a.register_forward_pre_hook(lambda m, args: (_round_fp16(args[0]),) + tuple(args[1:]))
        _operand_policy(mod, aligns)
    x, fb, ff, target = (v.to(dt) for v in prop_inputs(part))
    leaves = {"in:x": x.requires_grad_(True), "in:flows_backward": fb.requires_grad_(True),
              "in:flows_forward": ff.requires_grad_(True)}
    out = mod(x, fb, ff)
    margin = (out.detach() - target).abs().min().item()
    assert margin > 1.0, f"a propagation output comes within {margin} of its L1 target"
    loss = prop_loss(out, target)
    loss.backward()
    grads = {"p:" + PROP + "." + k: p.grad.double() for k, p in mod.named_parameters() if p.grad is not None}
    grads.update({k: v.grad.double() for k, v in leaves.items()})
    return loss.item(), out.detach().double()[..., ::OUT_STRIDE, ::OUT_STRIDE], grads


def run_part(part):
    runs = {prec: _run(part, prec) for prec in ("64", "32", "16")}
    g64 = runs["64"][2]
    res = {"out64": runs["64"][1].float().numpy(),
           "params": np.array(sorted(k[2:] for k in g64 if k.startswith("p:")))}
    for prec, (loss, _, grads) in runs.items():
        res["loss" + prec] = np.float64(loss)
        assert grads.keys() == g64.keys(), prec
    for k, d in g64.items():
        P = projections(k, d.numel(), SEED)
        for prec, (_, _, grads) in runs.items():
            res[f"P{prec}/{k}"] = (P @ grads[k].reshape(-1)).numpy()
        del P
        res["max/" + k] = np.float64(d.abs().max().item())
        if d.numel() <= FULL:
            res["full/" + k] = d.float().numpy()
            res["dev/" + k] = np.float64(max((runs[p][2][k] - d).abs().max().item() for p in ("32", "16")))
    return {f"{part}/{k}": v for k, v in res.items()}


if __name__ == "__main__":
    torch.manual_seed(0)
    out = {}
    for part in PARTS:
        out.update(run_part(part))
        print("done", part, flush=True)
    np.savez_compressed(os.path.join(GOLDEN, "train_prop.npz"), **out)
