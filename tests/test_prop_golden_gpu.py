"""H100: the feature propagation's training gradients against the unmodified reference (``oracle/gen_golden_prop.py``).

The golden's weights (``synth_state_dict(..., "stress", SEED)``) and inputs (``prop_inputs``) through the library's
``BidirectionalPropagation.forward``, the mean L1 loss and ``backward()``.  Per part (60x108 with b = 1, t = 5 and 13x19
with b = 2, t = 3): a second forward and backward give the same bits; the tensors that receive a gradient are the
reference's; the loss is within K times the G32 yardstick of G64 plus two fp32 ulps of it (a mean of up to 4M L1
terms, which the GPU reduces in another order: G32 may land closer than the result's own rounding) and the output within 2e-3 of its largest value; every
parameter, x and flow gradient passes test_train_golden_gpu.py's bound, imported from there:

    e <= K * max(y32, y16) + TAU * ||P G64||,

with e, y32, y16 the distances of ours, G32 and G16 from G64 seen through the golden's 8 projections (its docstring
derives K = 8 and TAU).  Tensors of at most 4096 elements are also held element by element to K * dev + TAU * max|G64|.
Ratios e / max(y32, y16) are printed per part (``-s``)."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle.gen_golden_dis import projections
from oracle.gen_golden_prop import PARTS, PROP, SEED, prop_inputs, prop_loss, prop_weights
from test_train_golden_gpu import K, TAU

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")

# Tensors whose bound is reported but not asserted, each with its measured ratio and reason.  Everything else is held.
UNBOUNDED = {}


def _step(cuda, part):
    g = importlib.import_module("model.e2fgvi").InpaintGenerator(init_weights=False)
    mod = g.feat_prop_module
    mod.load_state_dict(prop_weights(g), strict=True)
    mod = mod.to(cuda)
    x, fb, ff, target = (v.to(cuda) for v in prop_inputs(part))

    def step():
        mod.zero_grad(set_to_none=True)
        leaves = {"in:x": x.clone().requires_grad_(True), "in:flows_backward": fb.clone().requires_grad_(True),
                  "in:flows_forward": ff.clone().requires_grad_(True)}
        out = mod(leaves["in:x"], leaves["in:flows_backward"], leaves["in:flows_forward"])
        loss = prop_loss(out, target)
        loss.backward()
        grads = {f"p:{PROP}.{k}": p.grad.detach().clone() for k, p in mod.named_parameters() if p.grad is not None}
        grads.update({k: v.grad.detach().clone() for k, v in leaves.items()})
        return loss.item(), out.detach()[..., ::8, ::8], grads
    return step


@pytest.mark.parametrize("part", list(PARTS))
def test_gradients_against_reference_golden(cuda, part):
    gold = np.load(os.path.join(GOLDEN, "train_prop.npz"))

    def get(key):
        return gold[f"{part}/{key}"]
    step = _step(cuda, part)
    loss, out, grads = step()
    _, _, again = step()
    assert sorted(again) == sorted(grads)
    for k, gr in grads.items():
        assert torch.equal(gr, again[k]), k
    assert sorted(k[2:] for k in grads if k.startswith("p:")) == sorted(get("params").tolist())
    assert sorted(grads) == sorted(k[len(part) + 5:] for k in gold.files if k.startswith(f"{part}/P64/"))
    l64 = float(get("loss64"))
    assert abs(loss - l64) <= K * abs(float(get("loss32")) - l64) + 2 * float(np.spacing(np.float32(l64))), (loss, l64)
    want = torch.from_numpy(get("out64")).double()
    assert (out.double().cpu() - want).abs().max().item() < 2e-3 * want.abs().max().item()

    ratios, bad = {}, {}
    for k, gr in grads.items():
        gd = gr.double().cpu()
        p64 = torch.from_numpy(get("P64/" + k))
        y = max((torch.from_numpy(get(f"P{p}/{k}")) - p64).norm().item() for p in ("32", "16"))
        e = (projections(k, gd.numel(), SEED) @ gd.reshape(-1) - p64).norm().item()
        ratios[k] = e / y
        if k in UNBOUNDED:
            continue
        if e > K * y + TAU * p64.norm().item():
            bad[k] = f"e {e:.3e}, yardstick {y:.3e}, ratio {e / y:.2f}, |P G64| {p64.norm().item():.3e}"
        if f"{part}/full/{k}" in gold.files:
            full = torch.from_numpy(get("full/" + k)).double()
            bound = K * float(get("dev/" + k)) + TAU * full.abs().max().item()
            over = (gd - full).abs().max().item()
            if over > bound:
                bad[k + " (elements)"] = f"max error {over:.3e}, bound {bound:.3e}"
    top = sorted(ratios.items(), key=lambda kv: -kv[1])[:5]
    print(f"\n{part}: loss {loss:.9g} (G64 {l64:.9g}); e / yardstick: median {np.median(list(ratios.values())):.2f}, "
          "largest " + ", ".join(f"{k} {v:.2f}" for k, v in top))
    for k, v in bad.items():
        print(f"  over the bound: {k}: {v}")
    assert not bad, bad
