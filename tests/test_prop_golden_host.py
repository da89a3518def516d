"""CPU: the float64 restatement of the feature propagation (``oracle/restate.bidirectional_propagation``), which the GPU
propagation tests lean on, against the unmodified reference's gradient golden (``oracle/gen_golden_prop.py``), and the
golden's own sanity.

Autograd of the restatement reproduces the reference's float64 loss and every gradient of the small part (b = 2, t = 3
at 13x19) to about 1e-9: a misreading shared by the restatement and the backward (the flow index of either sweep, the
second-order flow composition, the fusion's source order) fails here.  The large part (60x108) is left out: restating
it takes minutes on the CPU, and it runs the same functions."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import restate
from oracle.gen_golden_dis import projections
from oracle.gen_golden_prop import PARTS, PROP, SEED, prop_inputs, prop_loss, prop_weights

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _gold():
    return np.load(os.path.join(GOLDEN, "train_prop.npz"))


def _get(gold, part, key):
    return gold[f"{part}/{key}"]


def _model():
    return importlib.import_module("model.e2fgvi").InpaintGenerator(init_weights=False)


def test_restatement_gradients_equal_the_reference():
    gold, part = _gold(), "small"
    sd = {f"{PROP}.{k}": v.double().requires_grad_(True) for k, v in prop_weights(_model()).items()}
    x, fb, ff, target = (v.double() for v in prop_inputs(part))
    leaves = {"p:" + k: v for k, v in sd.items()}
    for nm, v in (("x", x), ("flows_backward", fb), ("flows_forward", ff)):
        leaves["in:" + nm] = v.requires_grad_(True)
    out = restate.bidirectional_propagation(sd, PROP, x, fb, ff)
    loss = prop_loss(out, target)
    names = list(leaves)
    grads = dict(zip(names, torch.autograd.grad(loss, [leaves[k] for k in names])))
    l64 = float(_get(gold, part, "loss64"))
    assert abs(loss.item() - l64) <= 1e-12 * abs(l64)
    want_out = torch.from_numpy(_get(gold, part, "out64")).double()
    assert (out.detach()[..., ::8, ::8] - want_out).abs().max().item() <= 1e-6 * want_out.abs().max().item()
    assert sorted(grads) == sorted(k[len(part) + 5:] for k in gold.files if k.startswith(f"{part}/P64/"))
    errs = {}
    for k, g in grads.items():
        want = torch.from_numpy(_get(gold, part, "P64/" + k))
        errs[k] = ((projections(k, g.numel(), SEED) @ g.reshape(-1) - want).norm() / want.norm()).item()
        assert g.abs().max().item() == pytest.approx(float(_get(gold, part, "max/" + k)), rel=1e-9), k
        if f"{part}/full/{k}" in gold.files:
            full = torch.from_numpy(_get(gold, part, "full/" + k)).double()
            assert ((g - full).abs() <= 2 ** -23 * g.abs() + 1e-12 * full.abs().max()).all(), k
    assert max(errs.values()) < 1e-9, {k: v for k, v in errs.items() if v >= 1e-9}


@pytest.mark.parametrize("part", list(PARTS))
def test_golden_is_sane(part):
    """The parameters that receive a gradient are the propagation's 30, and both yardsticks are below 0.1 relative, the
    G32 one nonzero (G16's is zero for the fusion's bias, whose gradient the policy's roundings do not reach).  The largest, G16's 5.7e-2 for the 60x108 part's backward_ ``conv_offset.4.bias``, is a sum over every
    pixel that cancels; G16's split operands move the offsets and so flip many LeakyReLU and bilinear-cell decisions
    inside it."""
    gold = _gold()
    params = sorted(f"{PROP}.{k}" for k, _ in _model().feat_prop_module.named_parameters())
    assert len(params) == 30
    assert sorted(_get(gold, part, "params").tolist()) == params
    assert all(float(_get(gold, part, f"loss{p}")) != float(_get(gold, part, "loss64")) for p in ("32", "16"))
    for k in (k[len(part) + 5:] for k in gold.files if k.startswith(f"{part}/P64/")):
        p64 = _get(gold, part, "P64/" + k)
        r = {p: np.linalg.norm(_get(gold, part, f"P{p}/{k}") - p64) / np.linalg.norm(p64) for p in ("32", "16")}
        assert 0 < r["32"] < 0.1 and r["16"] < 0.1, (k, r)
