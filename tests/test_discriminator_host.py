"""Discriminator checks that need no GPU: state-dict layout, strict loading, the float64 restatement against the
reference goldens, the losses, and argument checking of the C ABI."""
import json
import os

import numpy as np
import pytest
import torch

from e2fgvi_b200 import synth
from e2fgvi_b200.loss import AdversarialLoss
from e2fgvi_b200.model.e2fgvi import Discriminator
from e2fgvi_b200.model.e2fgvi_hq import Discriminator as DiscriminatorHQ
from oracle import restate_dis
from oracle.gen_golden_dis import CASES, clips, projections

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _layout():
    with open(os.path.join(GOLDEN, "dis_layout.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("sn", [True, False])
def test_layout_matches_reference(sn):
    want = _layout()["spectral_norm" if sn else "plain"]
    got = [[k, list(v.shape)] for k, v in Discriminator(use_spectral_norm=sn).state_dict().items()]
    assert got == want
    assert DiscriminatorHQ is Discriminator


@pytest.mark.parametrize("sn", [True, False])
def test_golden_layout_loads_strictly(sn):
    sd = {k: torch.full(s, 0.5) for k, s in _layout()["spectral_norm" if sn else "plain"]}
    net = Discriminator(use_spectral_norm=sn)
    net.load_state_dict(sd, strict=True)
    assert all(torch.equal(v, sd[k]) for k, v in net.state_dict().items())


def test_init_weights():
    torch.manual_seed(0)
    net = Discriminator(init_weights=False)
    net.init_weights("normal", 0.02)                   # BaseNetwork's signature, through the weight_orig alias
    w = net.conv[2].weight_orig
    assert abs(w.std().item() - 0.02) < 0.002 and abs(w.mean().item()) < 0.002
    assert torch.equal(net.conv[10].bias, torch.zeros(128))
    plain = Discriminator(use_spectral_norm=False)
    assert all(torch.equal(plain.conv[2 * i].bias, torch.zeros(plain.conv[2 * i].bias.shape)) for i in range(6))


@pytest.mark.parametrize("case", list(CASES))
def test_restatement_matches_reference_goldens(case):
    b, t, h, w, sig, sn, seed = CASES[case]
    g = np.load(os.path.join(GOLDEN, f"dis_{case}.npz"))
    params = {k: v.double() for k, v in synth.synth_dis_state_dict(seed, use_spectral_norm=sn).items()}
    real, fake = clips(b, t, h, w, seed)
    with torch.no_grad():
        np.testing.assert_allclose(restate_dis.forward(dict(params), real, False, sig, sn).numpy(), g["eval_out"],
                                   rtol=0, atol=1e-12)
    for k in params:
        if k.endswith(("weight_orig", "weight", "bias")):
            params[k].requires_grad_(True)
    real_clip = restate_dis.forward(params, real, True, sig, sn)
    for k in [k for k in params if k.endswith("_u")]:
        np.testing.assert_allclose(params[k].numpy(), g["u1_" + k[:-2]], rtol=0, atol=1e-12)
    fake_clip = restate_dis.forward(params, fake, True, sig, sn)
    for k in [k for k in params if k.endswith("_u")]:
        np.testing.assert_allclose(params[k].numpy(), g["u2_" + k[:-2]], rtol=0, atol=1e-12)
        np.testing.assert_allclose(params[k[:-2] + "_v"].numpy(), g["v2_" + k[:-2]], rtol=0, atol=1e-12)
    np.testing.assert_allclose(real_clip.detach().numpy(), g["out_real"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(fake_clip.detach().numpy(), g["out_fake"], rtol=0, atol=1e-12)
    dis_loss = (restate_dis.hinge(real_clip, True, True) + restate_dis.hinge(fake_clip, False, True)) / 2
    names = [k for k in params if params[k].requires_grad]
    gd = torch.autograd.grad(dis_loss, [params[k] for k in names])
    comp = fake.clone().requires_grad_(True)
    gan_loss = restate_dis.hinge(restate_dis.forward(params, comp, True, sig, sn), True, False)
    gg = torch.autograd.grad(gan_loss, [comp] + [params[k] for k in names])
    assert abs(dis_loss.item() - g["dis_loss"]) < 1e-12 and abs(gan_loss.item() - g["gan_loss"]) < 1e-12
    np.testing.assert_allclose(gg[0].float().numpy(), g["gin"], rtol=1e-6, atol=1e-12)
    for k, d, e in zip(names, gd, gg[1:]):
        P = projections(k, d.numel(), seed)
        np.testing.assert_allclose((P @ d.reshape(-1)).numpy(), g["gd_" + k], rtol=1e-9, atol=1e-15)
        np.testing.assert_allclose((P @ e.reshape(-1)).numpy(), g["gg_" + k], rtol=1e-9, atol=1e-15)


def test_adversarial_loss_semantics():
    out = torch.tensor([[-2.0, -0.5, 0.3, 1.5]])
    hinge = AdversarialLoss("hinge")
    assert torch.isclose(hinge(out, True, True), torch.relu(1 - out).mean())
    assert torch.isclose(hinge(out, False, True), torch.relu(1 + out).mean())
    assert torch.isclose(hinge(out, True, False), -out.mean())
    p = torch.sigmoid(out)
    ns = AdversarialLoss("nsgan")
    assert torch.isclose(ns(p, True), torch.nn.functional.binary_cross_entropy(p, torch.ones_like(p)))
    assert torch.isclose(ns(p, False, True), torch.nn.functional.binary_cross_entropy(p, torch.zeros_like(p)))
    ls = AdversarialLoss("lsgan")
    assert torch.isclose(ls(out, True), ((out - 1) ** 2).mean())
    with pytest.raises(ValueError):
        AdversarialLoss("wgan")


def test_cpu_input_raises():
    with pytest.raises(RuntimeError, match="GPU"):
        Discriminator()(torch.zeros(1, 1, 3, 16, 16))


def test_abi_rejects_bad_arguments_before_cuda():
    from e2fgvi_b200 import _lib
    lib = _lib.load()
    a = 1 << 20                    # fake, aligned addresses: every call below must fail before touching them
    assert lib.e2f_dis_conv3d(None, a, 8, a, a, None, a, None, None, 1, 1, 16, 16, 32, 1, 1, None) == -1
    assert lib.e2f_dis_conv3d(a, a, 8, a, a, None, a, a, None, 1, 1, 16, 16, 32, 1, 1, None) == -1   # hi without lo
    assert lib.e2f_dis_conv3d(a, a, 8, a, a, None, a, None, None, 1, 1, 16, 16, 32, 3, 1, None) == -1  # pad 3
    assert lib.e2f_dis_conv3d(a, a, 8, a, a, None, a, None, None, 1, 0, 16, 16, 32, 2, 1, None) == -1  # t = 0
    assert lib.e2f_dis_conv3d(a, a, 8, a, a, None, a, None, None, 1, 1, 2, 16, 32, 1, 1, None) == -1   # too small
    assert lib.e2f_dis_conv3d(a, a, 3, a, a, None, a, None, None, 1, 1, 16, 16, 32, 1, 1, None) == -2  # cin % 8
    assert lib.e2f_dis_conv3d(a, a, 8, a, a, None, a, None, None, 1, 1, 16, 16, 256, 1, 1, None) == -2  # cout > 128
    assert lib.e2f_dis_conv3d(a, a, 8, a, a, None, a, None, None, 1, 1, 16, 16, 32, 1, 2, None) == -1  # leaky
    assert lib.e2f_dis_conv3d(a + 2, a, 8, a, a, None, a, None, None, 1, 1, 16, 16, 32, 1, 1, None) == -3
    assert lib.e2f_dis_conv3d_dgrad(a, a, 32, a, a, None, None, None, None, 1, 1, 16, 16, 8, 1, None) == -1
    assert lib.e2f_dis_conv3d_dgrad(a, a, 32, a, a, a, None, None, None, 1, 1, 16, 16, 3, 1, None) == -2
    assert lib.e2f_dis_conv3d_dgrad(a, a, 32, a, a, a, None, None, a + 4, 1, 1, 16, 16, 8, 1, None) == -3
    assert lib.e2f_dis_conv3d_wgrad_work_elems(1, 1, 16, 16, 8, 32, 0) < 0                          # pad 0
    assert lib.e2f_dis_conv3d_wgrad_work_elems(1, 1, 16, 16, 3, 32, 1) < 0                          # cin % 8
    assert lib.e2f_dis_conv3d_wgrad_work_elems(1, 1, 16, 16, 8, 32, 1) > 0
    assert lib.e2f_dis_conv3d_wgrad(a, a, a, a, None, None, 1, 1, 16, 16, 8, 32, 1, None) == -1    # no workspace
    assert lib.e2f_dis_conv3d_wgrad(a, a, a, a, None, a, 1, 1, 16, 16, 8, 36, 1, None) == -1       # cout % 8
    assert lib.e2f_dis_conv3d_wgrad(a + 4, a, a, a, None, a, 1, 1, 16, 16, 8, 32, 1, None) == -3
