"""Goldens of the Temporal PatchGAN discriminator: the unmodified reference ``Discriminator`` (model/e2fgvi.py:271-344)
run in float64 on the CPU with weights from ``synth.synth_dis_state_dict``.

``python -m oracle.gen_golden_dis`` writes ``tests/golden/dis_<case>.npz`` and ``tests/golden/dis_layout.json``.  Per
case, with the model in train() mode and the trainer's hinge losses (core/trainer.py:319-334, without the optimizer
step between the two losses):

* ``eval_out``: the eval()-mode output on the real clip (no power iteration);
* ``out_real``, ``out_fake``: the train()-mode outputs, and ``u1_*`` / ``v1_*`` / ``u2_*`` / ``v2_*`` the spectral-norm
  vectors after the first and the second forward;
* ``dis_loss``, ``gan_loss``: (hinge(real, real) + hinge(fake, fake)) / 2 and the generator-side hinge on a third
  forward of the fake clip;
* ``gin``: d gan_loss / d fake clip (float32);
* per parameter, the gradients of dis_loss (``gd_*``) and of gan_loss (``gg_*``) as projections onto 8 fixed random
  unit vectors (``P_*``, regenerated from the seed by ``projections``) together with their max-abs values.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from e2fgvi_b200.synth import synth_dis_state_dict  # noqa: E402
from oracle import reference_loader  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = {
    # name: (b, t, h, w, use_sigmoid, use_spectral_norm, seed)
    "base": (1, 5, 60, 108, False, True, 0),
    "odd": (2, 3, 37, 61, False, True, 1),
    "t1": (1, 1, 40, 72, False, True, 2),
    "sigmoid": (1, 2, 32, 48, True, True, 3),
    "nosn": (1, 2, 32, 48, False, False, 4),
}
NPROJ = 8


def clips(b, t, h, w, seed):
    """(real, fake) clips in [-1, 1], float64 (B, T, 3, H, W)."""
    g = torch.Generator().manual_seed(1000 + seed)
    real = torch.rand(b, t, 3, h, w, generator=g, dtype=torch.float64) * 2 - 1
    fake = torch.rand(b, t, 3, h, w, generator=g, dtype=torch.float64) * 2 - 1
    return real, fake


def projections(name, numel, seed):
    g = torch.Generator().manual_seed(_stable(name, seed))
    p = torch.randn(NPROJ, numel, generator=g, dtype=torch.float64)
    return p / p.norm(dim=1, keepdim=True)


def _stable(name, seed):
    return (sum((i + 1) * ord(c) for i, c in enumerate(name)) * 7919 + seed) % (2 ** 31)


def hinge(out, is_real, is_disc):
    if not is_disc:
        return (-out).mean()
    return torch.relu(1 + (-out if is_real else out)).mean()


def run_case(name):
    b, t, h, w, sig, sn, seed = CASES[name]
    ref = reference_loader.import_reference("model.e2fgvi")
    net = ref.Discriminator(use_sigmoid=sig, use_spectral_norm=sn).double()
    sd = {k: v.double() for k, v in synth_dis_state_dict(seed, use_spectral_norm=sn).items()}
    net.load_state_dict(sd, strict=True)
    real, fake = clips(b, t, h, w, seed)
    res = {}
    net.eval()
    with torch.no_grad():
        res["eval_out"] = net(real).numpy()
    net.train()
    sn_keys = [k[:-2] for k in sd if k.endswith("_u")]
    real_clip = net(real)
    for k in sn_keys:
        res["u1_" + k] = net.state_dict()[k + "_u"].numpy().copy()
        res["v1_" + k] = net.state_dict()[k + "_v"].numpy().copy()
    fake_clip = net(fake)
    for k in sn_keys:
        res["u2_" + k] = net.state_dict()[k + "_u"].numpy().copy()
        res["v2_" + k] = net.state_dict()[k + "_v"].numpy().copy()
    dis_loss = (hinge(real_clip, True, True) + hinge(fake_clip, False, True)) / 2
    params = dict(net.named_parameters())
    gd = torch.autograd.grad(dis_loss, list(params.values()))
    comp = fake.clone().requires_grad_(True)
    gan_loss = hinge(net(comp), True, False)
    gg = torch.autograd.grad(gan_loss, [comp] + list(params.values()))
    res["out_real"] = real_clip.detach().numpy()
    res["out_fake"] = fake_clip.detach().numpy()
    res["dis_loss"] = np.float64(dis_loss.item())
    res["gan_loss"] = np.float64(gan_loss.item())
    res["gin"] = gg[0].numpy().astype(np.float32)
    for (k, p), d, g in zip(params.items(), gd, gg[1:]):
        P = projections(k, p.numel(), seed)
        res["gd_" + k] = (P @ d.reshape(-1)).numpy()
        res["gg_" + k] = (P @ g.reshape(-1)).numpy()
        res["gdmax_" + k] = np.float64(d.abs().max().item())
        res["ggmax_" + k] = np.float64(g.abs().max().item())
    np.savez_compressed(os.path.join(GOLDEN, f"dis_{name}.npz"), **res)
    return res


def layout():
    ref = reference_loader.import_reference("model.e2fgvi")
    out = {}
    for sn in (True, False):
        sd = ref.Discriminator(use_spectral_norm=sn).state_dict()
        out["spectral_norm" if sn else "plain"] = [[k, list(v.shape)] for k, v in sd.items()]
    with open(os.path.join(GOLDEN, "dis_layout.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    torch.manual_seed(0)
    layout()
    for name in sys.argv[1:] or CASES:
        run_case(name)
        print("wrote", name)
