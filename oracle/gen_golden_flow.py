"""Goldens of the flow-completion step: the unmodified reference ``InpaintGenerator.forward_bidirect_flow``
(model/e2fgvi.py:210-234, model/e2fgvi_hq.py) and ``FlowCompletionLoss`` (model/modules/flow_comp.py:11-46) run in
float64 on the CPU, with ``synth.synth_spynet_state_dict`` weights for both SPyNets.

``python -m oracle.gen_golden_flow`` writes ``tests/golden/flow_<case>.npz`` and ``tests/golden/flow_layout.json``.
Per case:

* ``flows_forward``, ``flows_backward``: ``netG.forward_bidirect_flow(masked)`` (float32);
* ``loss``: ``FlowCompletionLoss()(pred_flows, gt)``;
* per ``update_spynet`` parameter, its gradient of ``loss`` as projections onto 8 fixed random unit vectors (``g_*``,
  ``gen_golden_dis.projections`` regenerates them) and its max-abs value (``gmax_*``).

The frames are in [0, 1] as the trainer passes them (``(masked_frames[:, :l_t] + 1) / 2``).  The update SPyNet's last
convs are scaled so that its flows reach a few pixels (they clamp at the border); the ground-truth SPyNet has other
weights.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from e2fgvi_b200.synth import synth_spynet_state_dict  # noqa: E402
from oracle import reference_loader  # noqa: E402
from oracle.gen_golden_dis import projections  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = {
    # name: (b, l_t, h, w, hq, seed): the training frame size; flows that are not a multiple of 32 (30x50 -> 32x64);
    # the HQ model
    "base": (1, 3, 240, 432, False, 0),
    "odd": (2, 2, 120, 200, False, 1),
    "hq": (1, 3, 120, 216, True, 2),
}
FLOW_SCALE = 0.25


def frames(b, l_t, h, w, seed):
    """(masked, gt) local frames in [0, 1], float64 (b, l_t, 3, h, w): a smooth moving pattern plus noise (the
    ground truth), and the same with a zeroed rectangle per frame (the masked input)."""
    g = torch.Generator().manual_seed(2000 + seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, h, dtype=torch.float64), torch.linspace(0, 1, w, dtype=torch.float64),
                            indexing="ij")
    gt = torch.empty(b, l_t, 3, h, w, dtype=torch.float64)
    for bi in range(b):
        for j in range(l_t):
            for c in range(3):
                ph = 0.7 * c + 0.9 * bi + 0.15 * j
                gt[bi, j, c] = 0.5 + 0.35 * torch.sin(9 * xx + 5 * yy + ph) * torch.cos(6 * yy - 3 * xx + 2 * ph)
    gt = (gt + 0.05 * torch.rand(gt.shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    masked = gt.clone()
    for bi in range(b):
        for j in range(l_t):
            y0, x0 = (h // 4) + 3 * j, (w // 3) + 5 * j
            masked[bi, j, :, y0: y0 + h // 4, x0: x0 + w // 4] = 0
    return masked, gt


def weights(seed):
    """(update_spynet, fix_spynet) state dicts of one case."""
    return synth_spynet_state_dict(seed, flow_scale=FLOW_SCALE), synth_spynet_state_dict(seed + 100)


def run_case(name):
    b, l_t, h, w, hq, seed = CASES[name]
    ref = reference_loader.import_reference("model.e2fgvi_hq" if hq else "model.e2fgvi")
    flow_comp = ref.__reference_modules__["model.modules.flow_comp"]
    net = ref.InpaintGenerator().double()
    loss_fn = flow_comp.FlowCompletionLoss().double()
    upd, fix = weights(seed)
    net.update_spynet.load_state_dict({k: v.double() for k, v in upd.items()}, strict=True)
    loss_fn.fix_spynet.load_state_dict({k: v.double() for k, v in fix.items()}, strict=True)
    masked, gt = frames(b, l_t, h, w, seed)
    pred = net.forward_bidirect_flow(masked)
    loss = loss_fn(pred, gt)
    params = dict(net.update_spynet.named_parameters())
    grads = torch.autograd.grad(loss, list(params.values()))
    res = {"flows_forward": pred[0].detach().float().numpy(), "flows_backward": pred[1].detach().float().numpy(),
           "loss": np.float64(loss.item())}
    for (k, p), d in zip(params.items(), grads):
        P = projections(k, p.numel(), seed)
        res["g_" + k] = (P @ d.reshape(-1)).numpy()
        res["gmax_" + k] = np.float64(d.abs().max().item())
    np.savez_compressed(os.path.join(GOLDEN, f"flow_{name}.npz"), **res)
    return res


def layout():
    """The reference ``FlowCompletionLoss``'s state-dict keys and shapes."""
    ref = reference_loader.import_reference("model.e2fgvi")
    flow_comp = ref.__reference_modules__["model.modules.flow_comp"]
    sd = flow_comp.FlowCompletionLoss().state_dict()
    with open(os.path.join(GOLDEN, "flow_layout.json"), "w") as f:
        json.dump([[k, list(v.shape)] for k, v in sd.items()], f, indent=1)


if __name__ == "__main__":
    torch.manual_seed(0)
    layout()
    for name in sys.argv[1:] or CASES:
        run_case(name)
        print("wrote", name)
