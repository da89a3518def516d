"""Time the Temporal PatchGAN discriminator at the training shape (configs/train_e2fgvi.json: 8 clips of 5 + 3 frames
at 240x432 per GPU) against a torch restatement on cuDNN.

* dis step: netD(real), netD(fake), hinge dis_loss, dis_loss.backward() (inputs need no gradient);
* gen step: netD(comp) with a frozen discriminator, hinge gan_loss, d gan_loss / d comp.

torch runs twice: with TF32 off (fp32 convolutions, the accuracy class of this library's bf16x3 kernels) and at
PyTorch's default (cuDNN convolutions in TF32).  TFLOP/s are algorithmic: 2 * MACs of the convolutions the step needs,
counted from the shapes.  Prints one JSON line.

    python tools/dis_bench.py [--batch 8] [--frames 8] [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from e2fgvi_b200.loss import AdversarialLoss  # noqa: E402
from e2fgvi_b200.model.e2fgvi import Discriminator  # noqa: E402
from e2fgvi_b200.synth import synth_dis_state_dict  # noqa: E402

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
    """MACs of each layer's forward conv (= its input gradient's = its weight gradient's)."""
    out = []
    for i in range(6):
        pad = 1 if i == 0 else 2
        h, w = (h + 2 * pad - 5) // 2 + 1, (w + 2 * pad - 5) // 2 + 1
        out.append(b * t * h * w * CH[i + 1] * CH[i] * 75)
    return out


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    return times[len(times) // 2], times[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--height", type=int, default=240)
    ap.add_argument("--width", type=int, default=432)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dis_bench needs a GPU")
    dev = torch.device("cuda")
    shape = (a.batch, a.frames, 3, a.height, a.width)
    g = torch.Generator(device=dev).manual_seed(0)
    real = torch.rand(shape, device=dev, generator=g) * 2 - 1
    fake = torch.rand(shape, device=dev, generator=g) * 2 - 1
    adv = AdversarialLoss("hinge")
    sd = synth_dis_state_dict(0)
    macs = conv_macs(a.batch, a.frames, a.height, a.width)
    # dis step: two forwards; per backward every weight gradient and the input gradients of layers 1..5
    dis_flop = 2 * (2 * sum(macs) + 2 * sum(macs) + 2 * sum(macs[1:]))
    gen_flop = 2 * sum(macs) + 2 * sum(macs)          # forward + every input gradient

    def steps(net):
        net.load_state_dict(sd, strict=True)
        net.to(dev).train()
        params = list(net.parameters())

        def dis_step():
            for p in params:
                p.grad = None
            loss = (adv(net(real), True, True) + adv(net(fake), False, True)) / 2
            loss.backward()

        def gen_step():
            for p in params:
                p.requires_grad_(False)
            comp = fake.clone().requires_grad_(True)
            torch.autograd.grad(adv(net(comp), True, False), [comp])
            for p in params:
                p.requires_grad_(True)
        return dis_step, gen_step

    res = {"shape": list(shape), "gpu": torch.cuda.get_device_name(),
           "dis_step_gflop": dis_flop / 1e9, "gen_step_gflop": gen_flop / 1e9}
    runs = [("e2fgvi_b200", Discriminator, None), ("torch_fp32", torch_discriminator, False),
            ("torch_tf32_default", torch_discriminator, True)]
    for name, make, tf32 in runs:
        if tf32 is not None:
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = False
        dis_step, gen_step = steps(make())
        for step, flop, tag in ((dis_step, dis_flop, "dis"), (gen_step, gen_flop, "gen")):
            med, best = timed(step, a.iters, a.warmup)
            res[f"{name}_{tag}_ms"] = round(med, 3)
            res[f"{name}_{tag}_min_ms"] = round(best, 3)
            res[f"{name}_{tag}_tflops"] = round(flop / med / 1e9, 1)
            print(f"{name:20s} {tag} step  {med:8.2f} ms (min {best:.2f})  {flop / med / 1e9:6.1f} TFLOP/s",
                  file=sys.stderr)
    torch.backends.cudnn.allow_tf32 = True
    print(json.dumps(res))


if __name__ == "__main__":
    main()
