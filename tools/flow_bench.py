"""Time the flow-completion step of train.py at the training shape (configs/train_e2fgvi.json: 8 clips of 5 + 3 frames
at 240x432, 64 (ref, supp) pairs at 64x128 per step) against a torch restatement on cuDNN.

Step: pred = netG.forward_bidirect_flow(masked local frames in [0, 1]) (tracks gradients into update_spynet),
loss = FlowCompletionLoss(pred, ground-truth local frames) (the ground-truth SPyNet under no_grad), loss.backward().

torch runs oracle/restate_flow.py in float32 (F.conv2d, F.grid_sample, autograd), twice: with TF32 off (fp32
convolutions, the accuracy class of this library's bf16x3 kernels) and with cuDNN TF32 on (PyTorch's default).
TFLOP/s are algorithmic: 2 * MACs of the 7x7 convolutions the step needs (both forwards, every weight gradient, the
input gradients of every conv except the coarsest level's first), counted from the shapes.  Also lists the library's
kernels by GPU time over one step (torch.profiler).  Prints one JSON line.

    python tools/flow_bench.py [--batch 8] [--local 5] [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from e2fgvi_b200.loss import FlowCompletionLoss  # noqa: E402
from e2fgvi_b200.model.modules.flow_comp import _LEVEL_CONVS, SPyNet  # noqa: E402
from e2fgvi_b200.synth import synth_spynet_state_dict  # noqa: E402
from oracle import restate_flow  # noqa: E402


class _Holder(torch.nn.Module):
    """What InpaintGenerator.forward_bidirect_flow needs of the generator: its update_spynet."""

    def __init__(self):
        super().__init__()
        self.update_spynet = SPyNet()


def conv_flop(pairs, hu, wu):
    per_px = sum(ci * co * 49 for ci, co in _LEVEL_CONVS)
    first = _LEVEL_CONVS[0][0] * _LEVEL_CONVS[0][1] * 49
    fwd = sum(pairs * (hu >> k) * (wu >> k) * per_px for k in range(6))
    dgrad = fwd - pairs * (hu >> 5) * (wu >> 5) * first
    return 2 * (2 * fwd + fwd + dgrad)          # update forward + ground-truth forward + weight grads + input grads


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
    ap.add_argument("--local", type=int, default=5)
    ap.add_argument("--height", type=int, default=240)
    ap.add_argument("--width", type=int, default=432)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flow_bench needs a GPU")
    from e2fgvi_b200.model.generator import InpaintGenerator
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    shape = (a.batch, a.local, 3, a.height, a.width)
    gt = torch.rand(shape, device=dev, generator=g)
    masked = gt.clone()
    masked[..., a.height // 4: a.height // 2, a.width // 3: a.width // 2] = 0
    upd, fix = synth_spynet_state_dict(0), synth_spynet_state_dict(100)
    h, w = a.height // 4, a.width // 4
    hu, wu = -(-h // 32) * 32, -(-w // 32) * 32
    flop = conv_flop(2 * a.batch * (a.local - 1), hu, wu)

    net = _Holder().to(dev)
    net.update_spynet.load_state_dict(upd)
    loss_fn = FlowCompletionLoss(pretrained=fix).to(dev)

    def ours():
        for p in net.parameters():
            p.grad = None
        pred = InpaintGenerator.forward_bidirect_flow(net, masked)
        loss_fn(pred, gt).backward()

    params = restate_flow.params_from_state_dict(upd, "", dtype=torch.float32, device=dev, requires_grad=True)
    gt_params = restate_flow.params_from_state_dict(fix, "", dtype=torch.float32, device=dev)
    mean, std = upd["mean"].to(dev), upd["std"].to(dev)

    def reference():
        for row in params:
            for pair in row:
                for t in pair:
                    t.grad = None
        pred = restate_flow.forward_bidirect_flow(params, mean, std, masked)
        restate_flow.flow_completion_loss(gt_params, mean, std, pred, gt).backward()

    res = {"shape": list(shape), "pairs": 2 * a.batch * (a.local - 1), "working_size": [hu, wu],
           "gpu": torch.cuda.get_device_name(), "step_gflop": round(flop / 1e9, 1)}
    torch.backends.cuda.matmul.allow_tf32 = False
    for name, fn, tf32 in (("e2fgvi_b200", ours, None), ("torch_fp32", reference, False),
                           ("torch_tf32_default", reference, True)):
        if tf32 is not None:
            torch.backends.cudnn.allow_tf32 = tf32
        med, best = timed(fn, a.iters, a.warmup)
        res[f"{name}_ms"] = round(med, 3)
        res[f"{name}_min_ms"] = round(best, 3)
        res[f"{name}_tflops"] = round(flop / med / 1e9, 1)
        print(f"{name:20s} {med:8.2f} ms (min {best:.2f})  {flop / med / 1e9:6.1f} TFLOP/s", file=sys.stderr)
    torch.backends.cudnn.allow_tf32 = True
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ours()
        torch.cuda.synchronize()
    per = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[ev.name.split("(")[0].replace("void ", "")] += ev.device_time_total / 1e3
    top = sorted(per.items(), key=lambda kv: -kv[1])[:10]
    res["e2fgvi_b200_kernel_ms"] = {k: round(v, 3) for k, v in top}
    for k, v in top:
        print(f"  {v:8.3f} ms  {k}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
