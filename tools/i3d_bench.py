"""Benchmark of the I3D feature extractor behind VFID: two 70-frame 432x240 videos as one batch (evaluate.py runs the
ground truth and the completed frames of a video), device-resident uint8, after a warm-up.  Times

  * this path (``InceptionI3d.features_u8``);
  * ``oracle/restate_i3d.py`` on cuDNN in fp32 (``allow_tf32 = False``) and with PyTorch's default TF32 convs (what
    evaluate.py gets), from the same frames (uint8 -> float / 255 is part of every timed call);

three alternated runs each, with CUDA events; then a per-kernel table of this path from ``torch.profiler`` in a run of
its own, with the algorithmic conv TFLOP/s computed here from the network's shapes.  Writes the JSON result to stdout
and, with --out, the profiler table to that directory.

    python tools/i3d_bench.py [--frames 70] [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from e2fgvi_b200 import synth  # noqa: E402
from e2fgvi_b200.i3d import MIXED, POOLS, InceptionI3d, same_pad  # noqa: E402
from oracle import restate_i3d  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return q.stdout.strip()


def conv_flops(b, t, h, w):
    """Algorithmic FLOPs (2 per multiply-add) of every conv of extract_features at input (b, 3, t, h, w)."""
    total = 0.0
    _, (t, h, w) = same_pad((7, 7, 7), (2, 2, 2), (t, h, w))
    total += 2.0 * b * t * h * w * 64 * 3 * 343
    size = same_pad(*POOLS["MaxPool3d_2a_3x3"], (t, h, w))[1]
    n = b * size[0] * size[1] * size[2]
    total += 2.0 * n * 64 * 64 + 2.0 * n * 192 * 64 * 27
    size = same_pad(*POOLS["MaxPool3d_3a_3x3"], size)[1]
    for name, cin, c in MIXED:
        if name == "Mixed_4b":
            size = same_pad(*POOLS["MaxPool3d_4a_3x3"], size)[1]
        if name == "Mixed_5b":
            size = same_pad(*POOLS["MaxPool3d_5a_2x2"], size)[1]
        n = b * size[0] * size[1] * size[2]
        total += 2.0 * n * (cin * (c[0] + c[1] + c[3] + c[5]) + 27 * (c[1] * c[2] + c[3] * c[4]))
    return total


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=70)
    ap.add_argument("--height", type=int, default=240)
    ap.add_argument("--width", type=int, default=432)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    t, h, w = args.frames, args.height, args.width
    sd = synth.synth_i3d_state_dict(0)
    model = InceptionI3d()
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    frames = torch.from_numpy(np.stack([synth.synth_video(t, h, w, seed=s)[0] for s in (0, 1)])).to(dev)

    def ours():
        return model.features_u8(frames)

    def cudnn():
        with torch.no_grad():
            x = frames.permute(0, 4, 1, 2, 3).float().div(255)
            return restate_i3d.extract_features(sd_dev, x)

    def run_fp32():
        torch.backends.cudnn.allow_tf32 = False
        try:
            return cudnn()
        finally:
            torch.backends.cudnn.allow_tf32 = tf32_default

    tf32_default = torch.backends.cudnn.allow_tf32
    ref = run_fp32()
    got = ours()
    tf = cudnn()
    torch.cuda.synchronize()
    err = (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())
    err_tf32 = (tf - ref).abs().max().item() / max(1.0, ref.abs().max().item())
    runs = {"ours_ms": [], "cudnn_fp32_ms": [], "cudnn_tf32_ms": []}
    for _ in range(3):
        runs["ours_ms"].append(timed(ours, args.reps))
        runs["cudnn_fp32_ms"].append(timed(run_fp32, args.reps))
        runs["cudnn_tf32_ms"].append(timed(cudnn, args.reps))
    flops = conv_flops(2, t, h, w)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            ours()
        torch.cuda.synchronize()
    table = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
            us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if us > 0:
                table[e.key] = {"calls_per_pass": e.count / args.reps, "ms_per_pass": us / 1e3 / args.reps}
    conv_ms = sum(v["ms_per_pass"] for k, v in table.items() if "conv3x3_kernel" in k)
    kernels = sorted(table.items(), key=lambda kv: -kv[1]["ms_per_pass"])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "i3d_kernels.json"), "w") as f:
            json.dump(kernels, f, indent=1)
    print(json.dumps({
        "workload": f"2 x {t} frames {w}x{h}, one batch, device-resident uint8",
        "card": card(), "conv_gflop": flops / 1e9, **runs,
        "ours_conv_tflops": [flops / (ms * 1e-3) / 1e12 for ms in runs["ours_ms"]],
        "conv_kernels_ms_per_pass": conv_ms, "conv_kernels_tflops": flops / (conv_ms * 1e-3) / 1e12 if conv_ms else None,
        "kernels": [(k[:90], round(v["calls_per_pass"], 1), round(v["ms_per_pass"], 3)) for k, v in kernels[:12]],
        "max_rel_err_vs_fp32": err, "cudnn_tf32_max_rel_err_vs_fp32": err_tf32}), flush=True)


if __name__ == "__main__":
    main()
