"""Benchmark of evaluate.py's metrics on the GPU: the fused PSNR / SSIM kernel (``e2fgvi_b200.metrics.frame_metrics``)
on a device-resident 70-frame 432x240 video, timed with CUDA events over many launches (uint8 frames against a float32
composite, and uint8 against uint8), next to the scipy restatement of skimage's SSIM per frame on the host (a CPU
number); then a per-stage breakdown of ``python -m e2fgvi_b200.evaluate`` on a synthetic dataset (decode, front end,
inpainting, metrics, I3D, PNG writes).  Prints one JSON line.

    python tools/eval_bench.py [--frames 70] [--reps 50] [--videos 3] [--video-size 480 854] [--host-frames 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from e2fgvi_b200 import metrics as M  # noqa: E402
from e2fgvi_b200.synth import synth_composite_pair  # noqa: E402

HBM_BPS = 3.35e12          # H100 SXM data sheet
FP64_VECTOR = 33.5e12      # H100 SXM data sheet, FP64 without tensor cores


def card():
    """Name, power limit and max SM clock of GPU 0, read in the same call as the measurement."""
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return q.stdout.strip()


def fp64_ops(n, h, w, c, win, tile=256):
    """fp64 operations the kernel issues, from shapes: per input pixel and channel of each tile's span 16 to add the
    row (x, y, squares, product, SSE) and 13 to drop it; per output row, span column and channel 5 quantities x 14 for
    the row scan; per output pixel and channel 31 for the window sums, means and S."""
    ho, wo = h - win + 1, w - win + 1
    tiles = -(-wo // tile)
    span_cols = min(tiles * (tile + win - 1), tiles * tile + w)       # input columns the tiles read, halos included
    return n * c * (h * span_cols * 29 + ho * span_cols * 70 + ho * wo * 31)


def time_kernel(a, b, reps):
    M.frame_metrics(a, b)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        M.frame_metrics(a, b)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_numbers(n, reps, dev):
    pairs = [synth_composite_pair(240, 432, 3, seed=s) for s in range(n)]
    ori = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
    comp = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
    out = {}
    for tag, b in (("u8_f32", comp), ("u8_u8", comp.to(torch.uint8))):
        ms = time_kernel(ori, b, reps)
        moved = ori.numel() * (1 + b.element_size())
        ops = fp64_ops(n, 240, 432, 3, 65)
        t_hbm, t_fp64 = moved / HBM_BPS, ops / FP64_VECTOR
        out[tag] = {"ms": ms, "frames_per_s": n / (ms * 1e-3), "bytes": moved, "bytes_per_s": moved / (ms * 1e-3),
                    "fp64_ops": ops, "fp64_ops_per_s": ops / (ms * 1e-3),
                    "bound": "fp64" if t_fp64 > t_hbm else "hbm",
                    "share_of_bound": max(t_hbm, t_fp64) / (ms * 1e-3)}
    return out, pairs


def host_ms_per_frame(pairs, k):
    from oracle import restate_ssim
    t0 = time.perf_counter()
    for ori, comp in pairs[:k]:
        restate_ssim.calc_psnr_and_ssim(ori, comp)
    return (time.perf_counter() - t0) * 1e3 / k


def command_breakdown(videos, n, size, dev):
    """Per-stage seconds of the evaluate command's per-video work, summed over ``videos`` synthetic videos."""
    import importlib
    import types
    import cv2
    from e2fgvi_b200 import evaluate as E
    from e2fgvi_b200 import synth
    from e2fgvi_b200.i3d import InceptionI3d
    from e2fgvi_b200.video import VideoInpainter, finalize, prepare_inputs
    gen = importlib.import_module("e2fgvi_b200.model.e2fgvi").InpaintGenerator()
    gen.load_state_dict(synth.synth_state_dict(gen, "stress", 2))
    gen = gen.eval().to(dev)
    i3d = InceptionI3d()
    i3d.load_state_dict(synth.synth_i3d_state_dict(0))
    i3d = i3d.to(dev).eval()
    drv = VideoInpainter(gen, neighbor_stride=E.NEIGHBOR_STRIDE, ref_length=E.REF_LENGTH, num_ref=-1)
    stages = dict.fromkeys(["decode", "front_end", "inpaint", "metrics", "i3d", "png_writes"], 0.0)
    with tempfile.TemporaryDirectory() as tmp:
        names = {f"v{k}": n for k in range(videos + 1)}            # v0 warms every shape up and is not counted
        root, _ = synth.write_eval_dataset(os.path.join(tmp, "data"), names, size=size)
        args = types.SimpleNamespace(data_root=root, dataset="davis")

        def clock(key, fn, count):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn()
            torch.cuda.synchronize()
            if count:
                stages[key] += time.perf_counter() - t0
            return r
        for k, name in enumerate(names):
            count = k > 0
            frames, masks = clock("decode", lambda: E.read_video(args, name, n), count)
            f, m = clock("front_end", lambda: prepare_inputs(frames, masks, E.SIZE, dev), count)
            comp = clock("inpaint", lambda: drv.composite(f, m), count)
            clock("metrics", lambda: M.frame_metrics(f, comp), count)
            u8 = finalize(comp)
            clock("i3d", lambda: i3d.features_u8(torch.stack([f, u8])).cpu(), count)
            out = os.path.join(tmp, "png", name)
            os.makedirs(out)

            def write():
                for i, fr in enumerate(u8.cpu().numpy()):
                    cv2.imwrite(os.path.join(out, f"{i:05d}.png"), cv2.cvtColor(fr, cv2.COLOR_RGB2BGR))
            clock("png_writes", write, count)
    return {k: v / videos * 1e3 for k, v in stages.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=70)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-frames", type=int, default=3)
    ap.add_argument("--videos", type=int, default=3)
    ap.add_argument("--video-size", type=int, nargs=2, default=(480, 854), metavar=("H", "W"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a GPU")
    dev = torch.device("cuda:0")
    kern, pairs = kernel_numbers(args.frames, args.reps, dev)
    host = host_ms_per_frame(pairs, args.host_frames)
    stages = command_breakdown(args.videos, args.frames, tuple(args.video_size), dev)
    print(json.dumps({
        "device": card(),
        "metrics_kernel": {"frames": args.frames, "size": [432, 240], "reps": args.reps, **kern},
        "host_scipy_ms_per_frame_cpu": host, "host_frames": args.host_frames,
        "command_ms_per_video": stages, "command_videos": args.videos, "command_frames_per_video": args.frames,
        "command_source_size": list(args.video_size)}), flush=True)


if __name__ == "__main__":
    main()
