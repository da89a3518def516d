"""Micro-benchmark of the video front end (test.py:56-70 ``read_mask``, :98-103 ``resize_frames``):
``e2fgvi_b200.video.prepare_inputs`` on N device-resident synthetic frames and 'L' mask planes, timed with CUDA events
after a warm-up, next to the host Pillow + OpenCV path test.py runs, on a few of the same frames.  Prints one JSON line.

    python tools/frontend_bench.py [--frames 60] [--height 1080] [--width 1920] [--size 432 240] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from e2fgvi_b200.synth import synth_video  # noqa: E402
from e2fgvi_b200.video import prepare_inputs  # noqa: E402


def power_limit_w(index):
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(q.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return None


def host_ms_per_frame(frames, planes, size):
    """test.py:100 and the body of read_mask (:62-68) per frame, single process; None without Pillow / OpenCV."""
    try:
        import cv2
        from PIL import Image
    except ImportError:
        return None
    kern = cv2.getStructuringElement(cv2.MORPH_CROSS, (3, 3))
    t0 = time.perf_counter()
    for f, p in zip(frames, planes):
        Image.fromarray(f).resize(size)
        m = np.array(Image.fromarray(p).resize(size, Image.NEAREST).convert("L"))
        cv2.dilate(np.array(m > 0).astype(np.uint8), kern, iterations=4)
    return (time.perf_counter() - t0) * 1e3 / len(frames)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--size", type=int, nargs=2, default=(432, 240), metavar=("W", "H"))
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-frames", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n, h, w, size = args.frames, args.height, args.width, tuple(args.size)
    vf, vm = synth_video(n, h, w, 22)
    vm = vm * 255
    f_d, m_d = torch.from_numpy(vf).to(dev), torch.from_numpy(vm).to(dev)
    prepare_inputs(f_d, m_d, size)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        prepare_inputs(f_d, m_d, size)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.reps
    moved = n * h * w * 4 + n * size[0] * size[1] * 4               # RGB + mask bytes read, written
    host = host_ms_per_frame(vf[:args.host_frames], vm[:args.host_frames], size)
    print(json.dumps({
        "frames": n, "from": [w, h], "to": list(size), "ms": ms, "frames_per_s": n / (ms * 1e-3),
        "bytes_per_s": moved / (ms * 1e-3), "bytes_moved": moved, "inputs": "device-resident uint8 (upload not timed)",
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
        "host_ms_per_frame": host, "host_frames": args.host_frames,
        "speedup_vs_host": None if host is None else host * n / ms}), flush=True)


if __name__ == "__main__":
    main()
