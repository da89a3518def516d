"""Time one encoder + decoder training step at the training shape: ``pred = netG.decode(netG.encoder(x))``, L1
against a target, ``backward()`` — this library's kernels against oracle/restate.encoder / decoder on cuDNN float32
(TF32 off and on).  Medians of --iters steps after --warmup.  Prints the algorithmic FLOP counts (from the layer
shapes below, on any machine), then the card, its power limit and a sampled SM clock with the timings.  --profile
instead takes the per-kernel split of our step with torch.profiler (a separate run: tracing slows the host).

    python tools/encdec_bench.py [--clips 8 --frames 8 --height 240 --width 432] [--profile] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (cin, cout, stride, groups) of the encoder convs (e2fgvi.py:75-94) and (cin, cout, upsample before) of the decoder's
ENC = ((3, 64, 2, 1), (64, 64, 1, 1), (64, 128, 2, 1), (128, 256, 1, 1), (256, 384, 1, 1),
       (640, 512, 1, 2), (768, 384, 1, 4), (640, 256, 1, 8), (512, 128, 1, 1))
DEC = ((128, 128, True), (128, 64, False), (64, 64, True), (64, 3, False))


def flops(h, w):
    """(forward, backward) algorithmic FLOPs of one frame: 2 * MACs of each 3x3 conv; the backward is the weight
    gradient of every conv plus the input gradient of every conv but the stem (nothing trains the frames)."""
    fwd = bwd = 0
    for k, (cin, cout, s, g) in enumerate(ENC):
        h, w = (h - 1) // s + 1, (w - 1) // s + 1
        f = 2 * h * w * cout * (cin // g) * 9
        fwd += f
        bwd += f * (2 if k else 1)
    for cin, cout, up in DEC:
        if up:
            h, w = 2 * h, 2 * w
        f = 2 * h * w * cout * cin * 9
        fwd += f
        bwd += 2 * f
    return fwd, bwd


def _smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--clips", type=int, default=8)
    ap.add_argument("--frames", type=int, default=8, help="frames per clip (5 local + 3 reference in train.py)")
    ap.add_argument("--height", type=int, default=240)
    ap.add_argument("--width", type=int, default=432)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="per-kernel split of our step under torch.profiler")
    ap.add_argument("--out", default=None, help="directory for the JSON result (and the profile table)")
    a = ap.parse_args()
    n = a.clips * a.frames
    fwd, bwd = flops(a.height, a.width)
    print(f"per {a.height}x{a.width} frame: forward {fwd / 1e9:.2f} GFLOP ({fwd / 2e9:.2f} GMAC), backward "
          f"{bwd / 1e9:.2f} GFLOP; "
          f"step of {n} frames: {n * (fwd + bwd) / 1e12:.3f} TFLOP")

    import torch
    if not torch.cuda.is_available():
        print("encdec_bench: no CUDA device; nothing was timed", file=sys.stderr)
        return 2
    import torch.nn.functional as F
    from e2fgvi_b200 import ops
    from e2fgvi_b200.model.generator import InpaintGenerator
    from oracle import restate

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    gen = InpaintGenerator().to(dev)
    x = torch.rand(n, 3, a.height, a.width, device=dev) * 2 - 1
    target = torch.rand(n, 3, a.height, a.width, device=dev) * 2 - 1
    params = [p for k, p in gen.named_parameters() if k.startswith(("encoder.", "decoder."))]
    sd = {k: p for k, p in gen.named_parameters() if k.startswith(("encoder.", "decoder."))}

    def ours():
        F.l1_loss(gen.decode(gen.encoder(x)), target).backward()

    def cudnn():
        F.l1_loss(torch.tanh(restate.decoder(sd, restate.encoder(sd, x))), target).backward()

    def timed(fn):
        times = []
        for i in range(a.warmup + a.iters):
            for p in params:
                p.grad = None
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                times.append(e0.elapsed_time(e1))
        return statistics.median(times)

    result = {"card": torch.cuda.get_device_name(0), "power_limit_w": _smi("power.limit"), "frames": n,
              "size": [a.height, a.width], "fwd_gflop_per_frame": fwd / 1e9, "bwd_gflop_per_frame": bwd / 1e9}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(a.warmup):
            ours()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ours()
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=30)
        print(table)
        result["profile"] = table
    else:
        old = torch.backends.cudnn.allow_tf32
        try:
            result["ours_ms"] = timed(ours)
            result["sm_clock_mhz"] = _smi("clocks.sm")
            torch.backends.cudnn.allow_tf32 = False
            result["cudnn_fp32_ms"] = timed(cudnn)
            torch.backends.cudnn.allow_tf32 = True
            result["cudnn_tf32_ms"] = timed(cudnn)
        finally:
            torch.backends.cudnn.allow_tf32 = old
        for k in ("ours", "cudnn_fp32", "cudnn_tf32"):
            result[k + "_tflops"] = n * (fwd + bwd) / (result[k + "_ms"] * 1e-3) / 1e12
        print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "encdec_bench" + ("_profile" if a.profile else "") + ".json"), "w") as f:
            json.dump(result, f, indent=1)
    ops.invalidate_weight_caches()
    return 0


if __name__ == "__main__":
    sys.exit(main())
