"""Time one step of the transformer's dense token path at the training shape: ``sc(ffn(ss(feat)), residual=feat)``,
L1 against a target, ``backward()`` into the three modules' parameters — this library's kernels against an fp32 torch
restatement (F.unfold / F.linear / F.fold, TF32 off and on).  Medians of --iters steps after --warmup.  Prints the
algorithmic FLOP count (from the layer shapes, on any machine), then the card, its power limit and a sampled SM clock
with the timings.  --profile instead takes the per-kernel split of our step with torch.profiler (a separate run).

    python tools/ffn_bench.py [--clips 8 --frames 8 --height 60 --width 108] [--profile] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

C, HIDDEN, FFN = 128, 512, 1960
T2T = dict(kernel_size=(7, 7), stride=(3, 3), padding=(3, 3))


def flops(tokens):
    """(forward, backward) algorithmic FLOPs: 2 * MACs of the four Linears; the backward is every weight gradient plus
    every input gradient but SoftSplit's (the features need no gradient here)."""
    ss = sc = 2 * tokens * C * 49 * HIDDEN
    ffn = 2 * 2 * tokens * HIDDEN * FFN
    return ss + sc + ffn, 2 * (sc + ffn) + ss


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
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--height", type=int, default=60, help="feature height (240 / 4)")
    ap.add_argument("--width", type=int, default=108, help="feature width (432 / 4)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="per-kernel split of our step under torch.profiler")
    ap.add_argument("--out", default=None, help="directory for the JSON result (and the profile table)")
    a = ap.parse_args()
    n = a.clips * a.frames
    size = (a.height, a.width)
    fh, fw = (a.height - 1) // 3 + 1, (a.width - 1) // 3 + 1
    tokens = n * fh * fw
    fwd, bwd = flops(tokens)
    print(f"{tokens} tokens: forward {fwd / 1e12:.3f} TFLOP, backward {bwd / 1e12:.3f} TFLOP")

    import torch
    if not torch.cuda.is_available():
        print("ffn_bench: no CUDA device; nothing was timed", file=sys.stderr)
        return 2
    import torch.nn.functional as F
    from e2fgvi_b200 import ops
    from e2fgvi_b200.model.modules.tfocal_transformer import FusionFeedForward, SoftComp, SoftSplit

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ss = SoftSplit(C, HIDDEN, **T2T).to(dev)
    sc = SoftComp(C, HIDDEN, size).to(dev)
    ffn = FusionFeedForward(HIDDEN, t2t_params=dict(T2T, output_size=size)).to(dev)
    params = list(ss.parameters()) + list(sc.parameters()) + list(ffn.parameters())
    feat = torch.randn(n, C, *size, device=dev).contiguous(memory_format=torch.channels_last)
    target = torch.randn(n, C, *size, device=dev)
    ones = F.fold(torch.ones(1, FFN, fh * fw, device=dev), size, **T2T)      # the feed-forward's 40-channel fold

    def ours():
        tok = ss(feat, a.clips, size)
        x = tok.reshape(a.clips, -1, HIDDEN)
        y = ffn(x, size, residual=x)
        F.l1_loss(sc(y.reshape(tok.shape), a.frames, size, residual=feat), target).backward()

    def torch_fp32():
        tok = F.linear(F.unfold(feat, **T2T).transpose(1, 2), ss.embedding.weight, ss.embedding.bias)
        h = F.linear(tok, ffn.conv1[0].weight, ffn.conv1[0].bias)
        u = F.unfold(F.fold(h.transpose(1, 2), size, **T2T) / ones, **T2T).transpose(1, 2)
        y = F.linear(F.gelu(u), ffn.conv2[1].weight, ffn.conv2[1].bias) + tok
        cols = F.linear(y, sc.embedding.weight, sc.embedding.bias)
        F.l1_loss(F.fold(cols.transpose(1, 2), size, **T2T) + sc.bias + feat, target).backward()

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

    result = {"card": torch.cuda.get_device_name(0), "power_limit_w": _smi("power.limit"), "tokens": tokens,
              "size": list(size), "clips": a.clips, "frames": a.frames, "fwd_tflop": fwd / 1e12, "bwd_tflop": bwd / 1e12}
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
        old = torch.backends.cuda.matmul.allow_tf32
        try:
            result["ours_ms"] = timed(ours)
            result["sm_clock_mhz"] = _smi("clocks.sm")
            torch.backends.cuda.matmul.allow_tf32 = False
            result["torch_fp32_ms"] = timed(torch_fp32)
            torch.backends.cuda.matmul.allow_tf32 = True
            result["torch_tf32_ms"] = timed(torch_fp32)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = old
        for k in ("ours", "torch_fp32", "torch_tf32"):
            result[k + "_tflops"] = (fwd + bwd) / (result[k + "_ms"] * 1e-3) / 1e12
        print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ffn_bench" + ("_profile" if a.profile else "") + ".json"), "w") as f:
            json.dump(result, f, indent=1)
    ops.invalidate_weight_caches()
    return 0


if __name__ == "__main__":
    sys.exit(main())
