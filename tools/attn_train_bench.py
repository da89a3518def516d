"""Time one training step of the focal window attention at the training shape: ``WindowAttention.attend(x, pooled)``,
L1 against a target, ``backward()`` into qkv, proj, x and pooled — this library's kernels against an fp32 torch
restatement (F.linear and the reference's literal key list, oracle/restate.py; TF32 off and on).  Medians of --iters
steps after --warmup.  Prints the algorithmic FLOP count (from the shapes, on any machine): the attention forward is 2
products (S = QK^T, PV), its backward 5 (S, dP = dO V^T, dV = P^T dO, dQ = dS K, dK = dS^T Q); then the card, its
power limit and a sampled SM clock with the timings.  --profile instead takes the per-kernel split of our step with
torch.profiler (a separate run).

    python tools/attn_train_bench.py [--clips 8 --frames 8 --height 20 --width 36] [--profile] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

C, HEADS, WIN, EXP, FOC = 512, 4, (5, 9), (2, 4), (5, 9)


def flops(b, t, h, w):
    """(forward, backward) algorithmic FLOPs: the two Linears (backward: weight and input gradients) and the attention
    products over the reference's key count (duplicated ring tokens merged)."""
    from e2fgvi_b200.ops import attention_flops
    tok, pool = b * t * h * w, b * t * (h // WIN[0]) * (w // WIN[1])
    lin = 2 * (tok + pool) * C * 3 * C + 2 * tok * C * C
    att = attention_flops(b, t, h, w, C, WIN, EXP, FOC)
    return lin + att, 2 * lin + 2.5 * att


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
    ap.add_argument("--height", type=int, default=20, help="token grid height")
    ap.add_argument("--width", type=int, default=36, help="token grid width")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="per-kernel split of our step under torch.profiler")
    ap.add_argument("--out", default=None, help="directory for the JSON result (and the profile table)")
    a = ap.parse_args()
    b, t, h, w = a.clips, a.frames, a.height, a.width
    fwd, bwd = flops(b, t, h, w)
    print(f"{b}x{t}x{h}x{w} tokens: forward {fwd / 1e12:.3f} TFLOP, backward {bwd / 1e12:.3f} TFLOP")

    import torch
    if not torch.cuda.is_available():
        print("attn_train_bench: no CUDA device; nothing was timed", file=sys.stderr)
        return 2
    import torch.nn.functional as F
    from e2fgvi_b200 import ops
    from e2fgvi_b200.model.modules.tfocal_transformer import WindowAttention, rolled_valid_indices
    from oracle import restate

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    mod = WindowAttention(C, EXP, WIN, FOC, 2, HEADS, True, "fc").to(dev)
    x = torch.randn(b, t, h, w, C, device=dev, requires_grad=True)
    pooled = torch.randn(b, h // WIN[0], w // WIN[1], t, C, device=dev, requires_grad=True)
    target = torch.randn(b, t, h, w, C, device=dev)
    valid = rolled_valid_indices(WIN, EXP).to(dev)
    params = list(mod.parameters()) + [x, pooled]

    def ours():
        F.l1_loss(mod.attend(x, pooled), target).backward()

    def torch_fp32():
        qkv = F.linear(x, mod.qkv.weight, mod.qkv.bias)
        qkv_p = F.linear(pooled.permute(0, 3, 1, 2, 4), mod.qkv.weight, mod.qkv.bias)
        with dev:                                      # the restatement builds its pooled mask on the default device
            att = restate.focal_window_attention(qkv, qkv_p, HEADS, WIN, EXP, FOC, mod.scale, valid)
        F.l1_loss(F.linear(att, mod.proj.weight, mod.proj.bias), target).backward()

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

    result = {"card": torch.cuda.get_device_name(0), "power_limit_w": _smi("power.limit"), "clips": b, "frames": t,
              "grid": [h, w], "fwd_tflop": fwd / 1e12, "bwd_tflop": bwd / 1e12}
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
        with open(os.path.join(a.out, "attn_train_bench" + ("_profile" if a.profile else "") + ".json"), "w") as f:
            json.dump(result, f, indent=1)
    ops.invalidate_weight_caches()
    return 0


if __name__ == "__main__":
    sys.exit(main())
