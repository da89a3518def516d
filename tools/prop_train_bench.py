"""Time a training step of the feature propagation at the trainer's shape (8 clips of 5 local frames, 128 channels at
60x108): ``BidirectionalPropagation.forward`` + L1 against a target + ``backward()`` into x, both flow tensors and every
parameter — this library's kernels against the fp32 torch autograd of the restatement
(oracle/restate.bidirectional_propagation; TF32 off and on).  Medians of --iters steps after --warmup, the card, its
power limit and a sampled SM clock from the same run, and ``torch.cuda.max_memory_allocated`` of our step.  A second,
profiled step (torch.profiler, a separate run) gives the per-kernel split and the radix sorts' share of the step.

    python tools/prop_train_bench.py [--b 8] [--t 5] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZE = (60, 108)


def _smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--b", type=int, default=8, help="clips (the training batch)")
    ap.add_argument("--t", type=int, default=5, help="local frames per clip")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print("prop_train_bench: no CUDA device; nothing was timed", file=sys.stderr)
        return 2
    import torch.nn.functional as F
    from e2fgvi_b200 import ops
    from e2fgvi_b200.model.modules.feat_prop import BidirectionalPropagation
    from oracle import restate

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    b, t, (h, w) = a.b, a.t, SIZE
    mod = BidirectionalPropagation(128).to(dev)
    for name in mod.DIRECTIONS:                                         # non-trivial offsets
        torch.nn.init.normal_(mod.deform_align[name].conv_offset[-1].weight, std=0.01)
    x = torch.randn(b, t, 128, h, w, device=dev, requires_grad=True)
    fb = (2 * torch.randn(b, t - 1, 2, h, w, device=dev)).requires_grad_()
    ff = (2 * torch.randn(b, t - 1, 2, h, w, device=dev)).requires_grad_()
    target = torch.randn(b, t, 128, h, w, device=dev)
    sd = {f"m.{k}": v for k, v in mod.named_parameters()}
    params = list(mod.parameters()) + [x, fb, ff]

    def ours():
        F.l1_loss(mod(x, fb, ff), target).backward()

    def torch_ref():
        F.l1_loss(restate.bidirectional_propagation(sd, "m", x, fb, ff), target).backward()

    def timed(fn):
        times = []
        for i in range(a.warmup + a.iters):
            for p in params:
                p.grad = None
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            with dev:                                  # the restatement builds its index tensors on the default device
                fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                times.append(e0.elapsed_time(e1))
        return statistics.median(times)

    def timed_or_oom(fn):
        try:
            return timed(fn)
        except torch.cuda.OutOfMemoryError:
            for p in params:
                p.grad = None
            torch.cuda.empty_cache()
            return "out of memory"

    result = {"card": torch.cuda.get_device_name(0), "power_limit_w": _smi("power.limit"), "b": b, "t": t,
              "features": list(SIZE), "channels": 128}
    torch.cuda.reset_peak_memory_stats()
    result["ours_ms"] = timed(ours)
    result["ours_max_memory_gb"] = torch.cuda.max_memory_allocated() / 1e9
    result["sm_clock_mhz"] = _smi("clocks.sm")

    from torch.profiler import ProfilerActivity, profile
    for p in params:
        p.grad = None
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ours()
        torch.cuda.synchronize()
    split, total = {}, 0.0
    for ev in prof.key_averages():
        if ev.device_time_total > 0:
            split[ev.key[:90]] = round(ev.device_time_total / 1e3, 4)
            total += ev.device_time_total / 1e3
    sort_ms = sum(v for k, v in split.items() if "cub::" in k or "Onesweep" in k or "RadixSort" in k)
    result["profile_ms"] = dict(sorted(split.items(), key=lambda kv: -kv[1]))
    result["profile_total_ms"] = total
    result["sort_ms"] = sort_ms
    result["sort_share"] = sort_ms / total if total else None

    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    try:
        for tf32 in (False, True):
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
            result[f"torch_{'tf32' if tf32 else 'fp32'}_ms"] = timed_or_oom(torch_ref)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prop_train_bench.json"), "w") as f:
            json.dump(result, f, indent=1)
    ops.invalidate_weight_caches()
    return 0


if __name__ == "__main__":
    sys.exit(main())
