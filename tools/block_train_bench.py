"""Time training steps of the temporal focal transformer at the training shape (8 clips x 8 frames, 60x108 features,
20x36 tokens): one ``TemporalFocalTransformerBlock`` (forward, L1 against a target, ``backward()`` into every
parameter and the tokens) and the eight-block trunk ``sc(transformer(ss(feat)), t, residual=feat)`` (forward, L1,
backward into every trunk parameter and feat) — this library's kernels against the fp32 torch autograd of the
restatement (oracle/restate.py; TF32 off and on).  Medians of --iters steps after --warmup, the card, its power limit
and a sampled SM clock from the same run, and ``torch.cuda.max_memory_allocated`` of our trunk step.  A torch
restatement that does not fit in memory is reported as such.  --profile instead takes the per-kernel split of our
block step with torch.profiler (a separate run), with the LayerNorm backward kernels' achieved bytes/s against the
data-sheet 3.35 TB/s; their algorithmic bytes come from the shapes:
  layernorm_backward_kernel      x, dy, the residual g read, dx1 written fp32 and as the bf16 pair: 5 x rows x 2 KB;
  layernorm_pool_backward_kernel x, [dxn; dpooled], dx1 read, dx written: 4 x rows x 2 KB + pooled rows x 2 KB.

    python tools/block_train_bench.py [--clips 8 --frames 8] [--profile] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

C, SIZE, T2T = 512, (60, 108), dict(kernel_size=(7, 7), stride=(3, 3), padding=(3, 3))
PEAK_BW = 3.35e12


def kernel_bytes(b, t, h=20, w=36):
    rows, pooled = b * t * h * w, b * t * (h // 5) * (w // 9)
    return {"layernorm_backward_kernel": 5 * rows * C * 4,
            "layernorm_pool_backward_kernel": 4 * rows * C * 4 + pooled * C * 4}


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
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="per-kernel split of our block step under torch.profiler")
    ap.add_argument("--out", default=None, help="directory for the JSON result (and the profile table)")
    a = ap.parse_args()
    b, t = a.clips, a.frames
    nbytes = kernel_bytes(b, t)
    print(f"{b}x{t}x20x36 tokens: " + ", ".join(f"{k} {v / 1e9:.3f} GB" for k, v in nbytes.items()))

    import torch
    if not torch.cuda.is_available():
        print("block_train_bench: no CUDA device; nothing was timed", file=sys.stderr)
        return 2
    import torch.nn.functional as F
    from e2fgvi_b200 import ops
    from e2fgvi_b200.model.modules.tfocal_transformer import SoftComp, SoftSplit, TemporalFocalTransformerBlock
    from oracle import restate

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    t2t = dict(T2T, output_size=SIZE)
    ss = SoftSplit(128, C, **T2T, t2t_param=t2t).to(dev)
    sc = SoftComp(128, C, SIZE).to(dev)
    blocks = torch.nn.Sequential(*[TemporalFocalTransformerBlock(C, 4, (5, 9), focal_level=2, focal_window=(5, 9),
                                                                 t2t_params=t2t, pool_method="fc")
                                   for _ in range(8)]).to(dev)
    blk = blocks[0]
    x = torch.randn(b, t, 20, 36, C, device=dev, requires_grad=True)
    target = torch.randn(b, t, 20, 36, C, device=dev)
    feat = torch.randn(b * t, 128, *SIZE, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_()
    feat_target = torch.randn(b * t, 128, *SIZE, device=dev)
    sd = {f"transformer.{i}.{k}": v for i, m in enumerate(blocks) for k, v in
          list(m.named_parameters()) + list(m.named_buffers())}
    params = list(blocks.parameters()) + list(ss.parameters()) + list(sc.parameters()) + [x, feat]

    def block_ours():
        F.l1_loss(blk(x), target).backward()

    def block_torch():
        F.l1_loss(restate.transformer_block(sd, "transformer.0", x, SIZE), target).backward()

    def trunk_ours():
        F.l1_loss(sc(blocks(ss(feat, b)), t, residual=feat), feat_target).backward()

    def trunk_torch():
        tok = F.linear(F.unfold(feat, **T2T).transpose(1, 2), ss.embedding.weight, ss.embedding.bias)
        tok = tok.reshape(b, t, 20, 36, C)
        for i in range(8):
            tok = restate.transformer_block(sd, f"transformer.{i}", tok, SIZE)
        cols = F.linear(tok.reshape(b * t, -1, C), sc.embedding.weight, sc.embedding.bias)
        img = F.fold(cols.transpose(1, 2), SIZE, **T2T) + sc.bias
        F.l1_loss(img + feat, feat_target).backward()

    def timed(fn):
        times = []
        for i in range(a.warmup + a.iters):
            for p in params:
                p.grad = None
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            with dev:                                  # the restatement builds its pooled mask on the default device
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

    result = {"card": torch.cuda.get_device_name(0), "power_limit_w": _smi("power.limit"), "clips": b, "frames": t,
              "features": list(SIZE), "tokens": [20, 36]}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(a.warmup):
            block_ours()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            block_ours()
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=40)
        print(table)
        result["profile"] = table
        for ev in prof.key_averages():
            for k, nb in nbytes.items():
                if k in ev.key and ev.count:
                    us = ev.device_time_total / ev.count
                    result[k] = {"us": us, "gb": nb / 1e9, "tb_per_s": nb / (us * 1e-6) / 1e12,
                                 "share_of_3.35": nb / (us * 1e-6) / PEAK_BW}
        print(json.dumps({k: result[k] for k in nbytes if k in result}))
    else:
        old = torch.backends.cuda.matmul.allow_tf32
        try:
            result["block_ours_ms"] = timed(block_ours)
            torch.cuda.reset_peak_memory_stats()
            result["trunk_ours_ms"] = timed(trunk_ours)
            result["trunk_ours_max_memory_gb"] = torch.cuda.max_memory_allocated() / 1e9
            result["sm_clock_mhz"] = _smi("clocks.sm")
            for tf32 in (False, True):
                torch.backends.cuda.matmul.allow_tf32 = tf32
                tag = "tf32" if tf32 else "fp32"
                result[f"block_torch_{tag}_ms"] = timed_or_oom(block_torch)
                result[f"trunk_torch_{tag}_ms"] = timed_or_oom(trunk_torch)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = old
        print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "block_train_bench" + ("_profile" if a.profile else "") + ".json"), "w") as f:
            json.dump(result, f, indent=1)
    ops.invalidate_weight_caches()
    return 0


if __name__ == "__main__":
    sys.exit(main())
