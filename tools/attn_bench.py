"""Micro-benchmark of the focal attention kernel alone (B clips, T=8, 20x36 tokens, 4 heads x 128)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from e2fgvi_b200 import ops  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
dev = torch.device("cuda:0")
g = torch.Generator(device="cpu").manual_seed(0)
qkv = torch.randn(B, 8, 20, 36, 1536, generator=g).half().to(dev)
pooled = torch.randn(B, 8, 4, 4, 1536, generator=g).half().to(dev)
flops = ops.attention_flops(B, 8, 20, 36, 512, (5, 9), (2, 4), (5, 9))
for _ in range(3):
    ops.focal_window_attention(qkv, pooled, 4, (5, 9), (2, 4), (5, 9), 128 ** -0.5, out_dtype=torch.float32)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
n = 20
e0.record()
for _ in range(n):
    ops.focal_window_attention(qkv, pooled, 4, (5, 9), (2, 4), (5, 9), 128 ** -0.5, out_dtype=torch.float32)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / n
print(f"ATTN B={B}: {ms * 1e3:.1f} us/launch  {flops / ms / 1e9:.1f} TFLOP/s")
