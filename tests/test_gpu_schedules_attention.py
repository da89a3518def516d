"""H100: which kernels the focal attention backward reaches and on what grids, read from a torch.profiler trace: the
row kernel once over (64-query tiles, heads, windows), then the key kernel (eight groups of key tiles per window and
head) and the gather once per chunk of (clip, head) pairs, and no vendor kernel.  None of the three is persistent:
each CTA owns one work item.  Numerics:
test_attention_train_gpu.py.  (A file of its own, ordered after every test that calls backward; see
test_gpu_schedules_encdec.py.)"""
import pytest
import torch

from e2fgvi_b200 import ops
from kernel_checks import TABLE, cdiv, run_traced

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,T,H,W,use_pooled", [(8, 8, 20, 36, 1), (2, 1, 5, 9, 0)])
def test_attention_backward_schedule(cuda, B, T, H, W, use_pooled):
    g = torch.Generator(device=cuda).manual_seed(B + T)
    qkv = torch.randn(B, T, H, W, 1536, device=cuda, generator=g).half()
    qkv_p = torch.randn(B, T, H // 5, W // 9, 1536, device=cuda, generator=g).half() if use_pooled else None
    dout = torch.randn(B, T, H, W, 512, device=cuda, generator=g)
    _, launches = run_traced(lambda: ops.focal_window_attention_backward(qkv, qkv_p, dout, 4, (5, 9), (2, 4), (5, 9),
                                                                         128 ** -0.5))
    ours = [k for k in launches if k.name.startswith("attn_grad_")]
    assert not [k.name for k in launches if "gemm" in k.name.lower() or "cutlass" in k.name.lower()]
    nW = (H // 5) * (W // 9)
    ring = 153                           # the 9 x 17 expanded-window positions, all listed (wrapped or not)
    nks = T * (ring + (45 if use_pooled else 0))
    units = B * 4
    chunk = max(1, min(units, (32 << 20) // (nW * (nks * 256 + 8 * T * 45 * 128))))
    tokens = T * H * W + (T * nW if use_pooled else 0)
    want = [("attn_grad_rows_kernel", (cdiv(T * 45, 64), 4, B * nW))]
    for u0 in range(0, units, chunk):
        n = min(chunk, units - u0)
        want += [("attn_grad_keys_kernel", (8, 1, n * nW)), ("attn_grad_gather_kernel", (tokens, n, 1))]
    assert [(k.name, k.grid) for k in ours] == want
    for k in ours[:3]:
        TABLE.append((f"attention backward {B}x{T}x{H}x{W} p{use_pooled}", k.name, k.grid, "-", 1, k.smem,
                      f"{len(ours)} launches, {chunk} (clip, head) pairs per chunk"))
