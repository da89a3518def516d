"""H100: the Linear weight gradient past one item per CTA — the grid the launcher sizes (items = tiles x split-K slices,
one persistent CTA per SM) read from a torch.profiler trace, with the fixed-order slice reduction after it and no
cuBLAS kernel in the call.  Numerics: test_transformer_ffn_train_gpu.py.  (A file of its own, ordered after every
test that calls backward; see test_gpu_schedules_encdec.py.)"""
import pytest
import torch

from e2fgvi_b200 import ops
from kernel_checks import cdiv, expect_schedule, run_traced, sms

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m,n,k,ld", [(46080, 1960, 512, 1984), (46080, 512, 1960, 1984), (3000, 256, 384, 384)])
def test_linear_wgrad_schedule_past_one_item(cuda, m, n, k, ld):
    g = torch.Generator(device=cuda).manual_seed(n)
    dy = ops.SplitMat(*ops.split_bf16(torch.randn(m, ld if n == 1960 else n, device=cuda, generator=g)))
    x = ops.SplitMat(*ops.split_bf16(torch.randn(m, ld if k == 1960 else k, device=cuda, generator=g)))
    (dw, db), launches = run_traced(lambda: ops.linear_wgrad(dy, x, shape=(n, k)))
    tiles = cdiv(n, 128) * cdiv(k, 128)
    slices = max(1, min(cdiv(264, tiles), m // 256, 64))
    items = tiles * slices
    ours = [k_ for k_ in launches if "linear_wgrad" in k_.name or k_.name.startswith("reduce_kernel")]
    per_cta = expect_schedule(f"linear_wgrad {m}x{n}x{k}", ours[0], "linear_wgrad_kernel", items,
                              f"{slices} slices")
    assert per_cta >= 2 or items <= sms()
    assert [k_.name for k_ in ours[1:]] == (["reduce_kernel"] if slices > 1 else [])
    assert not [k_.name for k_ in launches if "gemm" in k_.name.lower() or "cutlass" in k_.name.lower()]
