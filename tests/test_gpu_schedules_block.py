"""H100: which kernels the transformer block's backward reaches and on what grids, read from a torch.profiler trace:
the LayerNorm backward once per 64 rows and the LayerNorm + pooling backward once per (frame, window), each followed
by its fixed-order column sum over 32-column strips, and no vendor GEMM or reduction kernel anywhere in the backward.
Numerics: test_block_train_gpu.py.  The backward runs as a plain call of ``_block_backward`` on the kept operands, not
through autograd.  (A file of its own, ordered after every test that calls backward; see
test_gpu_schedules_encdec.py.)"""
import pytest
import torch

from e2fgvi_b200.model.modules.tfocal_transformer import TemporalFocalTransformerBlock, _block_backward
from kernel_checks import TABLE, cdiv, run_traced

pytestmark = pytest.mark.gpu

# every kernel of the block's forward and backward (linear_wgrad.cu's reduce_kernel adds its split-K slices)
LIBRARY = {"layernorm_pool_split_kernel", "layernorm_split_kernel", "linear_kernel", "focal_attn_kernel",
           "t2t_fold733_kernel", "split_bf16_kernel", "linear_wgrad_kernel", "reduce_kernel", "attn_grad_rows_kernel",
           "attn_grad_keys_kernel", "attn_grad_gather_kernel", "layernorm_backward_kernel",
           "layernorm_pool_backward_kernel", "column_sum_kernel"}


@pytest.mark.parametrize("B,T", [(2, 8), (1, 1)])
def test_block_backward_schedule(cuda, B, T):
    torch.manual_seed(B + T)
    blk = TemporalFocalTransformerBlock(512, 4, (5, 9), focal_level=2, focal_window=(5, 9), pool_method="fc",
                                        t2t_params=dict(kernel_size=(7, 7), stride=(3, 3), padding=(3, 3),
                                                        output_size=(60, 108))).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(2)
    x = torch.randn(B, T, 20, 36, 512, device=cuda, generator=g)
    grad = torch.randn(B, T, 20, 36, 512, device=cuda, generator=g)
    params = list(blk.params())

    def step():
        keep = {}
        with torch.no_grad():
            blk._forward(x, None, keep)
            return _block_backward(blk, keep, x, params, grad, True, [True] * 14)
    step()                                                   # the transposed-weight caches fill outside the trace
    (dx, grads), launches = run_traced(step)
    names = [k.name.split("<")[0] for k in launches]
    assert set(names) <= LIBRARY, sorted(set(names) - LIBRARY)
    assert {"layernorm_backward_kernel", "layernorm_pool_backward_kernel", "attn_grad_keys_kernel",
            "linear_wgrad_kernel"} <= set(names)
    rows = B * T * 20 * 36
    ln = [k for k in launches if k.name == "layernorm_backward_kernel"]
    pool = [k for k in launches if k.name == "layernorm_pool_backward_kernel"]
    sums = [k for k in launches if k.name == "column_sum_kernel"]
    assert [k.grid for k in ln] == [(cdiv(rows, 64), 1, 1)]
    assert [k.grid for k in pool] == [(16, B * T, 1)]
    assert [k.grid for k in sums] == [(32, 1, 1), (cdiv(2 * 512 + 46, 32), 1, 1)]
    assert dx is not None and all(gr is not None for gr in grads)
    for k in ln + pool:
        TABLE.append((f"block backward {B}x{T}x20x36", k.name, k.grid, "-", 1, k.smem, "one CTA per 64 rows / window"))
