"""H100: the encoder / decoder input gradient past one tile per CTA — the instantiation, grid and tile count the
launcher's arithmetic gives, read from a torch.profiler trace — including the stride-2 gradient's four phases of
different K length (1 / 2 / 2 / 4 taps), and no cuDNN / cuBLAS kernel in the call.  Numerics: test_encdec_train_gpu.py.
(A file of its own, ordered after every test that calls backward: on the H100 a profiler session followed in the same
process by autograd backward passes left later profiler sessions with no kernel records.)"""
import pytest
import torch

from e2fgvi_b200 import ops
from kernel_checks import cdiv, conv_tile, run_traced, sms

pytestmark = pytest.mark.gpu


def test_dgrad_schedules_past_one_tile(cuda):
    """Image counts from the SM count so that every CTA takes several tiles, the stride-2 phases (1 / 2 / 2 / 4 taps)
    included; the launch is the DACT instantiation the launcher's arithmetic picks, on the grid it sizes, and the
    backward calls no cuDNN / cuBLAS kernel."""
    h, w = 60, 108
    tw, th = conv_tile(cdiv(h, 2), cdiv(w, 2))
    per_img = cdiv(cdiv(h, 2), th) * cdiv(cdiv(w, 2), tw) * 4
    n = cdiv(3 * sms(), per_img)
    g = torch.Generator(device=cuda).manual_seed(3)
    dy = ops.split_nhwc(torch.randn(n, 128, 30, 54, device=cuda, generator=g))
    wt = torch.randn(128, 64, 3, 3, device=cuda, generator=g) * 0.05
    act = ops.split_nhwc(torch.randn(n, 64, h, w, device=cuda, generator=g))
    ops.conv_dgrad(dy, wt, stride=2, in_size=(h, w), act=act)          # weight packing outside the trace
    dx, launches = run_traced(lambda: ops.conv_dgrad(dy, wt, stride=2, in_size=(h, w), act=act))
    ours = [k for k in launches if k.name.startswith("conv3x3_dact_kernel")]
    assert [k.name for k in ours] == ["conv3x3_dact_kernel<64>"], [k.name for k in launches]
    tiles = n * per_img
    assert tiles >= 3 * sms() and ours[0].grid == (min(tiles, sms()), 1, 1)
    assert not [k.name for k in launches if "cudnn" in k.name.lower() or "gemm" in k.name.lower() or "cutlass" in k.name.lower()]
