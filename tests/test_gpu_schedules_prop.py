"""H100: which kernels the propagation's backward reaches and on what grids, read from a torch.profiler trace: the
flow-warp backward's sample kernels (one warp per pixel for NHWC features, one thread per pixel for the flow planes),
CUB's radix sort of the dx scatter list and the gathers.  No vendor GEMM.  The launch set follows what needs a gradient.
Numerics: test_prop_train_gpu.py.  The backward runs as a plain call of ``_prop_backward`` on the kept operands, not
through autograd.  (A file of its own, ordered after every test that calls backward; see test_gpu_schedules_encdec.py.)"""
import pytest
import torch

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.feat_prop import BidirectionalPropagation, _prop_backward
from kernel_checks import TABLE, cdiv, run_traced

pytestmark = pytest.mark.gpu

C = 128


def _setup(dev, b, t, h, w):
    torch.manual_seed(b + t + h)
    m = BidirectionalPropagation(C).to(dev)
    for name in m.DIRECTIONS:
        torch.nn.init.normal_(m.deform_align[name].conv_offset[-1].weight, std=0.01)
    x = torch.randn(b, t, C, h, w, device=dev)
    fb, ff = torch.randn(b, t - 1, 2, h, w, device=dev), torch.randn(b, t - 1, 2, h, w, device=dev)
    dy = torch.randn(b, t, C, h, w, device=dev)
    keep = {"mod": m, "flows": {"backward_": fb, "forward_": ff}}
    with torch.no_grad():
        x32 = x.permute(0, 1, 3, 4, 2).contiguous()
        m._propagate_keep(x32, *ops.split_bf16(x32), fb, ff, keep)
    return m, keep, dy


def _names(launches):
    return [k.name for k in launches]


@pytest.mark.parametrize("b,t,h,w", [(1, 3, 12, 20), (2, 5, 60, 108)])
def test_prop_backward_schedule(cuda, b, t, h, w):
    m, keep, dy = _setup(cuda, b, t, h, w)
    _prop_backward(m, dict(keep), dy, [True] * 3, [True] * 30)        # the caches fill outside the trace
    grads, launches = run_traced(lambda: _prop_backward(m, dict(keep), dy, [True] * 3, [True] * 30))
    assert all(g is not None for g in grads)
    names = _names(launches)
    assert not any(nm.startswith(("ampere", "sm90_", "cutlass")) for nm in names), names
    M = b * h * w
    steps = 2 * (t - 1)                          # aligned steps: cond_n1 warps
    second = 2 * (t - 2)                         # steps with a cond_n2 warp and a flows[:, i-2] warp
    s_nhwc = [k for k in launches if k.name == "sample_nhwc_kernel"]
    s_nchw = [k for k in launches if k.name == "sample_nchw_kernel"]
    g_nhwc = [k for k in launches if k.name == "gather_nhwc_kernel"]
    g_nchw = [k for k in launches if k.name == "gather_nchw_kernel"]
    assert len(s_nhwc) == steps + second and len(g_nhwc) == steps + second, names
    assert len(s_nchw) == second and len(g_nchw) == second, names
    assert {k.grid for k in s_nhwc} == {(cdiv(M, 8), 1, 1)}
    assert {k.grid for k in g_nhwc} == {(cdiv(M * C // 4, 256), 1, 1)}
    assert {k.grid for k in s_nchw + g_nchw} <= {(cdiv(M, 256), 1, 1)}
    assert any("Onesweep" in nm or "RadixSort" in nm for nm in names), names
    for k in s_nhwc[:1] + g_nhwc[:1] + s_nchw[:1] + g_nchw[:1]:
        TABLE.append((f"prop backward {b}x{t}x{h}x{w}", k.name, k.grid, "-", 1, k.smem,
                      "8 pixels / 256 (pixel, 4 channels) / 256 pixels per CTA"))


@pytest.mark.parametrize("case", ["all", "fusion_only", "no_flows", "flows_only", "frozen_alignment", "x_only"])
def test_only_what_is_needed_runs(cuda, case):
    """The launches follow what needs a gradient: with only the fusion trainable, only its weight gradient runs; without
    flow gradients no flow-plane warp runs; frozen alignments launch no DCN weight gradient."""
    m, keep, dy = _setup(cuda, 1, 4, 12, 16)
    need_in, need = [True] * 3, [True] * 30
    if case == "fusion_only":
        need_in, need = [False] * 3, [False] * 28 + [True, True]
    elif case == "no_flows":
        need_in = [True, False, False]
    elif case == "flows_only":
        need_in, need = [False, True, True], [False] * 30
    elif case == "frozen_alignment":
        for k in (0, 14):
            need[k: k + 10] = [False] * 10
    elif case == "x_only":
        need_in, need = [True, False, False], [False] * 30
    _prop_backward(m, dict(keep), dy, need_in, need)
    grads, launches = run_traced(lambda: _prop_backward(m, dict(keep), dy, need_in, need))
    names = _names(launches)
    assert not any(nm.startswith(("ampere", "sm90_", "cutlass")) for nm in names), names
    for i, g in enumerate(grads):
        assert (g is not None) == (need_in + need)[i], (case, i)
    wgrads = [n for n in names if "wgrad" in n]
    if case == "fusion_only":
        assert wgrads == ["linear_wgrad_kernel"] * 2, names           # the two halves of the fusion's weight
        assert not any("sample" in n or "gather" in n or "conv" in n or "linear_bf16x3" in n for n in names), names
    if case in ("no_flows", "x_only"):
        assert "sample_nchw_kernel" not in names, names
    if case in ("all", "flows_only"):
        assert "sample_nchw_kernel" in names, names
    if case in ("x_only", "flows_only"):
        assert not wgrads, names
    if case == "frozen_alignment":          # the fusion's two halves, not the DCNs'
        assert wgrads.count("linear_wgrad_kernel") == 2, names
    if case == "all":                       # the fusion's two halves and one per aligned step
        assert wgrads.count("linear_wgrad_kernel") == 2 + 2 * 3, names
