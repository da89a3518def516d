"""H100: which kernels the deformable alignment's backward reaches and on what grids, read from a torch.profiler trace:
dA on the linear kernel, the sampler adjoint once per 16 pixels, the weight gradient on the linear weight-gradient
kernel, CUB's radix sort of the dx scatter list, and the gather once per (destination, 4 channels).  No vendor GEMM.
Also: the launches follow what needs a gradient, and ``InpaintGenerator.forward`` under grad mode launches what it
launches under no_grad.  Numerics: test_align_train_gpu.py.  The backward runs as a plain call of ``_align_backward`` on
the kept operands, not through autograd.  (A file of its own, ordered after every test that calls backward; see
test_gpu_schedules_encdec.py.)"""
import pytest
import torch

from e2fgvi_b200.model.modules.feat_prop import SecondOrderDeformableAlignment, _align_backward
from kernel_checks import TABLE, cdiv, check_same_bits, run_traced

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,h,w", [(2, 12, 20), (1, 60, 108)])
def test_align_backward_schedule(cuda, n, h, w):
    torch.manual_seed(n + h)
    m = SecondOrderDeformableAlignment(256, 128, 3, padding=1, deform_groups=16).to(cuda)
    torch.nn.init.normal_(m.conv_offset[-1].weight, std=0.01)
    x = torch.randn(n, 256, h, w, device=cuda)
    extra = torch.randn(n, 384, h, w, device=cuda)
    f1, f2 = torch.randn(n, 2, h, w, device=cuda), torch.randn(n, 2, h, w, device=cuda)
    dy = torch.randn(n, 128, h, w, device=cuda)
    keep = {}
    with torch.no_grad():
        m._forward_keep(x, extra, f1, f2, keep)
    _align_backward(m, dict(keep), dy, [True] * 4, [True] * 10)
    _, launches = run_traced(lambda: _align_backward(m, dict(keep), dy, [True] * 4, [True] * 10))
    names = [k.name for k in launches]
    assert not any(nm.startswith(("ampere", "sm90_", "cutlass")) for nm in names), names
    M = n * h * w
    sample = [k for k in launches if k.name.startswith("sample_backward_kernel")]
    gather = [k for k in launches if k.name == "gather_kernel"]
    assert [k.name for k in sample] == ["sample_backward_kernel<true>"]
    assert [k.grid for k in sample] == [(cdiv(M, 16), 1, 1)]
    assert [k.grid for k in gather] == [(cdiv(M * 16 * 4, 256), 1, 1)]
    assert any("Onesweep" in nm or "RadixSort" in nm or "radix" in nm.lower() for nm in names), names
    assert names.count("linear_wgrad_kernel") == 1
    for k in sample + gather:
        TABLE.append((f"align backward {n}x{h}x{w}", k.name, k.grid, "-", 1, k.smem, "16 pixels / 64 outputs per CTA"))


COUT = 128


def _module(dev, seed, random_last):
    torch.manual_seed(seed)
    m = SecondOrderDeformableAlignment(2 * COUT, COUT, 3, padding=1, deform_groups=16)
    if random_last:
        torch.nn.init.normal_(m.conv_offset[-1].weight, std=0.01)
        torch.nn.init.normal_(m.conv_offset[-1].bias, std=0.1)
    return m.to(dev)


def _module_inputs(n, h, w, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(n, 2 * COUT, h, w, device=dev, generator=g)
    extra = torch.randn(n, 3 * COUT, h, w, device=dev, generator=g)
    f1, f2 = [torch.randn(n, 2, h, w, device=dev, generator=g) * 3 for _ in range(2)]
    return x, extra, f1, f2


def _names(launches):
    return [k.name for k in launches]


@pytest.mark.parametrize("case", ["all", "frozen_dcn", "frozen_head", "no_x", "x_only", "head_top_only"])
def test_only_what_is_needed_runs(cuda, case):
    """The backward's launches follow what needs a gradient: the DCN weight gradient, the x scatter, the sampler's
    offset/mask adjoint and each head conv's weight / input gradients."""
    m = _module(cuda, 11, True)
    x, extra, f1, f2 = _module_inputs(1, 12, 16, cuda, 3)
    need_in = [True, True, True, True]
    need = [True] * 10
    if case == "frozen_dcn":
        need[0] = need[1] = False
    elif case == "frozen_head":
        need[2:] = [False] * 8
        need_in[1:] = [False] * 3
    elif case == "no_x":
        need_in[0] = False
    elif case == "x_only":
        need = [False] * 10
        need_in = [True, False, False, False]
    elif case == "head_top_only":
        need = [False] * 8 + [True, True]
        need_in = [False] * 4
    keep = {}
    with torch.no_grad():
        m._forward_keep(x, extra, f1, f2, keep)
    dy = torch.randn(1, COUT, 12, 16, device=cuda)
    _align_backward(m, dict(keep), dy, need_in, need)        # the caches fill outside the trace
    grads, launches = run_traced(lambda: _align_backward(m, dict(keep), dy, need_in, need))
    names = _names(launches)
    head_adj = any(n.startswith("sample_backward_kernel<true") for n in names)
    assert head_adj == (case not in ("x_only", "frozen_head")), names
    assert ("gather_kernel" in names) == need_in[0], names
    assert ("linear_wgrad_kernel" in names) == (need[0] or need[1]), names
    assert not any(n.startswith(("ampere", "sm90_", "cutlass")) for n in names), names
    for i, gr in enumerate(grads):
        flag = (need_in + need)[i]
        assert (gr is not None) == flag, (case, i)


@pytest.mark.parametrize("hq", [False, True])
def test_generator_forward_unchanged_under_grad_mode(cuda, hq):
    """InpaintGenerator.forward with trainable parameters under grad mode launches the same kernels as under no_grad
    and predicts the same bits: the propagation's alignment stays untracked."""
    import importlib
    import warnings
    from e2fgvi_b200.synth import synth_frames, synth_state_dict
    net = importlib.import_module("model." + ("e2fgvi_hq" if hq else "e2fgvi"))
    g = net.InpaintGenerator().eval()
    g.load_state_dict(synth_state_dict(g, "stress", 3), strict=True)
    g = g.to(cuda)
    x = synth_frames(1, 5, 240, 432, seed=2).to(cuda)
    with torch.no_grad():
        g(x, 3)
        pred0, _ = g(x, 3)
        _, want = run_traced(lambda: g(x, 3))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        _, got = run_traced(lambda: g(x, 3))
        pred, _ = g(x, 3)
    assert pred.grad_fn is None
    assert sorted(_names(got)) == sorted(_names(want))
    check_same_bits(pred, pred0, "prediction under grad mode")
