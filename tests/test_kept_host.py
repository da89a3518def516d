"""CPU: the autograd boundary every trainable module shares (``KeptLaunches`` and ``tracked``), exercised with a
pure-torch launch sequence in place of the kernels: which gradients the backward is asked for, the refused second
backward, autograd's in-place check on the saved tensors and the ``None`` entries of the saved set."""
import pytest
import torch
import torch.nn as nn

from e2fgvi_b200.model._kept import KeptLaunches, tracked


class Owner:
    """Stands in for the module the real launch sequences receive as their first argument."""


def _run(keep, owner, x, y, w, scale, absent):
    """out = (x * w + y) * scale and x + w, keeping x; saves w and a None."""
    keep.update(owner=owner, x=x.detach(), scale=scale)
    return ((x * w + y) * scale, x + w), (w, absent)


class Back:
    """Records what the backward hands it and returns the exact gradients of ``_run``."""

    def __init__(self):
        self.calls = []

    def __call__(self, keep, saved, needs, g_out, g_sum):
        self.calls.append((keep, saved, needs))
        w, _ = saved
        scale = keep["scale"]
        dx = g_out * w * scale + g_sum if needs[1] else None
        dy = g_out * scale if needs[2] else None
        dw = g_out * keep["x"] * scale + g_sum if needs[3] else None
        return None, dx, dy, dw, None, None


def _inputs(seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(5, generator=g, requires_grad=True)
    y = torch.randn(5, generator=g)
    w = nn.Parameter(torch.randn(5, generator=g))
    return x, y, w


def test_backward_gets_needs_and_gives_the_gradients():
    x, y, w = _inputs()
    back = Back()
    owner = Owner()
    out, total = KeptLaunches.apply("Fake", _run, back, owner, x, y, w, 3.0, None)
    assert out.grad_fn is not None and total.grad_fn is not None
    (out.sum() + 2 * total.sum()).backward()
    (keep, saved, needs), = back.calls
    assert tuple(needs) == (False, True, False, True, False, False)
    assert keep["owner"] is owner
    assert saved[0] is w and saved[1] is None
    assert torch.equal(x.grad, w.detach() * 3.0 + 2)
    assert torch.equal(w.grad, x.detach() * 3.0 + 2)


def test_second_backward_raises():
    x, y, w = _inputs(1)
    out, _ = KeptLaunches.apply("Fake", _run, Back(), Owner(), x, y, w, 1.0, None)
    out.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="Fake: .* backpropagated a second time"):
        out.sum().backward()


def test_in_place_change_of_a_saved_tensor_raises():
    x, y, w = _inputs(2)
    back = Back()
    out, _ = KeptLaunches.apply("Fake", _run, back, Owner(), x, y, w, 1.0, None)
    with torch.no_grad():
        w.add_(1.0)                                     # as an optimizer.step() would
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.sum().backward()
    assert not back.calls


def test_tracked():
    x, y, w = _inputs(3)
    assert tracked([x], [])
    assert tracked([y, None, 3], [None, w])
    assert not tracked([y, None, "split operand"], [None])
    frozen = nn.Parameter(torch.zeros(2), requires_grad=False)
    assert not tracked([y], [frozen])
    with torch.no_grad():
        assert not tracked([x], [w])
