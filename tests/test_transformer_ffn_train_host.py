"""CPU: the transposed weight operands of the transformer's token-path backward, emulated in float64 torch against
autograd / F.fold, the C ABI's argument rejections for the new entry points (validated before any CUDA call), and the
refresh of the cached transposed operands after an in-place parameter update."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from e2fgvi_b200 import ops

T2T = dict(kernel_size=(7, 7), stride=(3, 3), padding=(3, 3))


def _soft_comp_emulated(tok, wp, c, size, k=7, s=3, p=3):
    """The phase / tap walk of ``soft_comp`` (``_soft_comp_tables``) in float64: output pixel (s a + ry, s b + rx) sums
    token (a + dy, b + dx) . Wp[c, tap] over the taps of its phase; tokens outside the grid are zero."""
    n, fh, fw, hidden = tok.shape
    h, w = size
    taps, phases, _ = ops._soft_comp_tables(k, s, p)
    wp = wp.view(c, len(taps), hidden)
    out = torch.zeros(n, c, h, w, dtype=tok.dtype)
    pad = F.pad(tok.permute(0, 3, 1, 2), (2, 2, 2, 2)).permute(0, 2, 3, 1)     # token (a, b) at (a + 2, b + 2)
    for ph, (t0, ry, rx) in enumerate(phases):
        t1 = phases[ph + 1][0] if ph + 1 < len(phases) else len(taps)
        oh, ow = len(range(ry, h, s)), len(range(rx, w, s))
        acc = torch.zeros(n, oh, ow, c, dtype=tok.dtype)
        for t in range(t0, t1):
            dy, dx = taps[t]
            acc += pad[:, 2 + dy: 2 + dy + oh, 2 + dx: 2 + dx + ow] @ wp[:, t].t()
        out[:, :, ry::s, rx::s] = acc.permute(0, 3, 1, 2)
    return out


def test_soft_comp_transposed_weight_is_soft_splits_input_gradient():
    """fold(dT . W_ss) on soft_comp's phase walk with ``soft_comp_weight(W_ss, transpose=True)`` == autograd's gradient
    of SoftSplit's input."""
    g = torch.Generator().manual_seed(0)
    c, hidden, size = 8, 64, (13, 20)
    w_ss = torch.randn(hidden, c * 49, generator=g, dtype=torch.float64)
    x = torch.randn(2, c, *size, generator=g, dtype=torch.float64, requires_grad=True)
    tok = F.unfold(x, **T2T).transpose(1, 2) @ w_ss.t()
    fh, fw = (size[0] - 1) // 3 + 1, (size[1] - 1) // 3 + 1
    dt = torch.randn(tok.shape, generator=g, dtype=torch.float64)
    tok.backward(dt)
    wp = ops.soft_comp_weight(w_ss, 7, 3, 3, transpose=True).double()
    got = _soft_comp_emulated(dt.view(2, fh, fw, hidden), wp, c, size)
    torch.testing.assert_close(got, x.grad, rtol=1e-6, atol=1e-6)   # the packer works in fp32


def test_soft_comp_weight_is_the_fold():
    g = torch.Generator().manual_seed(1)
    c, hidden, size = 4, 64, (11, 17)
    w_sc = torch.randn(c * 49, hidden, generator=g).double()
    fh, fw = (size[0] - 1) // 3 + 1, (size[1] - 1) // 3 + 1
    tok = torch.randn(2, fh, fw, hidden, generator=g, dtype=torch.float64)
    want = F.fold((tok.view(2, fh * fw, hidden) @ w_sc.t()).transpose(1, 2), size, **T2T)
    got = _soft_comp_emulated(tok, ops.soft_comp_weight(w_sc, 7, 3, 3).double(), c, size)
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)


def test_soft_split_transposed_weight_is_soft_comps_token_gradient():
    """conv2d(dfeat, ``soft_split_weight(W_sc, transpose=True)``, stride 3, pad 3) == autograd's gradient of SoftComp's
    tokens (fold(T . W_sc^T))."""
    g = torch.Generator().manual_seed(2)
    c, hidden, size = 8, 64, (13, 20)
    fh, fw = (size[0] - 1) // 3 + 1, (size[1] - 1) // 3 + 1
    w_sc = torch.randn(c * 49, hidden, generator=g).double()
    tok = torch.randn(2, fh * fw, hidden, generator=g, dtype=torch.float64, requires_grad=True)
    feat = F.fold((tok @ w_sc.t()).transpose(1, 2), size, **T2T)
    dfeat = torch.randn(feat.shape, generator=g, dtype=torch.float64)
    feat.backward(dfeat)
    wt = ops.soft_split_weight(w_sc, c, 7, transpose=True).double()
    got = F.conv2d(dfeat, wt, stride=3, padding=3).flatten(2).transpose(1, 2)
    torch.testing.assert_close(got, tok.grad, rtol=1e-12, atol=1e-12)


def test_padded_transposed_linear_weight():
    """dY . W with dY's rows padded 1960 -> 1984 by zero columns: W^T padded alike gives the input gradient."""
    g = torch.Generator().manual_seed(3)
    w = torch.randn(1960, 512, generator=g)
    wt = ops.transposed_linear_weight(w, 1984)
    assert wt.shape == (512, 1984) and torch.all(wt[:, 1960:] == 0)
    x = torch.randn(6, 512, dtype=torch.float64, requires_grad=True)
    y = x @ w.double().t()
    dy = torch.randn(6, 1960, generator=g, dtype=torch.float64)
    y.backward(dy)
    got = F.pad(dy, (0, 24)) @ wt.double().t()
    torch.testing.assert_close(got, x.grad, rtol=1e-12, atol=1e-12)


def test_transposed_operands_refresh_after_in_place_update(monkeypatch):
    """The transposed operands are cached per parameter under their own tags and rebuilt once the parameter changes in
    place (an optimizer step)."""
    monkeypatch.setattr(ops, "split_bf16", lambda t: (t.clone(), torch.zeros_like(t)))
    lin = nn.Linear(512, 1960)
    first = ops._derived_one(lin.weight, ("split_t", 1984), ops._padded_split, 1984, True)
    assert ops._derived_one(lin.weight, ("split_t", 1984), ops._padded_split, 1984, True) is first
    sc = nn.Linear(512, 128 * 49)
    pack = ops._derived_one(sc.weight, ("soft_split_t", 128, 7), lambda wt: ops.soft_split_weight(wt, 128, 7, True))
    with torch.no_grad():
        lin.weight.mul_(2.0)
        sc.weight.add_(1.0)
    again = ops._derived_one(lin.weight, ("split_t", 1984), ops._padded_split, 1984, True)
    assert again is not first and torch.equal(again[0], ops.transposed_linear_weight(lin.weight, 1984))
    pack2 = ops._derived_one(sc.weight, ("soft_split_t", 128, 7), lambda wt: ops.soft_split_weight(wt, 128, 7, True))
    assert pack2 is not pack and torch.equal(pack2, ops.soft_split_weight(sc.weight, 128, 7, True))


def test_abi_rejections_without_gpu(lib):
    # linear weight gradient
    assert lib.e2f_linear_wgrad_work_elems(10, 0, 16) == -1
    assert lib.e2f_linear_wgrad_bf16x3(None, 16, 16, 16, 16, 16, 16, None, None, 64, 16, 16, None) == -1
    assert b"null" in lib.e2f_last_error()
    assert lib.e2f_linear_wgrad_bf16x3(16, 16, 12, 16, 16, 16, 16, None, None, 64, 12, 16, None) == -1   # ldy % 8
    assert lib.e2f_linear_wgrad_bf16x3(16, 16, 16, 16, 16, 8, 16, None, None, 64, 16, 16, None) == -1    # ldx < k
    assert b"pitches" in lib.e2f_last_error()
    assert lib.e2f_linear_wgrad_bf16x3(16, 16, 64, 16, 16, 64, 16, None, None, 1 << 20, 64, 64, None) == -1  # no work
    assert b"workspace" in lib.e2f_last_error()
    assert lib.e2f_linear_wgrad_bf16x3(8, 16, 16, 16, 16, 16, 16, None, None, 64, 16, 16, None) == -3   # misaligned
    # fold / unfold training modes
    args = (16, 16, 16, None, None, 1, 8, 60, 108)
    assert lib.e2f_t2t_fold_unfold_train(16, None, 16, None, None, 1, 8, 60, 108, 7, 3, 3, 0, 0, None) == -1  # null u
    assert lib.e2f_t2t_fold_unfold_train(*args, 7, 3, 3, 2, 0, None) == -1                                    # mode
    assert lib.e2f_t2t_fold_unfold_train(*args, 5, 2, 2, 0, 0, None) == -2                                    # geometry
    assert lib.e2f_t2t_fold_unfold_train(*args, 7, 3, 3, 1, 390, None) == -1                                  # pitch
    assert lib.e2f_t2t_fold_unfold_train(16, 8, 16, None, None, 1, 8, 60, 108, 7, 3, 3, 1, 0, None) == -3     # misaligned


def test_other_geometries_raise_not_implemented():
    with pytest.raises(NotImplementedError):
        ops.t2t_fold_unfold_train(torch.zeros(1, 4, 8 * 25), (6, 6), 5, 2, 2)
