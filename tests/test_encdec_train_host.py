"""CPU: the operand layouts of the encoder / decoder backward — per-source transposed grouped weights, the stride-2
phase tap tables — emulated in float64 torch against autograd / F.conv_transpose2d, and the C ABI's argument
rejections (validated before any CUDA call)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.generator import _ENC


def _cat(xs, groups):
    n, _, h, w = xs[0].shape
    return torch.cat([x.reshape(n, groups, -1, h, w) for x in xs], 2).reshape(n, -1, h, w)


def _input_grads(dy, weight, chans, groups, stride, h, w):
    xs = [torch.zeros(dy.shape[0], c, h, w, dtype=torch.float64, requires_grad=True) for c in chans]
    F.conv2d(_cat(xs, groups) if len(xs) > 1 else xs[0], weight, None, stride, 1, 1, groups).backward(dy)
    return [x.grad for x in xs]


# every encoder conv with an input gradient: (source channels, cout, stride, groups)
CASES = [([cin] if k <= 4 else [256, cin - 256], cout, s, g) for k, (cin, cout, s, g) in enumerate(_ENC) if k > 0]


@pytest.mark.parametrize("chans,cout,stride,groups", [c for c in CASES if c[2] == 1])
def test_source_dgrad_weight_is_the_transposed_group_weight(chans, cout, stride, groups):
    """conv(dY, Wt_s) with the stride-1 per-source weight — and with its groups merged as the launcher packs it —
    equals autograd's gradient of that source."""
    g = torch.Generator().manual_seed(cout + groups)
    h, w = 5, 7
    # fp32-exact values: the packers work in fp32
    weight = torch.randn(cout, sum(chans) // groups, 3, 3, generator=g).double()
    dy = torch.randn(2, cout, h, w, generator=g, dtype=torch.float64)
    want = _input_grads(dy, weight, chans, groups, 1, h, w)
    for s, ref in enumerate(want):
        wt = ops.source_dgrad_weight(weight, groups, chans, s).double()
        assert wt.shape == (chans[s], cout // groups, 3, 3)
        torch.testing.assert_close(F.conv2d(dy, wt, None, 1, 1, 1, groups), ref, rtol=1e-12, atol=1e-12)
        merged, g_eff = ops.merge_conv_groups(wt, [cout], groups)
        torch.testing.assert_close(F.conv2d(dy, merged.double(), None, 1, 1, 1, g_eff), ref, rtol=1e-12, atol=1e-12)


def test_stride2_phase_tables():
    """The four output phases of the stride-2 input gradient hold 1 / 2 / 2 / 4 taps; gathering dY at the tables'
    offsets with the forward's (unrotated) weights gives F.conv_transpose2d's result at every pixel, odd sizes too."""
    taps = ops.conv_dgrad_s2_taps()
    assert [sum(1 for t in taps if t[0] == ph) for ph in range(4)] == [1, 2, 2, 4]
    g = torch.Generator().manual_seed(1)
    for h, w in ((120, 216), (13, 19), (6, 9)):
        weight = torch.randn(16, 8, 3, 3, generator=g, dtype=torch.float64)
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        dy = torch.randn(2, 16, ho, wo, generator=g, dtype=torch.float64)
        want = F.conv_transpose2d(dy, weight, None, 2, 1, (h + 1 - 2 * ho, w + 1 - 2 * wo))
        assert want.shape[2:] == (h, w)
        got = torch.zeros_like(want)
        pad = F.pad(dy, (0, 1, 0, 1))                      # dY past its edge reads zero (the TMA fill)
        for ph, ky, kx in taps:
            oy, ox = ph // 2, ph % 2
            dy_, dx_ = (oy + 1 - ky) // 2, (ox + 1 - kx) // 2
            gh, gw = (h - oy + 1) // 2, (w - ox + 1) // 2   # grid pixels of this phase inside the image
            src = pad[:, :, dy_: dy_ + gh, dx_: dx_ + gw]
            got[:, :, oy::2, ox::2] += torch.einsum("nchw,cd->ndhw", src, weight[:, :, ky, kx])
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def test_abi_rejections(lib):
    p = 16
    base = [p, p, 64, 0, p, p, None, None, p, None, None, 1, 8, 8, 64, 1, 3, 1, None]
    def dgrad(**kw):
        args = list(base)
        names = ["dy_hi", "dy_lo", "dy_c", "dy_lead", "wt_hi", "wt_lo", "act", "residual", "dx", "dx_hi", "dx_lo", "n",
                 "h_in", "w_in", "cin", "groups", "ks", "stride", "stream"]
        for k, v in kw.items():
            args[names.index(k)] = v
        return lib.e2f_conv_dgrad_bf16x3(*args)
    assert dgrad(ks=5) == -2 and b"ks=5" in lib.e2f_last_error()
    assert dgrad(ks=7, stride=2) == -2
    assert dgrad(groups=3) == -2
    assert dgrad(groups=2, stride=2) == -2
    assert dgrad(cin=520) == -2
    assert dgrad(dy_lead=1, dy_c=64) == -2                     # row-gapped dY holds <= 32 channels
    assert dgrad(dy_lead=3) == -1                              # lead != ks / 2
    assert dgrad(dx=None) == -1
    assert dgrad(dy_hi=None) == -1
    assert dgrad(residual=8) == -3
    src = (ctypes.c_void_p * 2)(16, 16)
    chans = (ctypes.c_int * 2)(64, 64)
    assert lib.e2f_conv3x3_wgrad_bf16x3(p, 3, src, src, chans, 0, p, None, p, 1, 8, 8, 64, 1, 1, None) == -1
    assert lib.e2f_conv3x3_wgrad_bf16x3(p, 2, src, src, chans, 1, p, None, p, 1, 8, 8, 64, 1, 1, None) == -1
    assert lib.e2f_conv3x3_wgrad_bf16x3(p, 2, src, src, chans, 0, p, None, p, 1, 8, 8, 64, 1, 3, None) == -1
    assert lib.e2f_conv3x3_wgrad_bf16x3(p, 2, src, src, chans, 0, p, None, None, 1, 8, 8, 64, 1, 1, None) == -1
    assert b"workspace" in lib.e2f_last_error()
    assert lib.e2f_conv3x3_wgrad_work_elems(1, 8, 8, 12, 64, 1, 1) == -1
    assert lib.e2f_conv3x3_wgrad_work_elems(1, 60, 108, 640, 512, 2, 1) > 0
    assert lib.e2f_upsample2x_backward(32, None, 32, None, None, 1, 4, 4, 12, None) == -1
    assert lib.e2f_upsample2x_backward(16, None, 32, None, None, 1, 4, 4, 64, None) == -3
    assert lib.e2f_tanh_backward_rows(p, p, p, p, p, 1, 9, 4, 4, 1, None) == -1
    assert lib.e2f_tanh_backward_rows(p, p, p, p, p, 1, 3, 4, 4, 0, None) == -1
    assert lib.e2f_leaky_relu_backward(p, p, p, None, None, 12, 0.2, None) == -1
    assert lib.e2f_leaky_relu_backward(p, None, p, None, None, 16, 0.2, None) == -1
