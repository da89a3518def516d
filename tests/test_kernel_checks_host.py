"""The checks of kernel_checks have teeth: on the CPU, at small shapes, an emulation of the kernels' bf16x3
arithmetic passes them, and each of the faults a multi-tile schedule or an epilogue could introduce fails them."""
import pytest
import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

from kernel_checks import assert_exact_grid, check_close, check_exact, f32_split, grid_values, int_values


def _split(t):
    """torch's bf16 rounding of the hi part and of the remainder, as fp32."""
    hi = t.bfloat16().float()
    return hi, (t - hi).bfloat16().float()


def _bf16x3_conv(x, w, pad, drop_lo_hi=False):
    """conv2d of the bf16x3 kernels: lo(x).hi(w) + hi(x).lo(w) + hi(x).hi(w), each term and the sum in fp32."""
    xh, xl = _split(x)
    wh, wl = _split(w)
    out = F.conv2d(xh, wl, padding=pad) + F.conv2d(xh, wh, padding=pad)
    if not drop_lo_hi:
        out = F.conv2d(xl, wh, padding=pad) + out
    return out


def _ref(x, w, pad):
    return F.conv2d(x.double(), w.double(), padding=pad), F.conv2d(x.double().abs(), w.double().abs(), padding=pad)


@pytest.fixture
def conv_case():
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 16, 10, 13, generator=g)
    w = torch.randn(8, 16, 7, 7, generator=g) / (16 * 49) ** 0.5
    return x, w


def test_bf16x3_emulation_passes(conv_case):
    x, w = conv_case
    ref, bound = _ref(x, w, 3)
    check_close(_bf16x3_conv(x, w, 3), ref, bound, 5e-5, "f32", "host bf16x3")
    hi, lo = f32_split(_bf16x3_conv(x, w, 3))
    check_close(hi.double() + lo.double(), ref, bound, 5e-5, "split", "host bf16x3 split")


def test_dropped_lo_hi_term_fails(conv_case):
    x, w = conv_case
    ref, bound = _ref(x, w, 3)
    with pytest.raises(AssertionError):
        check_close(_bf16x3_conv(x, w, 3, drop_lo_hi=True), ref, bound, 5e-5, "f32", "host lo.hi dropped")


def _per_tap_conv(x, w, pad, shift_tap=None):
    """conv2d in float64 as a sum over taps; ``shift_tap`` = (ky, kx) reads its input one pixel to the right."""
    n, c, h, wd = x.shape
    k = w.shape[2]
    xp = F.pad(x.double(), (pad, pad + 1, pad, pad))
    out = 0
    for ky in range(k):
        for kx in range(k):
            dx = 1 if (ky, kx) == shift_tap else 0
            patch = xp[:, :, ky: ky + h, kx + dx: kx + dx + wd]
            out = out + torch.einsum("nchw,oc->nohw", patch, w[:, :, ky, kx].double())
    return out


def test_shifted_tap_fails(conv_case):
    x, w = conv_case
    ref, bound = _ref(x, w, 3)
    check_close(_per_tap_conv(x, w, 3), ref, bound, 5e-5, "f32", "host per-tap")
    with pytest.raises(AssertionError):
        check_close(_per_tap_conv(x, w, 3, shift_tap=(2, 5)), ref, bound, 5e-5, "f32", "host shifted tap")
    # on exact-grid data the exact check sees it too
    g = torch.Generator().manual_seed(12)
    xe, we = grid_values(x.shape, g, 0.2), int_values(w.shape, g)
    ref, bound = _ref(xe, we, 3)
    assert_exact_grid(bound, xe)
    check_exact(_per_tap_conv(xe, we, 3).float(), ref.float())
    with pytest.raises(AssertionError):
        check_exact(_per_tap_conv(xe, we, 3, shift_tap=(2, 5)).float(), ref.float())


def _sliced_wgrad(x, dy, slices, drop=None):
    """dW of a 7x7 / pad 3 conv as the split-K weight gradient forms it: fp32 partials over ``slices`` ranges of whole
    64-pixel K blocks, added in slice order; ``drop`` = (slice, block) leaves that K block out."""
    n, cin, h, w = x.shape
    cout = dy.shape[1]
    pixels = n * h * w
    per = -(-pixels // slices)
    ln = -(-per // 64) * 64
    cols = F.unfold(x, 7, padding=3).permute(0, 2, 1).reshape(pixels, cin * 49)      # pixel-major K
    dyk = dy.permute(0, 2, 3, 1).reshape(pixels, cout)
    total = torch.zeros(cout, cin * 49)
    for z in range(slices):
        k0, k1 = z * ln, min(z * ln + ln, pixels)
        keep = torch.ones(pixels, dtype=torch.bool)
        keep[:k0] = False
        keep[k1:] = False
        if drop is not None and drop[0] == z:
            keep[k0 + 64 * drop[1]: k0 + 64 * drop[1] + 64] = False
        total = total + dyk[keep].t() @ cols[keep]
    return total.view(cout, cin, 7, 7)


def test_dropped_wgrad_k_block_fails():
    g = torch.Generator().manual_seed(13)
    n, cin, cout, h, w = 3, 8, 8, 12, 20                       # 720 pixels: 3 slices of 256 (4 K blocks)
    pixels = n * h * w
    dy = grid_values((n, cout, h, w), g, 64.0 / pixels, fine=True)
    x = int_values((n, cin, h, w), g, 2)
    ref = nn_grad.conv2d_weight(x.double(), (cout, cin, 7, 7), dy.double(), padding=3)
    bound = nn_grad.conv2d_weight(x.double().abs(), (cout, cin, 7, 7), dy.double().abs(), padding=3)
    assert_exact_grid(bound, dy)
    check_exact(_sliced_wgrad(x, dy, 3), ref.float(), "host wgrad")
    with pytest.raises(AssertionError):
        check_exact(_sliced_wgrad(x, dy, 3, drop=(1, 2)), ref.float(), "host wgrad dropped block")


def test_wrong_derivative_side_fails():
    """One element of an input gradient multiplied by the other side of LeakyReLU(0.2)'s derivative."""
    g = torch.Generator().manual_seed(14)
    dy = torch.randn(2, 8, 9, 11, generator=g)
    w = torch.randn(8, 16, 7, 7, generator=g) * 0.05
    act = torch.randn(2, 16, 9, 11, generator=g).bfloat16()
    factor = torch.where(act.double() > 0, 1.0, 0.2)
    s = F.conv_transpose2d(dy.double(), w.double(), padding=3)
    ref = s * factor
    bound = F.conv_transpose2d(dy.double().abs(), w.double().abs(), padding=3) * factor
    got = (s * factor).float()
    check_close(got, ref, bound, 1e-4, "f32", "host dact")
    flipped = factor.clone().view(-1)
    i = int((s.abs() * (factor == 1.0)).view(-1).argmax())   # a large positive-side element
    flipped[i] = 0.2
    with pytest.raises(AssertionError):
        check_close((s * flipped.view(s.shape)).float(), ref, bound, 1e-4, "f32", "host dact flipped")
    # exact-grid data
    dye, we = int_values(dy.shape, g), grid_values(w.shape, g, 0.1)
    se = F.conv_transpose2d(dye.double(), we.double(), padding=3).float()
    ref32 = torch.where(act.float() > 0, se, se * torch.tensor(0.2))
    wrong = ref32.clone().view(-1)
    j = int((se.abs() * (act.float() <= 0)).view(-1).argmax())   # a large element on the 0.2 side
    wrong[j] = se.view(-1)[j]
    # the same result computed in fp32 (an fp32 transposed conv, then the epilogue's multiply) passes the exact check
    got32 = F.conv_transpose2d(dye, we, padding=3)
    check_exact(torch.where(act.float() > 0, got32, got32 * torch.tensor(0.2)), ref32, "host dact exact")
    with pytest.raises(AssertionError):
        check_exact(wrong.view(ref32.shape), ref32, "host dact exact flipped")


def test_wrong_phase_mapping_at_clipped_edge_fails():
    """Input gradient of the discriminator conv (3x5x5, stride (1, 2, 2), pad 1) for an odd width: phase ox = 1 has a
    GEMM column gx = (w - 1) / 2 whose pixel 2 gx + 1 = w lies outside the image.  A mapping that stores it at
    column w - 1 (clamped instead of dropped) must fail."""
    g = torch.Generator().manual_seed(15)
    b, t, h, w, cin, cout, pad = 1, 2, 9, 13, 8, 16, 1
    ho, wo = (h + 2 * pad - 5) // 2 + 1, (w + 2 * pad - 5) // 2 + 1
    dy = torch.randn(b, cout, t, ho, wo, generator=g, dtype=torch.float64)
    wt = torch.randn(cout, cin, 3, 5, 5, generator=g, dtype=torch.float64) / 30
    kw = dict(stride=(1, 2, 2), padding=(1, pad, pad))
    ref = nn_grad.conv3d_input((b, cin, t, h, w), wt, dy, **kw)
    bound = nn_grad.conv3d_input((b, cin, t, h, w), wt.abs(), dy.abs(), **kw)
    # the same gather one column further: what phase 1's clipped GEMM column computes
    wide = nn_grad.conv3d_input((b, cin, t, h, w + 1), wt, dy, **kw)
    assert torch.allclose(wide[..., :w], ref)
    got = ref.clone()
    got[..., w - 1] = wide[..., w]
    check_close(ref.float(), ref, bound, 5e-5, "f32", "host phase map")
    with pytest.raises(AssertionError):
        check_close(got.float(), ref, bound, 5e-5, "f32", "host phase map clamped")
