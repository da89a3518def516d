"""GPU parity of the three C-ABI kernels against the CPU oracle (bit-level semantics, fp tolerances stated)."""
import math

import pytest
import torch

from e2fgvi_b200 import ops
from oracle import restate

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------ flow_warp
@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("shape", [(1, 128, 60, 108), (2, 128, 17, 23), (3, 8, 5, 7)])
def test_flow_warp_nhwc_fp32(cuda, pad, shape):
    g = torch.Generator().manual_seed(7)
    n, c, h, w = shape
    x = torch.randn(n, c, h, w, generator=g)
    flow = torch.randn(n, h, w, 2, generator=g) * 6.0          # includes far out-of-bounds samples
    flow[0, 0, 0] = torch.tensor([1e6, -1e6])
    flow[0, h - 1, w - 1] = torch.tensor([0.0, 0.0])            # exact corner
    want = restate.flow_warp(x, flow, padding_mode=pad)
    got = ops.flow_warp(x.to(cuda).contiguous(memory_format=torch.channels_last), flow.to(cuda), padding_mode=pad)
    assert got.shape == want.shape
    # fp32 bilinear blend: only the association order differs -> 1e-5 abs on O(1) data
    assert (got.cpu() - want).abs().max().item() < 1e-5


def test_flow_warp_nhwc_fp16(cuda):
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 128, 30, 54, generator=g).half()
    flow = torch.randn(2, 30, 54, 2, generator=g) * 3.0
    want = restate.flow_warp(x.float(), flow)
    got = ops.flow_warp(x.to(cuda).contiguous(memory_format=torch.channels_last), flow.to(cuda))
    assert got.dtype == torch.float16
    assert (got.float().cpu() - want).abs().max().item() < 4e-3   # one fp16 rounding of an O(4) value


@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("c", [2, 3])
def test_flow_warp_nchw_small_channels(cuda, pad, c):
    g = torch.Generator().manual_seed(9)
    x = torch.randn(4, c, 64, 128, generator=g)
    flow = torch.randn(4, 64, 128, 2, generator=g) * 5.0
    want = restate.flow_warp(x, flow, padding_mode=pad)
    got = ops.flow_warp(x.to(cuda), flow.to(cuda), padding_mode=pad)
    assert got.is_contiguous()
    assert (got.cpu() - want).abs().max().item() < 1e-5


def test_flow_warp_errors(cuda):
    x = torch.zeros(1, 8, 4, 4, device=cuda)
    with pytest.raises(ValueError):
        ops.flow_warp(x, torch.zeros(1, 4, 5, 2, device=cuda))
    with pytest.raises(RuntimeError):
        ops.flow_warp(x.cpu(), torch.zeros(1, 4, 4, 2))


# ------------------------------------------------------------------------------------------ DCN
def _dcn_inputs(n, h, w, seed, off_scale=3.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 256, h, w, generator=g)
    offset = torch.randn(n, 288, h, w, generator=g) * off_scale
    mask = torch.rand(n, 144, h, w, generator=g)
    weight = torch.randn(128, 256, 3, 3, generator=g) / math.sqrt(2304.0)
    bias = torch.randn(128, generator=g) * 0.1
    return x, offset, mask, weight, bias


@pytest.mark.parametrize("shape", [(1, 60, 108), (2, 9, 11), (1, 16, 8), (3, 5, 7)])
def test_modulated_deform_conv2d(cuda, shape):
    n, h, w = shape
    x, offset, mask, weight, bias = _dcn_inputs(n, h, w, seed=11)
    # the kernel multiplies fp16 operands: feed the oracle the same fp16-rounded x and weight so the comparison
    # isolates the kernel's own arithmetic (fp32 interpolation, one fp16 rounding of the sampled value, fp32 accum)
    xq, wq = x.half().float(), weight.half().float()
    want = restate.modulated_deform_conv2d(xq.double(), offset.double(), mask.double(), wq.double(), bias.double(),
                                           1, 1, 1, 1, 16).float()
    got = ops.modulated_deform_conv2d(x.to(cuda), offset.to(cuda), mask.to(cuda), weight.to(cuda), bias.to(cuda),
                                      1, 1, 1, 1, 16)
    assert got.shape == want.shape
    rel = _rel(got.cpu(), want)
    # A-operand rounding to fp16 (2^-11 relative per element) averaged over K=2304 products: << 1e-3 of max
    assert rel < 1.5e-3, rel


@pytest.mark.parametrize("shape", [(1, 60, 108), (2, 9, 11)])
def test_modulated_deform_conv2d_unrounded_fp32_oracle(cuda, shape):
    """The same operator against the oracle fed the ORIGINAL fp32 x and weight (no pre-rounding): bounds what the
    kernel's fp16 operand policy (BASELINE configs[1]: "fp16 deform-conv") costs against the fp32 reference.
    Each product x*w carries two independent 2^-12-rms roundings; over K = 2304 terms of magnitude |x||w| the error
    of one output is ~ sqrt(K) * |x||w| * 2^-11.3 while the output itself is ~ sqrt(K) * |x||w| * E[mask * blend]:
    a few 1e-4 of the output scale.  Stated tolerance: 1e-3 of max|out| (the e2e budget is 1e-3 absolute on O(1))
    and 7e-4 of rms(out) for the rms error (three independent 2^-12-rms
    roundings per product - x, weight, the sampled value - give ~5e-4)."""
    n, h, w = shape
    x, offset, mask, weight, bias = _dcn_inputs(n, h, w, seed=21)
    want = restate.modulated_deform_conv2d(x.double(), offset.double(), mask.double(), weight.double(), bias.double(),
                                           1, 1, 1, 1, 16)
    got = ops.modulated_deform_conv2d(x.to(cuda), offset.to(cuda), mask.to(cuda), weight.to(cuda), bias.to(cuda),
                                      1, 1, 1, 1, 16).cpu().double()
    err = got - want
    assert err.abs().max().item() < 1e-3 * want.abs().max().item(), err.abs().max().item() / want.abs().max().item()
    assert err.pow(2).mean().sqrt().item() < 7e-4 * want.pow(2).mean().sqrt().item()


def test_deform_align_fused_unrounded_fp32_oracle(cuda):
    """Fused tail of feat_prop.py:41-58 (10*tanh + flow, sigmoid, DCN) against the oracle on unrounded fp32 inputs."""
    g = torch.Generator().manual_seed(23)
    n, h, w = 2, 12, 20
    x = torch.randn(n, 256, h, w, generator=g)
    head = torch.randn(n, 432, h, w, generator=g) * 1.5
    f1 = torch.randn(n, 2, h, w, generator=g) * 2
    f2 = torch.randn(n, 2, h, w, generator=g) * 2
    weight = torch.randn(128, 256, 3, 3, generator=g) / 48.0
    bias = torch.randn(128, generator=g) * 0.1
    o1, o2, m = torch.chunk(head.double(), 3, dim=1)
    off = 10.0 * torch.tanh(torch.cat((o1, o2), 1))
    a, b = torch.chunk(off, 2, dim=1)
    off = torch.cat([a + f1.double().flip(1).repeat(1, 72, 1, 1), b + f2.double().flip(1).repeat(1, 72, 1, 1)], 1)
    want = restate.modulated_deform_conv2d(x.double(), off, torch.sigmoid(m), weight.double(), bias.double(),
                                           1, 1, 1, 1, 16)
    wp = ops.pack_dcn_weight(weight.to(cuda), 16)
    got = ops.deform_align_fused(x.to(cuda), head.to(cuda), f1.to(cuda), f2.to(cuda), wp, bias.to(cuda), 16, 10.0)
    err = got.cpu().double() - want
    assert err.abs().max().item() < 1e-3 * want.abs().max().item()
    assert err.pow(2).mean().sqrt().item() < 7e-4 * want.pow(2).mean().sqrt().item()


def test_modulated_deform_conv2d_border_cases(cuda):
    """Offsets that land exactly on -1, H, integer grid points and far outside (zero-padding rule)."""
    n, h, w = 1, 6, 10
    x, offset, mask, weight, bias = _dcn_inputs(n, h, w, seed=12, off_scale=0.0)
    offset[:, 0::2, 0, :] = -1.0     # dy pushes row 0 samples to y = -2..0
    offset[:, 1::2, :, 0] = -1.0
    offset[:, 0::2, h - 1, :] = 1.0
    offset[:, :, 2, 3] = 1e5
    offset[:, :, 3, 4] = -1e5
    xq, wq = x.half().float(), weight.half().float()
    want = restate.modulated_deform_conv2d(xq.double(), offset.double(), mask.double(), wq.double(), bias.double(),
                                           1, 1, 1, 1, 16).float()
    got = ops.modulated_deform_conv2d(x.to(cuda), offset.to(cuda), mask.to(cuda), weight.to(cuda), bias.to(cuda),
                                      1, 1, 1, 1, 16)
    assert _rel(got.cpu(), want) < 1.5e-3


def test_deform_align_fused_matches_unfused(cuda):
    """Fused tanh/flow/sigmoid prologue == torch epilogue + plain DCN (feat_prop.py:41-58)."""
    g = torch.Generator().manual_seed(13)
    n, h, w = 2, 12, 20
    x = torch.randn(n, 256, h, w, generator=g)
    head = torch.randn(n, 432, h, w, generator=g) * 1.5
    f1 = torch.randn(n, 2, h, w, generator=g) * 2
    f2 = torch.randn(n, 2, h, w, generator=g) * 2
    weight = torch.randn(128, 256, 3, 3, generator=g) / 48.0
    bias = torch.randn(128, generator=g) * 0.1
    o1, o2, m = torch.chunk(head, 3, dim=1)
    off = 10.0 * torch.tanh(torch.cat((o1, o2), 1))
    a, b = torch.chunk(off, 2, dim=1)
    off = torch.cat([a + f1.flip(1).repeat(1, 72, 1, 1), b + f2.flip(1).repeat(1, 72, 1, 1)], 1)
    want = restate.modulated_deform_conv2d(x.half().double(), off.double(), torch.sigmoid(m).double(),
                                           weight.half().double(), bias.double(), 1, 1, 1, 1, 16).float()
    wp = ops.pack_dcn_weight(weight.to(cuda), 16)
    got = ops.deform_align_fused(x.to(cuda), head.to(cuda), f1.to(cuda), f2.to(cuda), wp, bias.to(cuda), 16, 10.0)
    assert _rel(got.cpu(), want) < 1.5e-3
    got16 = ops.deform_align_fused(x.to(cuda), head.to(cuda), f1.to(cuda), f2.to(cuda), wp, bias.to(cuda), 16, 10.0,
                                   out_dtype=torch.float16)
    assert _rel(got16.float().cpu(), want) < 3e-3


def test_dcn_linearity_full_size(cuda):
    """Size-independent property at the BASELINE shape (60x108, batch 8): DCN is linear in x for fixed offsets."""
    n, h, w = 8, 60, 108
    x1, offset, mask, weight, bias = _dcn_inputs(n, h, w, seed=14)
    x2 = torch.randn(n, 256, h, w, generator=torch.Generator().manual_seed(15))
    d = lambda t: ops.modulated_deform_conv2d(t.to(cuda), offset.to(cuda), mask.to(cuda), weight.to(cuda), None,  # noqa
                                              1, 1, 1, 1, 16)
    y1, y2, y12 = d(x1), d(x2), d(x1 + x2)
    assert _rel(y12, y1 + y2) < 3e-3


# ------------------------------------------------------------------------------------------ focal attention
def _attn_case(cuda, B, T, H, W, seed, gain=1.0, use_pooled=True, heads=4, window=(5, 9), out_dtype=torch.float32):
    from e2fgvi_b200.model.modules.tfocal_transformer import rolled_valid_indices
    g = torch.Generator().manual_seed(seed)
    C = heads * 128
    wh, ww = window
    expand = (wh // 2, ww // 2)
    qkv = (torch.randn(B, T, H, W, 3 * C, generator=g) * gain).half()
    pooled = (torch.randn(B, T, H // wh, W // ww, 3 * C, generator=g) * gain).half() if use_pooled else None
    scale = 128 ** -0.5
    fk = (2 * (wh // 2) + 1, 2 * (ww // 2) + 1)
    want = restate.focal_window_attention(qkv.float(), None if pooled is None else pooled.float(), heads, window,
                                          expand, fk, scale, rolled_valid_indices(window, expand))
    got = ops.focal_window_attention(qkv.to(cuda), None if pooled is None else pooled.to(cuda), heads, window,
                                     expand, fk, scale, out_dtype=out_dtype)
    return got.float().cpu(), want


@pytest.mark.parametrize("case", [
    dict(B=1, T=2, H=10, W=18, seed=21),            # 2x2 windows: every ring wraps around the token grid
    dict(B=2, T=3, H=20, W=36, seed=22),            # base token grid, 4x4 windows, partial last q-tile
    dict(B=1, T=1, H=5, W=9, seed=23),              # a single window: the ring wraps onto the window itself
    dict(B=1, T=3, H=15, W=27, seed=24, use_pooled=False),
    dict(B=1, T=2, H=10, W=18, seed=25, gain=4.0),  # logits spread over >> 2^8: exercises the O rescale path
])
def test_focal_window_attention(cuda, case):
    got, want = _attn_case(cuda, **case)
    assert got.shape == want.shape
    # P is rounded to fp16 before P.V (2^-11 relative per weight), everything else is fp32
    assert _rel(got, want) < 2e-3, _rel(got, want)


def test_focal_window_attention_base_size_fp16_out(cuda):
    got, want = _attn_case(cuda, B=1, T=8, H=20, W=36, seed=26, out_dtype=torch.float16)
    assert _rel(got, want) < 3e-3


def test_focal_window_attention_split_out(cuda):
    """out_dtype="split": the bf16 (hi, lo) pair equals the fp32 output to the two-term split's 2^-17."""
    g = torch.Generator().manual_seed(28)
    qkv = torch.randn(2, 3, 10, 18, 1536, generator=g).half().to(cuda)
    pooled = torch.randn(2, 3, 2, 2, 1536, generator=g).half().to(cuda)
    args = (4, (5, 9), (2, 4), (5, 9), 128 ** -0.5)
    f32 = ops.focal_window_attention(qkv, pooled, *args, out_dtype=torch.float32)
    sp = ops.focal_window_attention(qkv, pooled, *args, out_dtype="split")
    assert isinstance(sp, ops.SplitMat) and sp.shape == f32.shape
    assert (sp.hi.float() + sp.lo.float() - f32).abs().max().item() < 2e-5 * f32.abs().max().item() + 1e-7


def test_focal_attention_rows_sum_property(cuda):
    """Size-independent property at a large size (B=8 clips): with v == 1 the output must be exactly
    (sum_j p_j) / (sum_j p_j + n_masked * exp(-100 - m)) ~= 1 for every token, whatever q and k are."""
    B, T, H, W, C = 8, 8, 20, 36, 512
    g = torch.Generator().manual_seed(27)
    qkv = torch.randn(B, T, H, W, 3 * C, generator=g).half()
    qkv[..., 2 * C:] = 1.0
    pooled = torch.randn(B, T, 4, 4, 3 * C, generator=g).half()
    pooled[..., 2 * C:] = 1.0
    got = ops.focal_window_attention(qkv.to(cuda), pooled.to(cuda), 4, (5, 9), (2, 4), (5, 9), 128 ** -0.5,
                                     out_dtype=torch.float32)
    assert (got - 1.0).abs().max().item() < 2e-3


# ------------------------------------------------------------------------------------------ T2T fold / unfold
@pytest.mark.parametrize("shape", [(3, 40, 60, 108), (2, 128, 30, 54), (1, 4, 7, 7), (2, 8, 61, 110)])
def test_t2t_unfold_fold(cuda, shape):
    F = torch.nn.functional
    bt, c, h, w = shape
    g = torch.Generator().manual_seed(31)
    img = torch.randn(bt, c, h, w, generator=g)
    want = F.unfold(img, (7, 7), padding=(3, 3), stride=(3, 3)).permute(0, 2, 1)
    got = ops.t2t_unfold(img.to(cuda), (7, 7), (3, 3), (3, 3))
    assert torch.equal(got.cpu(), want)                               # pure data movement: bit-exact
    got_g = ops.t2t_unfold(img.to(cuda), (7, 7), (3, 3), (3, 3), gelu=True)
    assert (got_g.cpu() - F.gelu(want)).abs().max().item() < 2e-6
    tok = torch.randn(bt, want.shape[1], c * 49, generator=g)
    folded = F.fold(tok.permute(0, 2, 1), (h, w), (7, 7), padding=(3, 3), stride=(3, 3))
    got_f = ops.t2t_fold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3))
    assert (got_f.cpu() - folded).abs().max().item() < 1e-5         # <= 9 fp32 adds in a different order
    ones = F.fold(torch.ones(1, 49, want.shape[1]), (h, w), (7, 7), padding=(3, 3), stride=(3, 3))
    bias = torch.randn(c, h, w, generator=g)
    got_n = ops.t2t_fold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3), normalize=True, bias=bias.to(cuda))
    want_n = folded / ones + bias[None]
    ok = torch.isfinite(want_n)
    assert (got_n.cpu()[ok] - want_n[ok]).abs().max().item() < 1e-5
    if c % 8 == 0:
        # channels_last image in (read in place, no NCHW copy) / out (+ residual added by the fold kernel)
        img_cl = img.to(cuda).contiguous(memory_format=torch.channels_last)
        assert torch.equal(ops.t2t_unfold(img_cl, (7, 7), (3, 3), (3, 3)), got)
        sp_a = ops.t2t_unfold(img_cl, (7, 7), (3, 3), (3, 3), gelu=True, out="split")
        sp_b = ops.t2t_unfold(img.to(cuda), (7, 7), (3, 3), (3, 3), gelu=True, out="split")
        assert torch.equal(sp_a.hi, sp_b.hi) and torch.equal(sp_a.lo, sp_b.lo)
        res = torch.randn(bt, c, h, w, generator=g)
        got_cl = ops.t2t_fold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3), bias=bias.to(cuda),
                              residual=res.to(cuda).contiguous(memory_format=torch.channels_last), channels_last=True)
        assert got_cl.shape == (bt, c, h, w) and got_cl.permute(0, 2, 3, 1).is_contiguous()
        assert (got_cl.cpu() - (folded + bias[None] + res)).abs().max().item() < 2e-5
        got_cl2 = ops.t2t_fold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3), normalize=True, channels_last=True)
        want2 = folded / ones
        assert (got_cl2.cpu()[torch.isfinite(want2)] - want2[torch.isfinite(want2)]).abs().max().item() < 1e-5


@pytest.mark.parametrize("shape", [(3, 40, 60, 108), (2, 12, 30, 54), (1, 4, 7, 7), (2, 8, 61, 110), (1, 40, 135, 240),
                                   (1, 4, 9, 1500), (1, 3, 16, 16)])
def test_t2t_fold_unfold_fused(cuda, shape):
    """One-kernel fold / fold(ones) -> unfold (-> GELU) against F.fold / F.unfold (tfocal_transformer.py:89-96):
    several bands (tall images), the large-shared-memory configuration (very wide image), image sizes that leave a
    ragged last patch, and the error for a channel count the token layout cannot hold (C*49 % 4 != 0)."""
    F = torch.nn.functional
    bt, c, h, w = shape
    g = torch.Generator().manual_seed(37)
    fh, fw = (h + 6 - 7) // 3 + 1, (w + 6 - 7) // 3 + 1
    tok = torch.randn(bt, fh * fw, c * 49, generator=g)
    folded = F.fold(tok.permute(0, 2, 1), (h, w), (7, 7), padding=(3, 3), stride=(3, 3))
    ones = F.fold(torch.ones(1, 49, fh * fw), (h, w), (7, 7), padding=(3, 3), stride=(3, 3))
    norm = torch.nan_to_num(folded / ones, nan=0.0, posinf=0.0, neginf=0.0)     # pixels no patch covers stay 0
    want = F.unfold(norm, (7, 7), padding=(3, 3), stride=(3, 3)).permute(0, 2, 1)
    if (c * 49) % 4:
        with pytest.raises(RuntimeError):
            ops.t2t_fold_unfold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3))
        return
    got = ops.t2t_fold_unfold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3))
    assert (got.cpu() - want).abs().max().item() < 1e-5
    sp = ops.t2t_fold_unfold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3), gelu=True, out="split")
    assert (_join(sp).cpu() - F.gelu(want)).abs().max().item() < 5e-5
    # padded rows (pitch): same values, zero columns behind; a Linear fed by them pads its weight with zero columns
    pitch = (c * 49 + 63) // 64 * 64 + 8
    spp = ops.t2t_fold_unfold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3), gelu=True, out="split", pitch=pitch)
    assert spp.shape == (bt, fh * fw, pitch)
    assert torch.equal(spp.hi[..., : c * 49], sp.hi) and torch.equal(spp.lo[..., : c * 49], sp.lo)
    assert float(spp.hi[..., c * 49:].float().abs().max()) == 0.0 and float(spp.lo[..., c * 49:].float().abs().max()) == 0.0
    if (c * 49) % 8 == 0:                                            # the unpadded GEMM needs K % 8 == 0
        wl = torch.nn.Parameter(torch.randn(24, c * 49, generator=g).to(cuda) / (c * 49) ** 0.5)
        assert _rel(ops.linear(spp, wl), ops.linear(sp, wl)) < 1e-6
    # agrees with the two-kernel composition it replaces
    img = ops.t2t_fold(tok.to(cuda), (h, w), (7, 7), (3, 3), (3, 3), normalize=True)
    two = ops.t2t_unfold(torch.nan_to_num(img, nan=0.0, posinf=0.0, neginf=0.0), (7, 7), (3, 3), (3, 3))
    assert (got - two).abs().max().item() < 1e-5


# ------------------------------------------------------------------------------------------ bf16x3 linear
@pytest.mark.parametrize("case", [
    dict(m=5760, k=512, n=1536, out=torch.float16),               # attn.qkv of one clip
    dict(m=300, k=1960, n=512, residual=True),                    # mlp.conv2: K tail (1960 = 30.6 x 64), M tail
    dict(m=720, k=512, n=1960, tile=128),                         # mlp.conv1: N tail
    dict(m=720, k=512, n=1960, tile=256),                         # ... tile_hint 256 is accepted; every hint runs 128 x 128 tiles
    dict(m=257, k=6272, n=512),                                   # ss.embedding: long K
    dict(m=129, k=512, n=6272, residual=True),                    # sc.embedding: wide N
    dict(m=1, k=8, n=4),                                          # degenerate
])
def test_linear_bf16x3(cuda, case):
    g = torch.Generator().manual_seed(41)
    m, k, n = case["m"], case["k"], case["n"]
    x = torch.randn(m, k, generator=g) * 2.0
    w = torch.nn.Parameter(torch.randn(n, k, generator=g) / (k ** 0.5))
    b = torch.randn(n, generator=g)
    r = torch.randn(m, n, generator=g) if case.get("residual") else None
    want = torch.nn.functional.linear(x.double(), w.detach().double(), b.double())
    if r is not None:
        want = want + r.double()
    wd = torch.nn.Parameter(w.detach().to(cuda))
    got = ops.linear(x.to(cuda), wd, b.to(cuda), None if r is None else r.to(cuda),
                     out_dtype=case.get("out", torch.float32), tile_hint=case.get("tile", 0))
    assert got.shape == (m, n)
    tol = 1.5e-3 if case.get("out") is torch.float16 else 5e-5    # fp16 store rounding vs 3-term bf16 split (~2^-16 of max|out|)
    assert _rel(got.cpu(), want) < tol, _rel(got.cpu(), want)


def test_linear_weight_cache_tracks_updates(cuda):
    w = torch.nn.Parameter(torch.randn(64, 64, device=cuda))
    x = torch.randn(16, 64, device=cuda)
    y1 = ops.linear(x, w)
    with torch.no_grad():
        w.mul_(2.0)
    y2 = ops.linear(x, w)
    assert _rel(y2, 2.0 * y1) < 1e-5


# ------------------------------------------------------------------------------------------ conv3x3 (bf16x3 implicit GEMM)
@pytest.mark.parametrize("case", [
    dict(n=2, h=60, w=108, src=[256], cout=384, slope=0.2),                     # encoder conv 4
    dict(n=1, h=30, w=54, src=[128, 128, 128, 4], cout=128, slope=0.1),         # offset-head conv 0 (4 sources, 4-ch flows)
    dict(n=2, h=20, w=36, src=[256, 384], cout=512, groups=2, slope=0.2),       # encoder conv 5 (grouped concat)
    dict(n=1, h=17, w=23, src=[256, 512], cout=384, groups=4, slope=0.2),       # encoder conv 6: 96 out ch / group
    dict(n=1, h=9, w=19, src=[256, 384], cout=256, groups=8, slope=0.2),        # conv 7: 32+48 ch / group (chunk spill)
    dict(n=1, h=12, w=20, src=[128], cout=128, residual=True),                  # backbone conv 2 (+ residual)
    dict(n=1, h=24, w=40, src=[64], cout=3),                                    # last decoder conv (3 output channels)
    dict(n=1, h=10, w=14, src=[128], cout=432),                                 # offset-head conv 6
    dict(n=1, h=7, w=5, src=[8], cout=16),                                      # tiny
    # low-Cout layers on the generic kernel: the HALO kernel's resident weights leave room for its halo ring only with
    # Cout <= 32 and ONE 64-channel K chunk (tests/test_gpu_schedules.py covers it); these four run conv3x3_kernel
    dict(n=3, h=40, w=44, src=[64], cout=64, slope=0.2),                        # encoder conv 1 / decoder conv 4 shape, BN = 64
    dict(n=2, h=33, w=21, src=[32, 16], cout=40, residual=True, slope=0.1),     # 2 sources, residual, BN = 64
    dict(n=1, h=16, w=8, src=[128], cout=16),                                   # 2 K chunks, BN = 32
    dict(n=2, h=50, w=30, src=[64, 64], cout=24),                               # 2 chunks from 2 sources, BN = 32
])
def test_conv3x3_bf16x3(cuda, case):
    F = torch.nn.functional
    g = torch.Generator().manual_seed(51)
    n, h, w, groups = case["n"], case["h"], case["w"], case.get("groups", 1)
    srcs = [torch.randn(n, c, h, w, generator=g) for c in case["src"]]
    cin = sum(case["src"])
    weight = torch.nn.Parameter(torch.randn(case["cout"], cin // groups, 3, 3, generator=g) / (9 * cin / groups) ** 0.5)
    bias = torch.randn(case["cout"], generator=g) * 0.1
    res = torch.randn(n, case["cout"], h, w, generator=g) if case.get("residual") else None
    if groups == 1:
        x = torch.cat(srcs, 1)
    else:
        x = torch.cat([s.reshape(n, groups, -1, h, w) for s in srcs], 2).reshape(n, -1, h, w)
    want = F.leaky_relu(F.conv2d(x.double(), weight.detach().double(), bias.double(), 1, 1, 1, groups),
                        case.get("slope", 1.0))
    if res is not None:
        want = want + res.double()
    wd = torch.nn.Parameter(weight.detach().to(cuda))
    got = ops.conv3x3([s.to(cuda).contiguous(memory_format=torch.channels_last) for s in srcs], wd, bias.to(cuda),
                      groups=groups, negative_slope=case.get("slope", 1.0),
                      residual=None if res is None else res.to(cuda))
    assert got.shape == want.shape
    assert _rel(got.cpu(), want) < 5e-5, _rel(got.cpu(), want)


# ------------------------------------------------------------------------------------------ fused producers
def _join(sp):
    return sp.hi.float() + sp.lo.float()


def test_upsample2x_split(cuda):
    F = torch.nn.functional
    g = torch.Generator().manual_seed(61)
    for shape in [(2, 64, 30, 54), (1, 128, 7, 9), (3, 8, 1, 5)]:
        x = torch.randn(*shape, generator=g)
        want = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        got = ops.upsample2x_split(x.to(cuda).contiguous(memory_format=torch.channels_last))
        assert got.shape == tuple(want.shape)
        back = _join(got).permute(0, 3, 1, 2).cpu()
        # bf16 two-term split keeps ~2^-17 relative; interpolation weights differ by fp32 rounding only
        assert (back - want).abs().max().item() < 5e-5


def test_layer_norm_split(cuda):
    F = torch.nn.functional
    g = torch.Generator().manual_seed(62)
    x = torch.randn(3, 5, 7, 512, generator=g) * 3 + 0.5
    w, b = torch.randn(512, generator=g), torch.randn(512, generator=g)
    want = F.layer_norm(x.double(), (512,), w.double(), b.double(), 1e-5)
    y32, ysp = ops.layer_norm(x.to(cuda), w.to(cuda), b.to(cuda), 1e-5, out="both")
    assert (y32.cpu() - want).abs().max().item() < 2e-5
    assert (_join(ysp).cpu() - want).abs().max().item() < 1e-4
    only = ops.layer_norm(x.to(cuda), w.to(cuda), b.to(cuda), 1e-5, out="split")
    assert torch.equal(only.hi, ysp.hi) and torch.equal(only.lo, ysp.lo)


def test_t2t_unfold_split_and_conv_split_outputs(cuda):
    F = torch.nn.functional
    g = torch.Generator().manual_seed(63)
    img = torch.randn(2, 40, 30, 54, generator=g)
    want = F.gelu(F.unfold(img, (7, 7), padding=(3, 3), stride=(3, 3)).permute(0, 2, 1))
    sp = ops.t2t_unfold(img.to(cuda), (7, 7), (3, 3), (3, 3), gelu=True, out="split")
    assert (_join(sp).cpu() - want).abs().max().item() < 5e-5
    # a Linear fed by the split equals the Linear fed by the fp32 tensor
    w = torch.nn.Parameter(torch.randn(64, 1960, generator=g).to(cuda) / 44.0)
    a = ops.linear(sp, w)
    b = ops.linear(want.to(cuda), w)
    assert _rel(a, b) < 2e-5
    # conv3x3 split / both outputs
    x = torch.randn(1, 64, 12, 20, generator=g).to(cuda).contiguous(memory_format=torch.channels_last)
    cw = torch.nn.Parameter(torch.randn(128, 64, 3, 3, generator=g).to(cuda) / 24.0)
    f32, both_sp = ops.conv3x3([x], cw, None, negative_slope=0.2, out="both")
    only_sp = ops.conv3x3([x], cw, None, negative_slope=0.2, out="split")
    assert torch.equal(both_sp.hi, only_sp.hi) and torch.equal(both_sp.lo, only_sp.lo)
    assert (_join(only_sp).permute(0, 3, 1, 2) - f32).abs().max().item() < 5e-5 * f32.abs().max().item() + 1e-6
    chained = ops.conv3x3([only_sp], torch.nn.Parameter(torch.randn(8, 128, 3, 3, generator=g).to(cuda) / 34.0))
    ref = ops.conv3x3([f32], torch.nn.Parameter(torch.randn(8, 128, 3, 3, generator=torch.Generator().manual_seed(63)).to(cuda)))
    assert chained.shape == ref.shape == (1, 8, 12, 20)


def test_deform_align_fused_grouped_layout(cuda):
    """The group-major input layout (dcn_pack_input) gives the same result as the NHWC path."""
    g = torch.Generator().manual_seed(71)
    n, h, w = 2, 14, 22
    a = torch.randn(n, 128, h, w, generator=g).to(cuda)
    b = torch.randn(n, 128, h, w, generator=g).to(cuda)
    head = (torch.randn(n, 432, h, w, generator=g) * 1.5).to(cuda)
    f1 = (torch.randn(n, 2, h, w, generator=g) * 2).to(cuda)
    f2 = (torch.randn(n, 2, h, w, generator=g) * 2).to(cuda)
    wp = ops.pack_dcn_weight((torch.randn(128, 256, 3, 3, generator=g) / 48.0).to(cuda), 16)
    bias = (torch.randn(128, generator=g) * 0.1).to(cuda)
    ref = ops.deform_align_fused(torch.cat([a, b], 1), head, f1, f2, wp, bias, 16, 10.0)
    got = ops.deform_align_fused(ops.dcn_pack_input(a, b), head, f1, f2, wp, bias, 16, 10.0)
    assert torch.equal(ref, got)          # identical arithmetic, only the addressing differs


@pytest.mark.parametrize("case", [
    dict(n=2, h=60, w=108, cin=64, cout=128, ks=3, stride=2),      # encoder conv 2 (stride 2)
    dict(n=1, h=48, w=88, cin=3, cout=64, ks=3, stride=2),         # encoder conv 0: 3 input channels, stride 2
    dict(n=1, h=17, w=23, cin=8, cout=16, ks=3, stride=2),         # odd sizes with stride 2
    dict(n=2, h=32, w=64, cin=8, cout=32, ks=7, stride=1),         # SPyNet level conv 0 (7x7)
    dict(n=1, h=4, w=8, cin=32, cout=64, ks=7, stride=1),          # SPyNet coarse level (image smaller than a tile)
    dict(n=3, h=2, w=4, cin=16, cout=2, ks=7, stride=1),           # SPyNet coarsest level, 2 output channels
])
def test_conv2d_kxk_stride(cuda, case):
    F = torch.nn.functional
    g = torch.Generator().manual_seed(52)
    n, h, w, cin, cout, ks, stride = (case[k] for k in ("n", "h", "w", "cin", "cout", "ks", "stride"))
    x = torch.randn(n, cin, h, w, generator=g)
    weight = torch.nn.Parameter(torch.randn(cout, cin, ks, ks, generator=g) / (ks * ks * cin) ** 0.5)
    bias = torch.randn(cout, generator=g) * 0.1
    want = F.relu(F.conv2d(x.double(), weight.detach().double(), bias.double(), stride, ks // 2))
    wd = torch.nn.Parameter(weight.detach().to(cuda))
    got = ops.conv3x3([x.to(cuda).contiguous(memory_format=torch.channels_last)], wd, bias.to(cuda),
                      negative_slope=0.0, stride=stride)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert _rel(got.cpu(), want) < 5e-5, _rel(got.cpu(), want)


# ------------------------------------------------------------------------------------------ window-packed small-channel convs
@pytest.mark.parametrize("case", [
    dict(n=2, h=32, w=64, cin=8, cout=32, ks=7, stride=1, out="rows"),      # SPyNet conv 0 -> row-gapped 32 channels
    dict(n=2, h=13, w=21, cin=32, cout=64, ks=7, stride=1, out="split"),    # SPyNet conv 1, ragged tile, 4 chunks/row
    dict(n=1, h=4, w=8, cin=32, cout=16, ks=7, stride=1, out="rows"),       # SPyNet conv 3, image smaller than a tile
    dict(n=3, h=2, w=4, cin=16, cout=2, ks=7, stride=1, out="f32"),         # SPyNet conv 4, coarsest level
    dict(n=2, h=30, w=54, cin=3, cout=64, ks=3, stride=2, out="split"),     # encoder stem: 3 channels in a 4-channel row
    dict(n=1, h=17, w=33, cin=3, cout=64, ks=3, stride=2, out="f32"),       # ... odd input size
    dict(n=1, h=9, w=20, cin=5, cout=8, ks=3, stride=1, out="rows"),        # 5 channels padded to 8, 3x3
    dict(n=1, h=12, w=40, cin=8, cout=24, ks=5, stride=2, out="f32"),       # 5x5 stride 2, one chunk per kernel row
    dict(n=1, h=12, w=40, cin=16, cout=8, ks=7, stride=2, out="rows"),      # stride 2, PX=4, 2 chunks per kernel row
])
def test_conv_rows_window_packed(cuda, case):
    """Window-packed K on the row-gapped layout equals F.conv2d (fp64) to bf16x3 accuracy; row-gapped outputs carry
    zero gaps / tail and the right content."""
    F = torch.nn.functional
    g = torch.Generator().manual_seed(77)
    n, h, w, cin, cout, ks, stride = (case[k] for k in ("n", "h", "w", "cin", "cout", "ks", "stride"))
    pad = ks // 2
    x = torch.randn(n, cin, h, w, generator=g)
    weight = torch.nn.Parameter(torch.randn(cout, cin, ks, ks, generator=g) / (ks * ks * cin) ** 0.5)
    bias = torch.randn(cout, generator=g) * 0.1
    want = F.relu(F.conv2d(x.double(), weight.detach().double(), bias.double(), stride, pad))
    wd = torch.nn.Parameter(weight.detach().to(cuda))
    rows = ops.pack_rows(x.to(cuda), lead=pad)
    assert rows.cin == ops.rows_channels(cin) and rows.lead == pad
    assert (rows.dense().cpu() - x).abs().max().item() < 4e-5           # bf16 two-term split of the input
    got = ops.conv3x3(rows, wd, bias.to(cuda), negative_slope=0.0, stride=stride, out=case["out"], out_lead=2)
    if case["out"] == "rows":
        ho, wo = want.shape[2:]
        assert got.shape == tuple(want.shape) and got.lead == 2 and got.cin == cout
        body = (got.hi.float() + got.lo.float())
        tail = ops._lib.load().e2f_conv_rows_tail(2, cout)
        assert body.numel() == (n * ho * (wo + 2) + tail) * cout
        grid = body[: n * ho * (wo + 2) * cout].view(n, ho, wo + 2, cout)
        assert float(grid[:, :, :2].abs().max()) == 0.0 and float(body[n * ho * (wo + 2) * cout:].abs().max()) == 0.0
        got = got.dense()
    elif case["out"] == "split":
        got = _join(got).permute(0, 3, 1, 2)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert _rel(got.cpu(), want) < 5e-5, _rel(got.cpu(), want)
    # same result as the tap-per-chunk path on the dense layout
    dense = ops.conv3x3([x.to(cuda)], wd, bias.to(cuda), negative_slope=0.0, stride=stride)
    assert _rel(got.cpu(), dense.cpu().double()) < 5e-5


def test_conv_rows_chain_matches_spynet_level(cuda):
    """The five 7x7 convs of one SPyNet level (flow_comp.py:181-215), chained through row-gapped / dense hand-offs."""
    F = torch.nn.functional
    g = torch.Generator().manual_seed(78)
    x = torch.randn(3, 8, 24, 40, generator=g)
    chans = [(8, 32), (32, 64), (64, 32), (32, 16), (16, 2)]
    ws = [torch.randn(co, ci, 7, 7, generator=g) / (49 * ci) ** 0.5 for ci, co in chans]
    bs = [torch.randn(co, generator=g) * 0.1 for _, co in chans]
    want = x.double()
    for i, (wt, b) in enumerate(zip(ws, bs)):
        want = F.conv2d(want, wt.double(), b.double(), 1, 3)
        if i < 4:
            want = F.relu(want)
    y = ops.pack_rows(x.to(cuda), lead=3)
    for i, (wt, b) in enumerate(zip(ws, bs)):
        wd = torch.nn.Parameter(wt.to(cuda))
        if i == 4:
            y = ops.conv3x3(y, wd, b.to(cuda), out="f32")
        elif chans[i + 1][0] <= 32:
            y = ops.conv3x3(y, wd, b.to(cuda), negative_slope=0.0, out="rows", out_lead=3)
        else:
            y = ops.conv3x3(y, wd, b.to(cuda), negative_slope=0.0, out="split")
    assert _rel(y.cpu(), want) < 1e-4, _rel(y.cpu(), want)


def test_conv_rows_argument_errors(cuda):
    x = torch.randn(1, 8, 8, 8, device=cuda)
    w = torch.nn.Parameter(torch.randn(16, 8, 3, 3, device=cuda))
    rows = ops.pack_rows(x, lead=2)                       # lead must equal the conv's padding (1)
    with pytest.raises(ValueError):
        ops.conv3x3(rows, w)
    with pytest.raises(ValueError):
        ops.pack_rows(torch.randn(1, 40, 8, 8, device=cuda), lead=1)
    with pytest.raises(ValueError):
        ops.conv3x3([x], torch.nn.Parameter(torch.randn(64, 8, 3, 3, device=cuda)), out="rows", out_lead=1)   # 64 channels


@pytest.mark.parametrize("shape", [(2, 8, 20, 36, 512, (5, 9)), (1, 3, 10, 18, 512, (5, 9)), (1, 2, 8, 6, 64, (4, 3))])
def test_window_pool(cuda, shape):
    """pool_layers[0] across each window's tokens (tfocal_transformer.py:508-516) from the split LayerNorm output."""
    B, T, H, W, C, (wh, ww) = shape
    g = torch.Generator().manual_seed(91)
    x = torch.randn(B, T, H, W, C, generator=g)
    lin = torch.nn.Linear(wh * ww, 1)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(1, wh * ww, generator=g) / (wh * ww))
        lin.bias.fill_(0.37)
    # reference chain: window_partition_noreshape -> (B,nWh,nWw,T,wh*ww,C) -> Linear over the window axis
    xw = x.view(B, T, H // wh, wh, W // ww, ww, C).permute(0, 2, 4, 1, 3, 5, 6).reshape(B, H // wh, W // ww, T, wh * ww, C)
    want = lin(xw.transpose(4, 5)).flatten(-2).permute(0, 3, 1, 2, 4).detach()          # (B,T,nWh,nWw,C)
    hi, lo = ops.split_bf16(x.to(cuda))
    sp = ops.SplitMat(hi.view(B, T, H, W, C), lo.view(B, T, H, W, C))
    got = ops.window_pool(sp, lin.weight.to(cuda), lin.bias.to(cuda), (wh, ww), out="f32")
    assert got.shape == want.shape
    assert (got.cpu() - want).abs().max().item() < 2e-5
    got_sp = ops.window_pool(sp, lin.weight.to(cuda), lin.bias.to(cuda), (wh, ww), out="split")
    assert (_join(got_sp).cpu() - want).abs().max().item() < 5e-5
    with pytest.raises(ValueError):
        ops.window_pool(ops.SplitMat(hi.view(B, T, H, W, C)[:, :, :-1], lo.view(B, T, H, W, C)[:, :, :-1]),
                        lin.weight.to(cuda), lin.bias.to(cuda), (wh, ww))


@pytest.mark.parametrize("shape", [(2, 8, 20, 36, (5, 9)), (1, 3, 10, 18, (5, 9)), (1, 16, 30, 54, (5, 9))])
def test_layer_norm_pool_fused(cuda, shape):
    """norm1 + pool_layers[0] in one kernel (tfocal_transformer.py:470, :508-516): token rows == LayerNorm, the
    trailing rows == the reference's window pooling of the normalised tokens, ordered (B,T,nWh,nWw)."""
    import torch.nn.functional as F
    B, T, H, W, (wh, ww) = shape
    C = 512
    g = torch.Generator().manual_seed(92)
    x = torch.randn(B, T, H, W, C, generator=g) * 1.7 + 0.3
    gamma = 1.0 + 0.1 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    lin = torch.nn.Linear(wh * ww, 1)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(1, wh * ww, generator=g) / (wh * ww))
        lin.bias.fill_(-0.21)
    yn = F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5)
    xw = yn.view(B, T, H // wh, wh, W // ww, ww, C).permute(0, 2, 4, 1, 3, 5, 6).reshape(B, H // wh, W // ww, T, wh * ww, C)
    want_pool = F.linear(xw.transpose(4, 5), lin.weight.double(), lin.bias.double()).flatten(-2).permute(0, 3, 1, 2, 4)
    rows, n_tok = ops.layer_norm_pool(x.to(cuda), gamma.to(cuda), beta.to(cuda), 1e-5, lin.weight.to(cuda),
                                      lin.bias.to(cuda), (wh, ww))
    assert n_tok == B * T * H * W and rows.shape == (n_tok + B * T * (H // wh) * (W // ww), C)
    got = _join(rows).cpu().double()
    assert (got[:n_tok].view(B, T, H, W, C) - yn).abs().max().item() < 5e-5
    assert (got[n_tok:].view(B, T, H // wh, W // ww, C) - want_pool).abs().max().item() < 5e-5
    with pytest.raises(ValueError):
        ops.layer_norm_pool(x[:, :, :-1].to(cuda), gamma.to(cuda), beta.to(cuda), 1e-5, lin.weight.to(cuda),
                            lin.bias.to(cuda), (wh, ww))


@pytest.mark.parametrize("shape", [(2, 64, 48, 80), (1, 64, 17, 23), (3, 16, 8, 8)])
def test_conv3x3_tanh_nchw(cuda, shape):
    """Decoder output conv + tanh + NCHW store in one epilogue (e2fgvi.py:149-150, :262)."""
    import torch.nn.functional as F
    n, c, h, w = shape
    g = torch.Generator().manual_seed(77)
    x = torch.randn(n, c, h, w, generator=g)
    conv = torch.nn.Conv2d(c, 3, 3, 1, 1)
    with torch.no_grad():
        conv.weight.mul_(3.0)                   # spread the pre-activations over tanh's curved range
    want = torch.tanh(F.conv2d(x.double(), conv.weight.double(), conv.bias.double(), 1, 1))
    conv = conv.to(cuda)
    with torch.no_grad():
        got = ops.conv3x3_tanh_nchw(x.to(cuda), conv.weight, conv.bias)
    assert got.shape == want.shape and got.is_contiguous() and got.dtype == torch.float32
    # pre-activations reach |8| here (weights x3): bf16x3 keeps ~5e-5 of max|pre-activation|, tanh' <= 1
    assert (got.cpu().double() - want).abs().max().item() < 1e-4


@pytest.mark.parametrize("case", [
    dict(n=3, cin=64, cout=32, ks=7, h=64, w=128, out="split", slope=0.0),     # SPyNet conv 2 at the finest level
    dict(n=2, cin=32, cout=16, ks=7, h=17, w=29, out="split", slope=0.0),      # SPyNet conv 3, ragged tiles
    dict(n=5, cin=16, cout=2, ks=7, h=2, w=4, out="f32", residual=True),       # SPyNet conv 4, coarsest level (2x4 pixels)
    dict(n=2, cin=16, cout=2, ks=7, h=32, w=64, out="f32", residual=True),
    dict(n=2, cin=64, cout=3, ks=3, h=48, w=80, out="f32", tanh_nchw=True),    # decoder output conv
    dict(n=1, cin=64, cout=3, ks=3, h=31, w=61, out="f32"),
    dict(n=1, cin=128, cout=24, ks=3, h=9, w=33, out="both", slope=0.2),       # two K chunks, Cout not a power of two
])
def test_conv_kxn(cuda, case):
    """kx-in-N conv kernel (kernel-column taps in the GEMM's N, horizontal shift-add by warp shuffles in the epilogue)
    against F.conv2d in fp64: flow_comp.py:181-215 (64->32, 32->16, 16->2 with the flow_up residual), e2fgvi.py:149-150."""
    import torch.nn.functional as F
    c = dict(slope=1.0, residual=False, tanh_nchw=False)
    c.update(case)
    g = torch.Generator().manual_seed(55)
    x = torch.randn(c["n"], c["cin"], c["h"], c["w"], generator=g)
    conv = torch.nn.Conv2d(c["cin"], c["cout"], c["ks"], 1, c["ks"] // 2)
    res = torch.randn(c["n"], c["cout"], c["h"], c["w"], generator=g) if c["residual"] else None
    want = F.leaky_relu(F.conv2d(x.double(), conv.weight.double(), conv.bias.double(), 1, c["ks"] // 2), c["slope"])
    if res is not None:
        want = want + res.double()
    if c["tanh_nchw"]:
        want = torch.tanh(want)
    conv = conv.to(cuda)
    with torch.no_grad():
        got = ops.conv_kxn(x.to(cuda), conv.weight, conv.bias, negative_slope=c["slope"],
                           residual=None if res is None else res.to(cuda).contiguous(memory_format=torch.channels_last),
                           out=c["out"], tanh_nchw=c["tanh_nchw"])
    outs = got if isinstance(got, tuple) else (got,)
    for o in outs:
        if isinstance(o, ops.SplitNHWC):
            o = (o.hi.float() + o.lo.float()).permute(0, 3, 1, 2)
        assert o.shape == want.shape
        assert _rel(o.cpu(), want) < 5e-5
    if c["tanh_nchw"]:
        assert got.is_contiguous()


@pytest.mark.parametrize("shape", [(2, 12, 20), (1, 60, 108)])
def test_conv_kxn_grouped_two_sources(cuda, shape):
    """Encoder conv 7 (e2fgvi.py:97,103-108): 640 -> 256, groups 8, input = group-wise cat of x0 (256 ch) and the previous
    output (384 ch), on the kx-in-N kernel with one tile per (pixels, group); the cat is never built."""
    import torch.nn.functional as F
    n, h, w = shape
    g = torch.Generator().manual_seed(56)
    x0 = torch.randn(n, 256, h, w, generator=g)
    x1 = torch.randn(n, 384, h, w, generator=g)
    conv = torch.nn.Conv2d(640, 256, 3, 1, 1, groups=8)
    xcat = torch.cat([x0.view(n, 8, -1, h, w), x1.view(n, 8, -1, h, w)], 2).view(n, -1, h, w)
    want = F.leaky_relu(F.conv2d(xcat.double(), conv.weight.double(), conv.bias.double(), 1, 1, 1, 8), 0.2)
    conv = conv.to(cuda)
    with torch.no_grad():
        t32, sp = ops.conv_kxn([x0.to(cuda), x1.to(cuda)], conv.weight, conv.bias, negative_slope=0.2, out="both", groups=8)
        old = ops.conv3x3([x0.to(cuda), x1.to(cuda)], conv.weight, conv.bias, groups=8, negative_slope=0.2)
    assert _rel(t32.cpu(), want) < 5e-5
    assert _rel((sp.hi.float() + sp.lo.float()).permute(0, 3, 1, 2).cpu(), want) < 5e-5
    assert _rel(old.cpu(), want) < 5e-5


# ------------------------------------------------------------------------------------------ SoftSplit / SoftComp as gather convs
@pytest.mark.parametrize("shape", [(3, 128, 60, 108), (2, 64, 15, 27), (1, 128, 45, 81), (2, 128, 30, 54)])
def test_soft_split_matches_unfold_linear(cuda, shape):
    """ops.soft_split (7x7 / stride-3 implicit-GEMM conv, tile 12x10 / 18x7, TMA element strides 3) against
    tfocal_transformer.py:39-46 evaluated literally in fp64 on the CPU."""
    import torch.nn.functional as F
    n, c, h, w = shape
    g = torch.Generator().manual_seed(31)
    x = torch.randn(n, c, h, w, generator=g)
    lin = torch.nn.Linear(c * 49, 512)
    want = F.linear(F.unfold(x.double(), 7, padding=3, stride=3).permute(0, 2, 1), lin.weight.double(), lin.bias.double())
    lin = lin.to(cuda)
    with torch.no_grad():
        got = ops.soft_split(x.to(cuda).contiguous(memory_format=torch.channels_last), lin.weight, lin.bias, 7, 3, 3)
    assert got.shape == want.shape and got.dtype == torch.float32
    # bf16 3-term split: ~2^-17 relative per product, K = 49*C terms
    assert _rel(got.cpu(), want) < 5e-5


@pytest.mark.parametrize("shape", [(3, 60, 108), (2, 15, 27), (1, 45, 81)])
@pytest.mark.parametrize("mode", ["base", "hq"])
def test_soft_comp_matches_linear_fold(cuda, shape, mode):
    """ops.soft_comp (nine-phase transposed conv, bias map, residual, fp32 or split output) against
    tfocal_transformer.py:65-72 / _hq.py:67-79 evaluated literally in fp64 on the CPU."""
    import torch.nn.functional as F
    n, h, w = shape
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    g = torch.Generator().manual_seed(32)
    tok = torch.randn(n, fh, fw, 512, generator=g)
    lin = torch.nn.Linear(512, 128 * 49)
    extra = torch.nn.Parameter(torch.randn(128, h, w, generator=g) * 0.3)
    res = torch.randn(n, 128, h, w, generator=g)
    want = F.fold(F.linear(tok.double().view(n, fh * fw, 512), lin.weight.double(), lin.bias.double()).permute(0, 2, 1),
                  (h, w), 7, padding=3, stride=3)
    lin = lin.to(cuda)
    with torch.no_grad():
        if mode == "base":
            want = want + extra.double() + res.double()
            got = ops.soft_comp(tok.to(cuda), lin.weight, lin.bias, (h, w), 7, 3, 3,
                                bias_map_extra=torch.nn.Parameter(extra.detach().to(cuda)),
                                residual=res.to(cuda).contiguous(memory_format=torch.channels_last))
        else:
            sp = ops.soft_comp(tok.to(cuda), lin.weight, lin.bias, (h, w), 7, 3, 3, out="split")
            got = (sp.hi.float() + sp.lo.float()).permute(0, 3, 1, 2)
    assert got.shape == want.shape
    assert _rel(got.cpu(), want) < 5e-5


# ------------------------------------------------------------------------------------------ propagation vs oracle taps
@pytest.mark.parametrize("fused", [True, False])
def test_bidirectional_propagation_matches_oracle_taps(cuda, fused):
    """BidirectionalPropagation (feat_prop.py:81-149) on the GPU against the CPU oracle, step by step: every
    deformable-alignment output of both sweeps (restate.bidirectional_propagation(..., taps)) and the final fused
    features.  Stress weights: live offset conv (offsets = flow + up to +-10 px), biases, O(1) activations."""
    import importlib
    from e2fgvi_b200.synth import synth_state_dict
    net = importlib.import_module("model.e2fgvi")
    model = net.InpaintGenerator().eval()
    sd = synth_state_dict(model, "stress", 0)
    model.load_state_dict(sd, strict=True)
    prop = model.feat_prop_module.to(cuda)
    prop.fused_prologue = fused
    g = torch.Generator().manual_seed(91)
    b, t, c, h, w = 2, 4, 128, 20, 36
    x = torch.randn(b, t, c, h, w, generator=g) * 0.5
    fb = torch.randn(b, t - 1, 2, h, w, generator=g) * 2.5
    ff = torch.randn(b, t - 1, 2, h, w, generator=g) * 2.5
    taps = []
    with torch.no_grad():
        want = restate.bidirectional_propagation({k: v.double() for k, v in sd.items() if v.is_floating_point()},
                                                 "feat_prop_module", x.double(), fb.double(), ff.double(), taps)
    got_taps = []
    originals = {}
    for name, mod in prop.deform_align.items():
        originals[name] = (mod.align, mod.align_split)

        def recorder(*a, _orig=mod.align, _name=name, **kw):
            out = _orig(*a, **kw)
            got_taps.append((_name, out))
            return out

        def recorder_split(*a, _orig=mod.align_split, _name=name, **kw):      # frame-slice fast path: (fp32, SplitNHWC)
            out = _orig(*a, **kw)
            got_taps.append((_name, out[0]))
            # the bf16 pair written by the DCN epilogue must be the split of the fp32 output
            assert (out[1].hi.float() + out[1].lo.float() - out[0].permute(0, 2, 3, 1)).abs().max().item() < 1e-4
            return out
        mod.align, mod.align_split = recorder, recorder_split
    try:
        with torch.no_grad():
            got = prop(x.to(cuda), fb.to(cuda), ff.to(cuda))
    finally:
        for name, mod in prop.deform_align.items():
            mod.align, mod.align_split = originals[name]
    assert len(got_taps) == len(taps) == 2 * (t - 1)
    for (name, out), tap in zip(got_taps, taps):
        assert name == tap["dir"]
        ref = tap["out"]
        # fp16 operands in the deformable GEMM (see test_modulated_deform_conv2d_unrounded_fp32_oracle); errors of
        # earlier steps propagate through the recurrence, hence 2e-3 of max per step
        rel = (out.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
        assert rel < 2e-3, (name, tap["step"], rel)
    rel = (got.cpu().double() - want).abs().max().item() / want.abs().max().item()
    assert got.shape == want.shape and rel < 2e-3, rel


# ------------------------------------------------------------------------------------------ fused propagation prologue
@pytest.mark.parametrize("second_order", [True, False])
def test_prop_prologue_matches_unfused_sequence(cuda, second_order):
    """ops.prop_prologue == flow_warp x3 + add + split_nhwc + dcn_pack_input (feat_prop.py:106-126), bit for bit."""
    g = torch.Generator().manual_seed(81)
    b, t, c, h, w = 2, 4, 128, 13, 22
    flows = (torch.randn(b, t - 1, 2, h, w, generator=g) * 3).to(cuda)
    prop = torch.randn(b, c, h, w, generator=g).to(cuda).contiguous(memory_format=torch.channels_last)
    feat2 = torch.randn(b, c, h, w, generator=g).to(cuda).contiguous(memory_format=torch.channels_last)
    flow_n1 = flows[:, 1]
    flow_prev = flows[:, 0] if second_order else None
    xg, c1, c2, fl, f1, f2 = ops.prop_prologue(prop, feat2 if second_order else None, flow_n1, flow_prev)
    grid = flow_n1.permute(0, 2, 3, 1)
    want_c1 = ops.split_nhwc(ops.flow_warp(prop, grid))
    if second_order:
        want_f2 = flow_n1 + ops.flow_warp(flows[:, 0], grid)
        want_c2 = ops.split_nhwc(ops.flow_warp(feat2, want_f2.permute(0, 2, 3, 1)))
        want_x = ops.dcn_pack_input(prop, feat2)
    else:
        want_f2 = torch.zeros_like(flow_n1)
        want_c2 = ops.split_nhwc(torch.zeros_like(prop))
        want_x = ops.dcn_pack_input(prop, torch.zeros_like(prop))
    want_fl = ops.split_nhwc(torch.cat([flow_n1, want_f2], 1))
    assert torch.equal(f1, flow_n1) and torch.equal(f2, want_f2)
    for got, want in ((c1, want_c1), (c2, want_c2), (fl, want_fl)):
        assert got.shape == want.shape
        assert torch.equal(got.hi, want.hi) and torch.equal(got.lo, want.lo)
    assert torch.equal(xg.data, want_x.data) and xg.shape == want_x.shape
    assert f1.permute(0, 2, 3, 1).is_contiguous() and f2.permute(0, 2, 3, 1).is_contiguous()
