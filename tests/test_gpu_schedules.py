"""The persistent wgmma kernels past one tile per CTA.

The linear GEMM (gemm.cu), the implicit-GEMM conv with its generic and HALO kernels (conv.cu, 2-D and the I3D 3-D
instantiation) and the kx-in-N conv (conv_kxn.cu) launch min(tiles, SMs) CTAs, and CTA b walks tiles b, b + grid, ...
The ring positions and mbarrier parities carried from tile to tile, the linear kernel's two ping-pong warpgroups
and every epilogue after a CTA's first tile only run when a CTA owns two or more tiles.  Every case here:

* runs under torch.profiler and asserts the kernel instantiation it reaches, grid == min(tiles, SMs) with the tile
  count derived from the launcher's tile arithmetic, and shapes built from the SM count, so the regime (tiles per CTA)
  holds on any H100;
* compares with a float64 reference computed by plain torch on the GPU, twice: the rel-of-max tolerance of
  test_gpu_ops.py, and a per-element bound |got - ref| <= C * A (+ the output format's own rounding), where A is the
  same operation on |x| and |w| plus |bias| and |residual|.  An error confined to small outputs (a tail tile, a lost
  residual, a low-magnitude channel) passes the first check and fails the second.

C = 2^-14.  Each fp32 operand is a bf16 pair hi + lo: |x - hi| <= 2^-8 |x| and the rounding of lo leaves at most
2^-16 |x|, typically 2^-17 or less; the dropped lo.lo product is <= 2^-16 |x||w|, typically 2^-18.  Per product that
is at most 3 * 2^-16 of |x||w| (0.75 C) and on average several times less, and the fp32 accumulation adds
a few 2^-24 of A per accumulator update, whose errors largely cancel over long K.

No kernel uses atomics or split-K, so an output's arithmetic is fixed by its coordinates: permuting rows (linear) or
images (conv) must permute the result bit for bit.  That is checked at production sizes (the 8-clip step: 46,080
token rows, 64 images), after asserting that both calls ran the same kernel on the same grid.

Reachability (dispatch as of this file): conv3x3_halo_kernel<64> is never chosen (its resident weights leave room for
fewer than three halo slots), nor is the HALO kernel with more than one K chunk; conv_kxn_kernel<true, 7, *> is never
chosen (the kx-in-N halo variant is taken for 3x3 kernels only).  Tests for those paths belong with a change that makes
them reachable."""
import math

import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from kernel_checks import (cdiv as _cdiv, check_close, conv3x3_tanh_nchw_entry, conv_bn, conv_tile, expect_schedule, generic_tiles, halo_tiles, images_for, kxn_tiles, persistent_launch, print_tables, run_traced,
                           same_launch as _same_launch, sms)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def schedule_table():
    yield
    print_tables()


# ------------------------------------------------------------------------------------------------ linear
def _linear_case(s, name):
    """(m, k, n, bias, residual, out, expected tiles) of each named regime; S = SM count."""
    return {
        # tiles per CTA exactly 1 on a full grid, K = 8: one K block
        "tiles=S k=8": (128 * s, 8, 128, True, False, "f32", s),
        # CTA 0's second tile is the M-tail tile; residual; K = 64: one K block
        "tiles=S+1 Mtail res k=64": (128 * s + 37, 64, 128, True, True, "f32", s + 1),
        # no bias, fp16, M and N tails, 2 K blocks
        "tiles=2S Mtail Ntail nobias f16 kb=2": (128 * s - 5, 128, 200, False, False, "f16", 2 * s),
        # residual, N tail of 96, 3 K blocks (= STAGES)
        "tiles=2S+1 Ntail res kb=3": (128 * (2 * s + 1), 192, 96, True, True, "f32", 2 * s + 1),
        # mlp.conv2's K = 1960: 31 K blocks with a K tail; residual; N = 124
        "tiles=3S-1 Ktail kb=31 res": (128 * (3 * s - 1) - 100, 1960, 124, True, True, "f32", 3 * s - 1),
        # residual without bias, M tail of one row
        "tiles=3S res nobias kb=2": (128 * (3 * s - 1) + 1, 128, 128, False, True, "f32", 3 * s),
        # >= 5S + r: fp16 with residual, 5 N tiles with a tail, 4 K blocks
        "tiles=5S+5 f16 res kb=4": (128 * (s + 1), 256, 600, True, True, "f16", 5 * s + 5),
        # 4 output columns of a 128-wide tile, one K block of 8
        "tiles=2S+1 N=4 k=8": (128 * (2 * s + 1) - 3, 8, 4, True, False, "f32", 2 * s + 1),
    }[name]


LINEAR_CASES = ["tiles=S k=8", "tiles=S+1 Mtail res k=64", "tiles=2S Mtail Ntail nobias f16 kb=2",
                "tiles=2S+1 Ntail res kb=3", "tiles=3S-1 Ktail kb=31 res", "tiles=3S res nobias kb=2",
                "tiles=5S+5 f16 res kb=4", "tiles=2S+1 N=4 k=8"]


def _linear_tiles(m, n):
    return _cdiv(m, 128) * _cdiv(n, 128)


def _linear_ref(x64, w64, b64, r64):
    """(reference, bound A) in float64."""
    ref = F.linear(x64, w64, b64)
    bound = F.linear(x64.abs(), w64.abs(), None if b64 is None else b64.abs())
    if r64 is not None:
        ref, bound = ref + r64, bound + r64.abs()
    return ref, bound


@pytest.mark.parametrize("case", LINEAR_CASES)
def test_linear_multi_tile(cuda, case):
    m, k, n, has_bias, has_res, out, tiles = _linear_case(sms(), case)
    assert _linear_tiles(m, n) == tiles
    g = torch.Generator(device=cuda).manual_seed(101)
    x = torch.randn(m, k, device=cuda, generator=g) * 2.0
    w = torch.nn.Parameter(torch.randn(n, k, device=cuda, generator=g) / k ** 0.5)
    b = torch.randn(n, device=cuda, generator=g) if has_bias else None
    r = torch.randn(m, n, device=cuda, generator=g) if has_res else None
    dt = torch.float16 if out == "f16" else torch.float32
    got, launches = run_traced(lambda: ops.linear(x, w, b, r, out_dtype=dt))
    kernel = "linear_kernel<__half>" if out == "f16" else "linear_kernel<float>"
    expect_schedule(f"linear {case}", persistent_launch(launches), kernel, tiles)
    ref, bound = _linear_ref(x.double(), w.detach().double(), None if b is None else b.double(),
                             None if r is None else r.double())
    check_close(got, ref, bound, 1.5e-3 if out == "f16" else 5e-5, out, "linear " + case)


def test_linear_split_operand_with_pitch(cuda):
    """A ``SplitMat`` from t2t_fold_unfold with padded rows (pitch 1992 for K = 1960: 32 K blocks, the last one
    8 zero columns + zero fill), residual and bias, >= 2S + 1 tiles (mlp.conv2 of the FFN)."""
    s = sms()
    c, h, w = 40, 60, 108
    fh, fw = 20, 36
    ck = c * 49
    pitch = (ck + 63) // 64 * 64 + 8
    n = 512
    bt = 1
    while _linear_tiles(bt * fh * fw, n) < 2 * s + 1:
        bt += 1
    m = bt * fh * fw
    g = torch.Generator(device=cuda).manual_seed(102)
    tok = torch.randn(bt, fh * fw, ck, device=cuda, generator=g)
    sp = ops.t2t_fold_unfold(tok, (h, w), (7, 7), (3, 3), (3, 3), gelu=True, out="split", pitch=pitch)
    wl = torch.nn.Parameter(torch.randn(n, ck, device=cuda, generator=g) / ck ** 0.5)
    b = torch.randn(n, device=cuda, generator=g)
    r = torch.randn(bt, fh * fw, n, device=cuda, generator=g)
    got, launches = run_traced(lambda: ops.linear(sp, wl, b, r))
    expect_schedule("linear SplitMat pitch=1992 kb=32 res", persistent_launch(launches), "linear_kernel<float>",
                    _linear_tiles(m, n))
    x64 = (sp.hi.double() + sp.lo.double())[..., :ck].reshape(m, ck)
    ref, bound = _linear_ref(x64, wl.detach().double(), b.double(), r.double().reshape(m, n))
    check_close(got.reshape(m, n), ref, bound, 5e-5, "f32", "split pitch")


# ------------------------------------------------------------------------------------------------ conv
def conv_ref(x64, w64, b64, groups=1, stride=1, pad=1, slope=1.0, r64=None, tanh=False):
    """(reference, bound A) of leaky_relu(conv(x) + b) (+ r) (-> tanh) in float64.  LeakyReLU and tanh are
    1-Lipschitz, so the pre-activation's bound holds after them."""
    pre = F.conv2d(x64, w64, b64, stride, pad, 1, groups)
    bound = F.conv2d(x64.abs(), w64.abs(), None if b64 is None else b64.abs(), stride, pad, 1, groups)
    ref = F.leaky_relu(pre, slope)
    if r64 is not None:
        ref, bound = ref + r64, bound + r64.abs()
    if tanh:
        ref = torch.tanh(ref)
    return ref, bound


def _group_cat(srcs, groups):
    if groups == 1:
        return torch.cat(srcs, 1)
    n, _, h, w = srcs[0].shape
    return torch.cat([s.reshape(n, groups, -1, h, w) for s in srcs], 2).reshape(n, -1, h, w)


def _conv_operands(cuda, seed, n, src, h, w, cout, cin_g, ks, res_hw=None, bias=True):
    g = torch.Generator(device=cuda).manual_seed(seed)
    srcs = [torch.randn(n, c, h, w, device=cuda, generator=g) for c in src]
    weight = torch.nn.Parameter(torch.randn(cout, cin_g, ks, ks, device=cuda, generator=g) / (ks * ks * cin_g) ** 0.5)
    b = torch.randn(cout, device=cuda, generator=g) * 0.1 if bias else None
    res = torch.randn(n, cout, *res_hw, device=cuda, generator=g) if res_hw else None
    return srcs, weight, b, res


def _joined(sp):
    return (sp.hi.double() + sp.lo.double()).permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ generic conv
GENERIC_CASES = {
    # BN 32: two sources (2 K chunks: too many weights for the HALO kernel), residual
    "bn32 2src res": dict(src=[64, 64], cout=32, h=30, w=54, slope=0.1, residual=True, bn=32),
    # BN 64: both outputs
    "bn64 both": dict(src=[128], cout=64, h=30, w=54, slope=0.2, out="both", bn=64),
    # BN 96: encoder conv 6 (groups 4 of 96 outputs, two sources), residual
    "bn96 groups4 2src res": dict(src=[256, 512], cout=384, groups=4, h=17, w=23, slope=0.2, residual=True, bn=96),
    # BN 128: stride 2, two N tiles, residual
    "bn128 stride2 res": dict(src=[128], cout=256, h=60, w=108, stride=2, slope=0.2, residual=True, bn=128),
    # BN 128: encoder conv 5 (groups 2, two sources), both outputs
    "bn128 groups2 2src both": dict(src=[256, 384], cout=512, groups=2, h=20, w=36, slope=0.2, out="both", bn=128),
}


@pytest.mark.parametrize("case", list(GENERIC_CASES))
def test_conv_generic_multi_tile(cuda, case):
    c = dict(groups=1, stride=1, slope=1.0, residual=False, out="f32")
    c.update(GENERIC_CASES[case])
    s, groups, stride = sms(), c["groups"], c["stride"]
    oh, ow = (c["h"] - 1) // stride + 1, (c["w"] - 1) // stride + 1
    n = images_for(lambda k: generic_tiles(k, oh, ow, c["cout"], groups, stride)[1], 2 * s + 1)
    bn, tiles = generic_tiles(n, oh, ow, c["cout"], groups, stride)
    assert bn == c["bn"] and tiles >= 2 * s + 1
    cin_g = sum(c["src"]) // groups
    srcs, weight, b, res = _conv_operands(cuda, 103, n, c["src"], c["h"], c["w"], c["cout"], cin_g, 3,
                                          (oh, ow) if c["residual"] else None)
    got, launches = run_traced(lambda: ops.conv3x3(srcs, weight, b, groups=groups, negative_slope=c["slope"],
                                                   residual=res, out=c["out"], stride=stride))
    expect_schedule(f"conv {case}", persistent_launch(launches), f"conv3x3_kernel<{bn}, false>", tiles)
    ref, bound = conv_ref(_group_cat(srcs, groups).double(), weight.detach().double(), b.double(), groups, stride, 1,
                          c["slope"], None if res is None else res.double())
    if c["out"] == "both":
        t32, sp = got
        check_close(t32, ref, bound, 5e-5, "f32", "conv " + case)
        check_close(_joined(sp), ref, bound, 5e-5, "split", "conv " + case + " split")
    else:
        check_close(got, ref, bound, 5e-5, "f32", "conv " + case)


# ------------------------------------------------------------------------------------------------ HALO conv
HALO_CASES = {
    # ragged 8 x 16 tiles on both axes, residual, 40 channels (one K chunk), 24 outputs (per-element stores)
    "res ragged": dict(src=40, cout=24, h=33, w=21, slope=0.1, residual=True),
    # fp32 + bf16 split outputs, 32 channels (staged stores)
    "both": dict(src=64, cout=32, h=40, w=44, slope=0.2, out="both"),
    # split only, no bias, 8 input channels, ragged tiles
    "split nobias ragged": dict(src=8, cout=16, h=37, w=43, out="split", bias=False),
}


@pytest.mark.parametrize("case", list(HALO_CASES))
def test_conv_halo_multi_tile(cuda, case):
    c = dict(slope=1.0, residual=False, out="f32", bias=True)
    c.update(HALO_CASES[case])
    s = sms()
    n = images_for(lambda k: halo_tiles(k, c["h"], c["w"]), 3 * s)
    tiles = halo_tiles(n, c["h"], c["w"])
    srcs, weight, b, res = _conv_operands(cuda, 104, n, [c["src"]], c["h"], c["w"], c["cout"], c["src"], 3,
                                          (c["h"], c["w"]) if c["residual"] else None, c["bias"])
    got, launches = run_traced(lambda: ops.conv3x3(srcs, weight, b, negative_slope=c["slope"], residual=res,
                                                   out=c["out"]))
    expect_schedule(f"conv HALO {case}", persistent_launch(launches), "conv3x3_halo_kernel<32>", tiles)
    ref, bound = conv_ref(srcs[0].double(), weight.detach().double(), None if b is None else b.double(), 1, 1, 1,
                          c["slope"], None if res is None else res.double())
    if c["out"] == "both":
        check_close(got[0], ref, bound, 5e-5, "f32", "HALO " + case)
        check_close(_joined(got[1]), ref, bound, 5e-5, "split", "HALO " + case + " split")
    elif c["out"] == "split":
        check_close(_joined(got), ref, bound, 5e-5, "split", "HALO " + case)
    else:
        check_close(got, ref, bound, 5e-5, "f32", "HALO " + case)


def test_conv_halo_tanh_nchw_multi_tile(cuda):
    """The decoder output conv (64 -> 3, tanh, NCHW store) on the HALO kernel: the C entry e2f_conv3x3_tanh_nchw goes
    through launch_conv3x3 (ops.conv3x3_tanh_nchw runs this layer on the kx-in-N kernel)."""
    s = sms()
    h, w = 48, 80
    n = images_for(lambda k: halo_tiles(k, h, w), 3 * s)
    (x,), weight, b, _ = _conv_operands(cuda, 105, n, [64], h, w, 3, 64, 3)
    with torch.no_grad():
        weight.mul_(3.0)                       # pre-activations over tanh's curved range
    got, launches = run_traced(lambda: conv3x3_tanh_nchw_entry(x, weight, b))
    expect_schedule("conv HALO tanh/NCHW", persistent_launch(launches), "conv3x3_halo_kernel<32>",
                    halo_tiles(n, h, w))
    assert got.is_contiguous() and got.shape == (n, 3, h, w)
    ref, bound = conv_ref(x.double(), weight.detach().double(), b.double(), tanh=True)
    # as test_conv3x3_tanh_nchw: pre-activations reach |8| while |out| <= 1, so the output is held to 1e-4 of its max
    check_close(got, ref, bound, 1e-4, "f32", "HALO tanh")


# ------------------------------------------------------------------------------------------------ kx-in-N conv
KXN_CASES = {
    # SPyNet conv 2 (64 -> 32, 7x7): split output
    "7x7 64->32 split": dict(cin=[64], cout=32, ks=7, h=64, w=128, out="split", slope=0.0, kernel="<false, 7, 32>"),
    # SPyNet conv 3 (32 -> 16), ragged tiles
    "7x7 32->16 split ragged": dict(cin=[32], cout=16, ks=7, h=17, w=29, out="split", slope=0.0,
                                    kernel="<false, 7, 16>"),
    # SPyNet conv 4 (16 -> 2) + the flow residual
    "7x7 16->2 res": dict(cin=[16], cout=2, ks=7, h=32, w=64, residual=True, kernel="<false, 7, 16>"),
    # decoder output conv: tanh + NCHW store
    "3x3 64->3 tanh nchw": dict(cin=[64], cout=3, ks=3, h=48, w=80, tanh=True, kernel="<false, 3, 16>"),
    # one K chunk, 24 outputs, residual, both outputs
    "3x3 64->24 res both": dict(cin=[64], cout=24, ks=3, h=31, w=61, residual=True, out="both", slope=0.2,
                                kernel="<false, 3, 32>"),
    # two K chunks: the halo variant, residual
    "3x3 128->16 res halo": dict(cin=[128], cout=16, ks=3, h=30, w=54, residual=True, kernel="<true, 3, 16>"),
    # two K chunks, tanh + NCHW on the halo variant
    "3x3 128->3 tanh nchw halo": dict(cin=[128], cout=3, ks=3, h=24, w=40, tanh=True, kernel="<true, 3, 16>"),
    # two K chunks, both outputs
    "3x3 128->24 both halo": dict(cin=[128], cout=24, ks=3, h=9, w=33, out="both", slope=0.2,
                                  kernel="<true, 3, 32>"),
    # encoder conv 7: groups 8, two sources, the group-wise cat never built
    "3x3 grouped 2src halo": dict(cin=[256, 384], cout=256, groups=8, ks=3, h=12, w=20, out="both", slope=0.2,
                                  kernel="<true, 3, 32>"),
}


@pytest.mark.parametrize("case", list(KXN_CASES))
def test_conv_kxn_multi_tile(cuda, case):
    c = dict(groups=1, slope=1.0, residual=False, out="f32", tanh=False)
    c.update(KXN_CASES[case])
    s, groups, ks = sms(), c["groups"], c["ks"]
    n = images_for(lambda k: kxn_tiles(k, c["h"], c["w"], ks, groups), 2 * s)
    tiles = kxn_tiles(n, c["h"], c["w"], ks, groups)
    cin_g = sum(c["cin"]) // groups
    srcs, weight, b, res = _conv_operands(cuda, 106, n, c["cin"], c["h"], c["w"], c["cout"], cin_g, ks,
                                          (c["h"], c["w"]) if c["residual"] else None)
    if c["tanh"]:
        with torch.no_grad():
            weight.mul_(3.0)
    if res is not None:
        res = res.contiguous(memory_format=torch.channels_last)
    x = srcs if len(srcs) > 1 else srcs[0]
    with torch.no_grad():
        got, launches = run_traced(lambda: ops.conv_kxn(x, weight, b, negative_slope=c["slope"], residual=res,
                                                        out=c["out"], tanh_nchw=c["tanh"], groups=groups))
    expect_schedule(f"kxn {case}", persistent_launch(launches), "conv_kxn_kernel" + c["kernel"], tiles)
    ref, bound = conv_ref(_group_cat(srcs, groups).double(), weight.detach().double(), b.double(), groups, 1, ks // 2,
                          c["slope"], None if res is None else res.double(), c["tanh"])
    # tanh: held to 1e-4 of its O(1) max as in test_conv3x3_tanh_nchw (pre-activations reach |8|)
    tol = 1e-4 if c["tanh"] else 5e-5
    if c["tanh"]:
        assert got.is_contiguous()
    if c["out"] == "both":
        check_close(got[0], ref, bound, tol, "f32", "kxn " + case)
        check_close(_joined(got[1]), ref, bound, tol, "split", "kxn " + case + " split")
    elif c["out"] == "split":
        check_close(_joined(got), ref, bound, tol, "split", "kxn " + case)
    else:
        check_close(got, ref, bound, tol, "f32", "kxn " + case)


# ------------------------------------------------------------------------------------------------ I3D 3-D conv
def _unit3d(cin, cout, k, seed):
    from e2fgvi_b200.i3d import Unit3D
    u = Unit3D(cin, cout, (k,) * 3)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        u.conv3d.weight.normal_(0, (2.0 / (cin * k ** 3)) ** 0.5, generator=g)
        u.bn.weight.copy_(1 + 0.1 * torch.randn(cout, generator=g))
        u.bn.bias.copy_(0.1 * torch.randn(cout, generator=g))
        u.bn.running_mean.copy_(0.1 * torch.randn(cout, generator=g))
        u.bn.running_var.copy_(1 + 0.3 * torch.rand(cout, generator=g))
    return u


def _conv3d_call(cuda, u, x, b, size, coff, wide, fill=7.0):
    from e2fgvi_b200.i3d import InceptionI3d, _Act
    hi, lo = ops.split_bf16(x)
    out = InceptionI3d._alloc(b, size, wide, cuda)
    out.f32.fill_(fill)
    InceptionI3d()._conv(u, _Act(None, hi, lo, size, x.shape[-1]), b, out, coff)
    return out


def conv3d_tiles(b, size, cout):
    tw, th = conv_tile(size[1], size[2])
    bn = conv_bn(cout)
    return bn, b * size[0] * _cdiv(size[1], th) * _cdiv(size[2], tw) * _cdiv(cout, bn)


@pytest.mark.parametrize("cin,cout,k", [(64, 64, 1), (192, 96, 1), (16, 32, 3), (64, 192, 3)])
def test_conv3d_multi_tile(cuda, cin, cout, k):
    """Unit3D (conv, folded BN, ReLU) into a channel slice of a wider output, >= 2S tiles.  1x1x1 with 64 input
    channels is one K block per tile, fewer than the pipeline's stages."""
    from e2fgvi_b200.i3d import same_pad
    s = sms()
    size = (4, 28, 28)
    b = images_for(lambda k: conv3d_tiles(k, size, cout)[1], 2 * s)
    bn, tiles = conv3d_tiles(b, size, cout)
    u = _unit3d(cin, cout, k, cin + cout).to(cuda).eval()
    x = torch.randn((b,) + size + (cin,), device=cuda, generator=torch.Generator(device=cuda).manual_seed(107)).relu_()
    coff, wide = 8, cout + 24
    out, launches = run_traced(lambda: _conv3d_call(cuda, u, x, b, size, coff, wide))
    expect_schedule(f"conv3d {cin}->{cout} k{k}", persistent_launch(launches), f"conv3x3_kernel<{bn}, true>", tiles)
    pads, _ = same_pad((k,) * 3, (1, 1, 1), size)
    x64 = F.pad(x.permute(0, 4, 1, 2, 3).double(), [pads[4], pads[5], pads[2], pads[3], pads[0], pads[1]])
    bnm = u.bn
    scale = bnm.weight.double() / torch.sqrt(bnm.running_var.double() + bnm.eps)
    wf = u.conv3d.weight.double() * scale.view(-1, 1, 1, 1, 1)
    bf = bnm.bias.double() - bnm.running_mean.double() * scale
    ref = F.conv3d(x64, wf, bf).relu().permute(0, 2, 3, 4, 1)
    bound = F.conv3d(x64.abs(), wf.abs(), bf.abs()).permute(0, 2, 3, 4, 1)
    check_close(out.f32[..., coff:coff + cout], ref, bound, 1e-4, "f32", f"conv3d {cin}->{cout} k{k}")
    check_close(out.hi[..., coff:coff + cout].double() + out.lo[..., coff:coff + cout].double(), ref, bound, 1e-4,
                "split", f"conv3d {cin}->{cout} k{k} split")
    assert torch.all(out.f32[..., :coff] == 7.0) and torch.all(out.f32[..., coff + cout:] == 7.0)


# ------------------------------------------------------------------------------------------------ bitwise schedule invariance
def test_linear_row_permutation_bitwise(cuda):
    """attn.qkv (fp16) and attn.proj (+ residual, fp32) of the 8-clip step, M = 46,080 token rows: permuting the rows
    permutes the result bit for bit; sampled rows equal a one-row call."""
    g = torch.Generator(device=cuda).manual_seed(108)
    m = 8 * 5760
    x = torch.randn(m, 512, device=cuda, generator=g)
    perm = torch.randperm(m, device=cuda, generator=g)
    wq = torch.nn.Parameter(torch.randn(1536, 512, device=cuda, generator=g) / 512 ** 0.5)
    bq = torch.randn(1536, device=cuda, generator=g)
    y, la = run_traced(lambda: ops.linear(x, wq, bq, out_dtype=torch.float16))
    yp, lb = run_traced(lambda: ops.linear(x[perm], wq, bq, out_dtype=torch.float16))
    k = _same_launch(la, lb)
    expect_schedule("linear attn.qkv M=46080 (permutation)", k, "linear_kernel<__half>", _linear_tiles(m, 1536))
    assert torch.equal(y[perm], yp)
    for i in torch.randint(0, m, (6,), device=cuda, generator=g).tolist() + [0, m - 1]:
        y1, l1 = run_traced(lambda: ops.linear(x[i:i + 1], wq, bq, out_dtype=torch.float16))
        assert persistent_launch(l1).name == k.name
        assert torch.equal(y1[0], y[i]), i
    wp = torch.nn.Parameter(torch.randn(512, 512, device=cuda, generator=g) / 512 ** 0.5)
    bp = torch.randn(512, device=cuda, generator=g)
    r = torch.randn(m, 512, device=cuda, generator=g)
    z, la = run_traced(lambda: ops.linear(x, wp, bp, r))
    zp, lb = run_traced(lambda: ops.linear(x[perm], wp, bp, r[perm]))
    expect_schedule("linear attn.proj M=46080 res (permutation)", _same_launch(la, lb), "linear_kernel<float>",
                    _linear_tiles(m, 512))
    assert torch.equal(z[perm], zp)


def _perm_check(cuda, case, fn, x_list, res, kernel, tiles, seed):
    """fn(sources, residual) on the batch and on a permutation of its images: bitwise equal after permuting."""
    n = x_list[0].shape[0]
    perm = torch.randperm(n, device=cuda, generator=torch.Generator(device=cuda).manual_seed(seed))
    a, la = run_traced(lambda: fn(x_list, res))
    b, lb = run_traced(lambda: fn([t[perm] for t in x_list], None if res is None else res[perm]))
    expect_schedule(case, _same_launch(la, lb), kernel, tiles)
    outs_a = a if isinstance(a, tuple) else (a,)
    outs_b = b if isinstance(b, tuple) else (b,)
    for oa, ob in zip(outs_a, outs_b):
        if isinstance(oa, ops.SplitNHWC):
            assert torch.equal(oa.hi[perm], ob.hi) and torch.equal(oa.lo[perm], ob.lo), case
        else:
            assert torch.equal(oa[perm], ob), case


def test_conv_image_permutation_bitwise(cuda):
    """Generic, HALO, kx-in-N convs at 64 images (8 clips x 8 frames) of the 432 x 240 model: permuting the images
    permutes the result bit for bit."""
    n = 64
    g = torch.Generator(device=cuda).manual_seed(109)

    def param(*shape):
        return torch.nn.Parameter(torch.randn(*shape, device=cuda, generator=g) / math.sqrt(math.prod(shape[1:])))

    def rnd(*shape):
        return torch.randn(*shape, device=cuda, generator=g)

    # encoder conv 4: 256 -> 384 at 60 x 108 (BN 128, 3 N tiles)
    x = rnd(n, 256, 60, 108).contiguous(memory_format=torch.channels_last)
    w4, b4 = param(384, 256, 3, 3), rnd(384)
    bn, tiles = generic_tiles(n, 60, 108, 384)
    _perm_check(cuda, "perm conv encoder4 n=64", lambda xs, r: ops.conv3x3(xs, w4, b4, negative_slope=0.2),
                [x], None, f"conv3x3_kernel<{bn}, false>", tiles, 1)
    # encoder conv 2: 64 -> 128, stride 2, from 120 x 216, split output
    x = rnd(n, 64, 120, 216).contiguous(memory_format=torch.channels_last)
    w2, b2 = param(128, 64, 3, 3), rnd(128)
    bn, tiles = generic_tiles(n, 60, 108, 128, stride=2)
    _perm_check(cuda, "perm conv encoder2 s2 n=64", lambda xs, r: ops.conv3x3(xs, w2, b2, negative_slope=0.2,
                                                                             stride=2, out="both"),
                [x], None, f"conv3x3_kernel<{bn}, false>", tiles, 2)
    # HALO: 64 -> 32 at 60 x 108 with a residual
    x = rnd(n, 64, 60, 108).contiguous(memory_format=torch.channels_last)
    wh, bh = param(32, 64, 3, 3), rnd(32)
    res = rnd(n, 32, 60, 108)
    _perm_check(cuda, "perm conv HALO 64->32 res n=64",
                lambda xs, r: ops.conv3x3(xs, wh, bh, negative_slope=0.1, residual=r, out="both"),
                [x], res, "conv3x3_halo_kernel<32>", halo_tiles(n, 60, 108), 3)
    # kx-in-N: decoder output conv 64 -> 3 (tanh, NCHW) at 240 x 432, and encoder conv 7 (groups 8, two sources)
    x = rnd(n, 64, 240, 432)
    wd, bd = param(3, 64, 3, 3), rnd(3)
    with torch.no_grad():
        _perm_check(cuda, "perm kxn decoder out 240x432 n=64", lambda xs, r: ops.conv3x3_tanh_nchw(xs[0], wd, bd),
                    [x], None, "conv_kxn_kernel<false, 3, 16>", kxn_tiles(n, 240, 432, 3), 4)
        x0, x1 = rnd(n, 256, 60, 108), rnd(n, 384, 60, 108)
        w7, b7 = param(256, 80, 3, 3), rnd(256)
        _perm_check(cuda, "perm kxn encoder7 grouped n=64",
                    lambda xs, r: ops.conv_kxn(xs, w7, b7, negative_slope=0.2, out="both", groups=8),
                    [x0, x1], None, "conv_kxn_kernel<true, 3, 32>", kxn_tiles(n, 60, 108, 3, 8), 5)
        # the same decoder output conv on the HALO kernel (the C entry e2f_conv3x3_tanh_nchw)
        x = rnd(n, 64, 120, 216)
        _perm_check(cuda, "perm HALO tanh/NCHW 120x216 n=64", lambda xs, r: conv3x3_tanh_nchw_entry(xs[0], wd, bd),
                    [x], None, "conv3x3_halo_kernel<32>", halo_tiles(n, 120, 216), 6)


def test_conv3d_video_permutation_bitwise(cuda):
    """I3D 3x3x3 (64 -> 192) over 8 videos: permuting the videos permutes the result bit for bit."""
    b, size = 8, (4, 28, 28)
    u = _unit3d(64, 192, 3, 7).to(cuda).eval()
    x = torch.randn((b,) + size + (64,), device=cuda, generator=torch.Generator(device=cuda).manual_seed(110)).relu_()
    perm = torch.randperm(b, device=cuda, generator=torch.Generator(device=cuda).manual_seed(111))
    oa, la = run_traced(lambda: _conv3d_call(cuda, u, x, b, size, 0, 192))
    ob, lb = run_traced(lambda: _conv3d_call(cuda, u, x[perm].contiguous(), b, size, 0, 192))
    bn, tiles = conv3d_tiles(b, size, 192)
    expect_schedule("perm conv3d 64->192 k3 b=8", _same_launch(la, lb), f"conv3x3_kernel<{bn}, true>", tiles)
    assert torch.equal(oa.f32[perm], ob.f32) and torch.equal(oa.hi[perm], ob.hi) and torch.equal(oa.lo[perm], ob.lo)


# ------------------------------------------------------------------------------------------------ conv_frames in place
@pytest.mark.parametrize("ks", [3, 1])
def test_conv_frames_in_place(cuda, ks):
    """Sources, residual and ``into=`` outputs are frame slices of (b, t, h, w, c) buffers prefilled with a sentinel
    (the propagation's backbone conv, ks = 3, and its 1x1 fusion, ks = 1): fp64 reference, bit-identical to the
    call on contiguous copies, and nothing outside the written slice changes."""
    b, t, h, w, c = 4, 5, 60, 108, 128
    i_a, i_b, i_out = 1, 3, 2
    g = torch.Generator(device=cuda).manual_seed(112 + ks)
    sentinel = 7.0
    src_hi = torch.full((2, b, t, h, w, c), sentinel, dtype=torch.bfloat16, device=cuda)
    src_lo = torch.full_like(src_hi, sentinel)
    frames = [torch.randn(b, h, w, c, device=cuda, generator=g) for _ in range(2)]
    for j, (f, i) in enumerate(zip(frames, (i_a, i_b))):
        hi, lo = ops.split_bf16(f)
        src_hi[j, :, i], src_lo[j, :, i] = hi, lo
    srcs = [ops.SplitNHWC(src_hi[j, :, i], src_lo[j, :, i], (b, c, h, w)) for j, i in enumerate((i_a, i_b))]
    res_buf = torch.full((b, t, h, w, c), sentinel, device=cuda)
    res_buf[:, i_out] = torch.randn(b, h, w, c, device=cuda, generator=g)
    weight = torch.nn.Parameter(torch.randn(c, 2 * c, ks, ks, device=cuda, generator=g) / (2 * c * ks * ks) ** 0.5)
    bias = torch.randn(c, device=cuda, generator=g) * 0.1
    o32 = torch.full((b, t, h, w, c), sentinel, device=cuda)
    ohi = torch.full((b, t, h, w, c), sentinel, dtype=torch.bfloat16, device=cuda)
    olo = torch.full_like(ohi, sentinel)
    keep = [src_hi.clone(), src_lo.clone(), res_buf.clone()]
    into = (o32[:, i_out], ohi[:, i_out], olo[:, i_out])
    residual = res_buf[:, i_out].permute(0, 3, 1, 2)
    (got32, got_sp), la = run_traced(lambda: ops.conv_frames(srcs, weight, bias, negative_slope=0.1,
                                                             residual=residual, out="both", into=into))
    assert got32.data_ptr() == o32[:, i_out].data_ptr() and got_sp.hi.data_ptr() == ohi[:, i_out].data_ptr()
    tw, th = ops._best_tile(h, w, 1)
    bn, tiles = generic_tiles(b, h, w, c, tile=(tw, th))
    assert tiles > sms()
    expect_schedule(f"conv_frames k{ks} in place", persistent_launch(la), f"conv3x3_kernel<{bn}, false>", tiles)
    # fp64 reference
    x64 = torch.cat([(s.hi.double() + s.lo.double()) for s in srcs], -1).permute(0, 3, 1, 2)
    r64 = res_buf[:, i_out].double().permute(0, 3, 1, 2)
    ref, bound = conv_ref(x64, weight.detach().double(), bias.double(), pad=ks // 2, slope=0.1, r64=r64)
    check_close(o32[:, i_out].permute(0, 3, 1, 2), ref, bound, 5e-5, "f32", f"conv_frames k{ks}")
    check_close((ohi[:, i_out].double() + olo[:, i_out].double()).permute(0, 3, 1, 2), ref, bound, 5e-5, "split",
                f"conv_frames k{ks} split")
    # bit-identical to the same conv on contiguous copies
    dense = [ops.SplitNHWC(s.hi.contiguous(), s.lo.contiguous(), s.shape) for s in srcs]
    (c32, c_sp), lc = run_traced(lambda: ops.conv_frames(dense, weight, bias, negative_slope=0.1,
                                                         residual=residual.contiguous(memory_format=torch.channels_last),
                                                         out="both"))
    _same_launch(la, lc)
    assert torch.equal(c32.permute(0, 2, 3, 1), o32[:, i_out])
    assert torch.equal(c_sp.hi, ohi[:, i_out]) and torch.equal(c_sp.lo, olo[:, i_out])
    # nothing outside the written slice moved; the inputs are untouched
    outside = [j for j in range(t) if j != i_out]
    for buf in (o32, ohi, olo):
        assert torch.all(buf[:, outside] == sentinel)
    assert torch.equal(src_hi, keep[0]) and torch.equal(src_lo, keep[1]) and torch.equal(res_buf, keep[2])
