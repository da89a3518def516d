"""The training convs past one tile per CTA: the discriminator's Conv3d (forward, 4-phase input gradient, split-K
weight gradient), SPyNet's 7x7 input and weight gradients, and SoftComp / SoftSplit.

Every persistent conv here runs on conv3x3_kernel or conv3x3_dact_kernel, whose two consumer warpgroups take alternate
tiles of a CTA; a tile's ring position is the sum of num_kb over the CTA's earlier tiles, and the gather convs' phases
have different K lengths.  Every case:

* runs under torch.profiler and asserts the instantiation, the grid and the tile (or slice) count derived here from
  the launcher's arithmetic, with image counts built from the SM count S so that the regime holds on any H100;
* runs the kernel a second time on the same inputs and asserts the same bits (a ring or ping-pong race, or a read of
  memory nothing wrote, shows as a run-to-run difference before it shows as a wrong value);
* compares random data with a float64 reference computed by plain torch on the GPU, with cuDNN off (im2col and
  cuBLAS GEMMs: the same arithmetic on every run, exact on exact data): rel-of-max, and per element
  |got - ref| <= C * A + rounding (kernel_checks), A being the same operation on absolute values times the derivative
  factor where there is one;
* compares exact-grid data (kernel_checks.grid_values with an integer-valued other operand) with the float64
  reference bit for bit (kernel_checks.check_exact);
* prints its row of the regime table and the worst margin of each per-element check (pytest -s).

Weight and bias gradients: their K is the pixel count (up to 5 * 10^5 here), and the accumulation order is fixed:
within a slice, 12 wgmma accumulations per 64-pixel K block (4 k16 steps x 3 split terms), then the slices are
added in slice order.  Each fp32 accumulation rounds a partial sum of magnitude <= A by at most 2^-24 of it, so on
top of the split error C * A the per-element bound carries the accumulation term 2^-24 * (12 * K blocks per slice +
slices) * A.  The bias partials are fp32 sums of dY itself (no split): bias_partial_kernel adds `len` pixels one
after the other, bias_partial_rows_kernel adds fewer along any path (per-thread sums, a tree of 8, <= 256 row
partials), so 2^-24 * (len + 256 + slices) * sum |dY| bounds both.

No kernel here uses atomics, so permuting clips or images permutes the result bit for bit; that is checked after
asserting that both calls ran the same kernel on the same grid."""
import pytest
import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

from e2fgvi_b200 import _lib, ops
from kernel_checks import (TABLE, assert_exact_grid, cdiv, check_close, check_exact, check_same_bits, conv_tile,
                           cta_tiles, expect_schedule, f32_split, grid_values, images_for, int_values,
                           persistent_launch, print_tables, reference_math, run_traced, same_launch, sms)

pytestmark = pytest.mark.gpu

F32_02 = torch.tensor(0.2, dtype=torch.float32)      # the LeakyReLU slope as the kernels hold it
U = 2.0 ** -24                                        # fp32 unit roundoff (round to nearest)


@pytest.fixture(scope="module", autouse=True)
def schedule_table():
    yield
    print_tables()


def _density(terms, target=256.0):
    """Nonzero probability of the sparse exact-grid operand: about ``target`` / 4 nonzero products per output (E|x|
    is about 2.2, E|w| about 1.7), so A stays far below 2^12."""
    return min(1.0, target / (4.0 * terms))


def _leaky32(v, slope):
    """The kernels' epilogue on an exact fp32 value: v if v > 0 else v * slope, one fp32 rounding."""
    return v if slope == 1.0 else torch.where(v > 0, v, v * F32_02.to(v.device))


def _phase_regime(tiles, grid, kb_of):
    """(distinct num_kb values of the CTA with the most, whether any CTA's tiles have two or more) over the CTAs
    of a persistent launch that walks tiles b, b + grid, ..."""
    sets = [{kb_of(i) for i in r} for r in cta_tiles(tiles, grid)]
    most = max(sets, key=len)
    return sorted(most), any(len(s) > 1 for s in sets)


# ------------------------------------------------------------------------------------------------ discriminator forward
def dis_bn(cout):
    return 32 if cout <= 32 else 64 if cout <= 64 else 128


def dis_tiles(bt, gh, gw, cout, nphase=1):
    """(BN, tiles) of launch_dis_conv on a gh x gw GEMM grid per phase: the tile search of launch_conv3x3 without a
    stride limit, no N-tile halving."""
    tw, th = conv_tile(gh, gw)
    bn = dis_bn(cout)
    return bn, bt * cdiv(gh, th) * cdiv(gw, tw) * nphase * cdiv(cout, bn)


DIS_FWD = {
    "dis fwd bn32 8->32 pad1 37x61": dict(cin=8, cout=32, pad=1, h=37, w=61, t=3, leaky=True, bn=32),
    "dis fwd bn64 32->64 pad2 30x54": dict(cin=32, cout=64, pad=2, h=30, w=54, t=3, leaky=True, bn=64),
    "dis fwd bn128 128->128 pad2 20x36": dict(cin=128, cout=128, pad=2, h=20, w=36, t=2, leaky=True, bn=128),
    # 4 x 7 output: the tile is the image
    "dis fwd bn64 4x7 out, tile = image": dict(cin=32, cout=64, pad=2, h=8, w=13, t=3, leaky=False, bn=64),
    # one tile per image, S + 1 images of one frame: CTA 0 alone owns a second tile
    "dis fwd bn32 tiles=S+1": dict(cin=8, cout=32, pad=1, h=9, w=17, t=1, leaky=True, bn=32, s_plus_1=True),
}


@reference_math()
def _dis_fwd_ref(x64, w64, b64, pad, leaky):
    """(reference before the activation, bound A) in float64, NDHWC."""
    pre = F.conv3d(x64.permute(0, 4, 1, 2, 3), w64, b64, stride=(1, 2, 2), padding=(1, pad, pad))
    bound = F.conv3d(x64.abs().permute(0, 4, 1, 2, 3), w64.abs(), b64.abs(), stride=(1, 2, 2), padding=(1, pad, pad))
    return pre.permute(0, 2, 3, 4, 1), bound.permute(0, 2, 3, 4, 1)


@pytest.mark.parametrize("case", list(DIS_FWD))
def test_dis_forward_multi_tile(cuda, case):
    c = DIS_FWD[case]
    s, pad, cin, cout = sms(), c["pad"], c["cin"], c["cout"]
    ho, wo = ops.dis_out_size(c["h"], pad), ops.dis_out_size(c["w"], pad)
    t = c["t"]
    if c.get("s_plus_1"):
        b = s + 1
        assert dis_tiles(b * t, ho, wo, cout)[1] == s + 1
    else:
        b = images_for(lambda k: dis_tiles(k * t, ho, wo, cout)[1], 2 * s + 1)
    bn, tiles = dis_tiles(b * t, ho, wo, cout)
    assert bn == c["bn"]
    slope = 0.2 if c["leaky"] else 1.0
    g = torch.Generator(device=cuda).manual_seed(201)
    # random data
    x = torch.randn(b, t, c["h"], c["w"], cin, device=cuda, generator=g)
    wt = torch.randn(cout, cin, 3, 5, 5, device=cuda, generator=g) / (cin * 75) ** 0.5
    bias = torch.randn(cout, device=cuda, generator=g) * 0.1
    x_hi, x_lo = ops.split_bf16(x)
    w_hi, w_lo = ops.dis_pack_weight(wt, cin)
    (out, o_hi, o_lo), launches = run_traced(lambda: ops.dis_conv3d(x_hi, x_lo, w_hi, w_lo, bias, cout, pad, c["leaky"]))
    expect_schedule(case, persistent_launch(launches), f"conv3x3_kernel<{bn}, true>", tiles)
    check_same_bits((out, o_hi, o_lo), ops.dis_conv3d(x_hi, x_lo, w_hi, w_lo, bias, cout, pad, c["leaky"]), case)
    pre, bound = _dis_fwd_ref(x.double(), wt.double(), bias.double(), pad, c["leaky"])
    ref = F.leaky_relu(pre, slope)
    check_close(out, ref, bound, 1e-4, "f32", case)
    check_close(o_hi.double() + o_lo.double(), ref, bound, 1e-4, "split", case + " split")
    # exact-grid data: x on the grid, integer weights and bias
    x = grid_values((b, t, c["h"], c["w"], cin), g, _density(75 * cin))
    wt = int_values((cout, cin, 3, 5, 5), g)
    bias = int_values((cout,), g)
    x_hi, x_lo = ops.split_bf16(x)
    w_hi, w_lo = ops.dis_pack_weight(wt, cin)
    out, o_hi, o_lo = ops.dis_conv3d(x_hi, x_lo, w_hi, w_lo, bias, cout, pad, c["leaky"])
    pre, bound = _dis_fwd_ref(x.double(), wt.double(), bias.double(), pad, c["leaky"])
    assert_exact_grid(bound, x, case)
    ref32 = _leaky32(pre.float(), slope)
    check_exact(out, ref32, case + " exact")
    hi, lo = f32_split(ref32)
    check_exact(o_hi, hi, case + " exact hi")
    check_exact(o_lo, lo, case + " exact lo")


# ------------------------------------------------------------------------------------------------ discriminator dgrad
def dis_dgrad_regime(tiles, grid, bn, cin_s):
    """Whether any CTA's tiles span two phases: decode_tile orders tiles N tile, group, phase, so tile i has phase
    (i // N tiles) % 4."""
    ng = cdiv(cin_s, bn)
    kbs, mixed = _phase_regime(tiles, grid, lambda i: (i // ng) % 4)
    if ng == 1:                           # closed form: CTA b's phases are (b + i * grid) % 4
        assert mixed == (grid % 4 != 0 and tiles > grid), (grid, tiles)
    return mixed


DIS_DGRAD = {
    # dgrad output = the forward's input channels; first layer: 8 channels (the direct store path), no activation
    "dis dgrad 32->8 pad1 37x61 no act": dict(cin=8, cout=32, pad=1, h=37, w=61, t=3, act=False, bn=32),
    "dis dgrad 64->32 pad1 31x53 act split": dict(cin=32, cout=64, pad=1, h=31, w=53, t=2, act=True, bn=32),
    "dis dgrad 64->32 pad2 30x54 act split": dict(cin=32, cout=64, pad=2, h=30, w=54, t=3, act=True, bn=32),
    "dis dgrad 128->128 pad2 19x35 act split": dict(cin=128, cout=128, pad=2, h=19, w=35, t=2, act=True, bn=128),
}


@reference_math()
def _dis_dgrad_ref(dy64, w64, size, pad, factor):
    """(reference, bound A) in float64, NDHWC: the input gradient of the forward conv times ``factor``."""
    b, t, h, w, cin = size
    dyc = dy64.permute(0, 4, 1, 2, 3)
    kw = dict(stride=(1, 2, 2), padding=(1, pad, pad))
    ref = nn_grad.conv3d_input((b, cin, t, h, w), w64, dyc, **kw).permute(0, 2, 3, 4, 1)
    bound = nn_grad.conv3d_input((b, cin, t, h, w), w64.abs(), dyc.abs(), **kw).permute(0, 2, 3, 4, 1)
    return ref * factor, bound * factor


@pytest.mark.parametrize("case", list(DIS_DGRAD))
def test_dis_dgrad_multi_tile(cuda, case):
    c = DIS_DGRAD[case]
    s, pad, cin, cout, h, w, t = sms(), c["pad"], c["cin"], c["cout"], c["h"], c["w"], c["t"]
    ho, wo = ops.dis_out_size(h, pad), ops.dis_out_size(w, pad)
    gh, gw = (h + 1) // 2, (w + 1) // 2
    b = images_for(lambda k: dis_tiles(k * t, gh, gw, cin, 4)[1], 2 * s + 1)
    bn, tiles = dis_tiles(b * t, gh, gw, cin, 4)
    assert bn == c["bn"]
    mixed = dis_dgrad_regime(tiles, min(tiles, s), bn, cin)
    # taps per phase (launch_dis_conv's table): ky = oy + pad, kx = ox + pad (mod 2)
    tap_counts = [sum(1 for kt in range(3) for ky in range(5) for kx in range(5)
                      if (oy + pad - ky) % 2 == 0 and (ox + pad - kx) % 2 == 0) for oy in (0, 1) for ox in (0, 1)]
    assert tap_counts == ([12, 18, 18, 27] if pad == 1 else [27, 18, 18, 12])
    g = torch.Generator(device=cuda).manual_seed(202)
    act = None
    factor = 1.0
    if c["act"]:
        act = torch.randn(b, t, h, w, cin, device=cuda, generator=g).bfloat16()
        act[torch.rand(act.shape, device=cuda, generator=g) < 0.1] = 0       # LeakyReLU(0) = 0: slope 0.2 there
        factor = torch.where(act.double() > 0, 1.0, 0.2)
    # random data
    dy = torch.randn(b, t, ho, wo, cout, device=cuda, generator=g)
    wt = torch.randn(cout, cin, 3, 5, 5, device=cuda, generator=g) / (cout * 18) ** 0.5
    dy_hi, dy_lo = ops.split_bf16(dy)
    t_hi, t_lo = ops.dis_pack_weight_t(wt, pad, cin)
    (dx, dx_hi, dx_lo), launches = run_traced(
        lambda: ops.dis_conv3d_dgrad(dy_hi, dy_lo, t_hi, t_lo, act, h, w, cin, pad, split=True))
    expect_schedule(case, persistent_launch(launches), f"conv3x3_kernel<{bn}, true>", tiles,
                    f"K blocks/phase {[k * cdiv(cout, 64) for k in tap_counts]}, phases mixed per CTA: {mixed}")
    check_same_bits((dx, dx_hi, dx_lo), ops.dis_conv3d_dgrad(dy_hi, dy_lo, t_hi, t_lo, act, h, w, cin, pad, split=True),
                    case)
    ref, bound = _dis_dgrad_ref(dy.double(), wt.double(), (b, t, h, w, cin), pad, factor)
    check_close(dx, ref, bound, 1e-4, "f32", case)
    check_close(dx_hi.double() + dx_lo.double(), ref, bound, 1e-4, "split", case + " split")
    # exact-grid data: integer dY, weights on the grid (the weight's lo part contributes)
    dy = int_values((b, t, ho, wo, cout), g)
    wt = grid_values((cout, cin, 3, 5, 5), g, _density(27 * cout))
    dy_hi, dy_lo = ops.split_bf16(dy)
    t_hi, t_lo = ops.dis_pack_weight_t(wt, pad, cin)
    dx, dx_hi, dx_lo = ops.dis_conv3d_dgrad(dy_hi, dy_lo, t_hi, t_lo, act, h, w, cin, pad, split=True)
    s64, bound = _dis_dgrad_ref(dy.double(), wt.double(), (b, t, h, w, cin), pad, 1.0)
    assert_exact_grid(bound, wt, case)
    ref32 = s64.float()
    if act is not None:
        ref32 = torch.where(act.float() > 0, ref32, ref32 * F32_02.to(cuda))
    check_exact(dx, ref32, case + " exact")
    hi, lo = f32_split(ref32)
    check_exact(dx_hi, hi, case + " exact hi")
    check_exact(dx_lo, lo, case + " exact lo")


# ------------------------------------------------------------------------------------------------ SPyNet input gradient
def rows_nhwc(flat, r):
    """(n, h, w, c) view of the content of a row-gapped buffer laid out like RowsNHWC ``r``; asserts that its gaps,
    pad channels and tail are zero."""
    n, c, h, w = r.shape
    body = flat[: n * h * r.pitch * r.cin].view(n, h, r.pitch, r.cin)
    gaps = torch.ones(r.pitch, dtype=torch.bool, device=flat.device)
    gaps[r.lead: r.lead + w] = False
    assert torch.count_nonzero(body[:, :, gaps]) == 0 and torch.count_nonzero(body[:, :, :, c:]) == 0
    assert torch.count_nonzero(flat[n * h * r.pitch * r.cin:]) == 0
    return body[:, :, r.lead: r.lead + w, :c]


def spynet_tile(h, w, rows):
    """launch_conv3x3's tile for a 7x7 / stride 1 conv: the image itself below 16 x 8, 16 x 8 for a row-gapped
    source, else the fewest-tiles search."""
    if w < 16 or h < 8:
        return min(w, 16), min(h, 8)
    return (16, 8) if rows else conv_tile(h, w)


# (cin, cout) of the forward conv: the input gradient runs cout -> cin; act layout (None: no ReLU before the conv) and
# the next operand's format
SPYNET = {
    "8<-32 rows dY, no act, out rows": dict(cin=8, cout=32, act=None, out="rows", kernel="conv3x3_kernel<32, false>",
                                            num_kb=7 * 4),
    "32<-64 dense dY, act rows, out split": dict(cin=32, cout=64, act="rows", out="split",
                                                 kernel="conv3x3_dact_kernel<32>", num_kb=49),
    "32<-16 rows dY, act split, out rows": dict(cin=32, cout=16, act="split", out="rows",
                                               kernel="conv3x3_dact_kernel<32>", num_kb=7 * 2),
    "16<-2 rows dY, act rows, out f32": dict(cin=16, cout=2, act="rows", out="f32", kernel="conv3x3_dact_kernel<32>",
                                             num_kb=7 * 1),
    "64<-32 rows dY, act split, out split": dict(cin=64, cout=32, act="split", out="split",
                                                 kernel="conv3x3_dact_kernel<64>", num_kb=7 * 4),
}
SPYNET_SIZES = {"64x 64x128": (64, 64, 128), "ragged 13x21": (None, 13, 21), "64x 4x8": (64, 4, 8)}


def spynet_num_kb(cout):
    """K blocks per tile of the input gradient: window-packed K for a row-gapped dY of c = max(8, rows_channels(cout))
    channels (7 kernel rows x ceil(7 / (64 / c)) windows of 64 / c pixels), 49 taps x 64-channel chunks for a dense
    one."""
    if cout <= 32:
        return 7 * cdiv(7, 64 // max(8, ops.rows_channels(cout)))
    return 49 * cdiv(cout, 64)


def _spynet_operands(dy, act, c):
    dy_op = ops.pack_rows(dy, lead=3, cin=max(8, ops.rows_channels(c["cout"]))) if c["cout"] <= 32 else ops.split_nhwc(dy)
    act_op = None
    if c["act"] == "rows":
        act_op = ops.pack_rows(act, lead=3)
    elif c["act"] == "split":
        act_op = ops.split_nhwc(act)
    return dy_op, act_op


def _act_hi(act_op):
    if isinstance(act_op, ops.RowsNHWC):
        return rows_nhwc(act_op.hi, act_op).float()
    return act_op.hi.float()


def _next_operand(nxt, out):
    """(hi, lo) of the next operand as (n, h, w, c) tensors, or None for out = 'f32'."""
    if out == "rows":
        return rows_nhwc(nxt.hi, nxt), rows_nhwc(nxt.lo, nxt)
    if out == "split":
        return nxt.hi, nxt.lo
    assert nxt is None
    return None


@reference_math()
def _spynet_dgrad_ref(dy64, w64):
    ref = F.conv_transpose2d(dy64, w64, padding=3).permute(0, 2, 3, 1)
    bound = F.conv_transpose2d(dy64.abs(), w64.abs(), padding=3).permute(0, 2, 3, 1)
    return ref, bound


@pytest.mark.parametrize("size", list(SPYNET_SIZES))
@pytest.mark.parametrize("conv", list(SPYNET))
def test_spynet_dgrad_multi_tile(cuda, conv, size):
    c = SPYNET[conv]
    s, cin, cout = sms(), c["cin"], c["cout"]
    n, h, w = SPYNET_SIZES[size]
    rows = cout <= 32
    tw, th = spynet_tile(h, w, rows)
    bn = 32 if cin <= 32 else 64
    per = cdiv(h, th) * cdiv(w, tw)
    if n is None:
        n = images_for(lambda k: k * per, 2 * s + 1)
    tiles = n * per
    case = f"spynet dgrad {conv} {n}x{h}x{w}"
    g = torch.Generator(device=cuda).manual_seed(203 + cin + cout + h)
    act = torch.relu(torch.randn(n, cin, h, w, device=cuda, generator=g)) if c["act"] else None
    # random data
    dy = torch.randn(n, cout, h, w, device=cuda, generator=g)
    wt = torch.randn(cout, cin, 7, 7, device=cuda, generator=g) * 0.05
    dy_op, act_op = _spynet_operands(dy, act, c)
    (dx, nxt), launches = run_traced(lambda: ops.conv2d_dgrad(dy_op, wt, act=act_op, out=c["out"]))
    assert spynet_num_kb(cout) == c["num_kb"]
    expect_schedule(case, persistent_launch(launches), c["kernel"], tiles, f"num_kb {c['num_kb']}")
    dx2, nxt2 = ops.conv2d_dgrad(dy_op, wt, act=act_op, out=c["out"])
    check_same_bits((dx,) + ((nxt.hi, nxt.lo) if nxt is not None else ()),
                    (dx2,) + ((nxt2.hi, nxt2.lo) if nxt2 is not None else ()), case)
    factor = 1.0 if act_op is None else (_act_hi(act_op) > 0).double()
    ref, bound = _spynet_dgrad_ref(dy.double(), wt.double())
    ref, bound = ref * factor, bound * factor
    check_close(dx, ref, bound, 1e-4, "f32", case)
    parts = _next_operand(nxt, c["out"])
    if parts is not None:
        check_close(parts[0].double() + parts[1].double(), ref, bound, 1e-4, "split", case + " " + c["out"])
    # exact-grid data, the grid on alternate sides: dY (the activation side of the GEMM) or the weight
    dy_on_grid = cin in (8, 16, 64)
    if dy_on_grid:
        dy, wt = grid_values((n, cout, h, w), g, _density(49 * cout)), int_values((cout, cin, 7, 7), g)
    else:
        dy, wt = int_values((n, cout, h, w), g), grid_values((cout, cin, 7, 7), g, _density(49 * cout))
    dy_op, act_op = _spynet_operands(dy, act, c)
    dx, nxt = ops.conv2d_dgrad(dy_op, wt, act=act_op, out=c["out"])
    s64, bound = _spynet_dgrad_ref(dy.double(), wt.double())
    assert_exact_grid(bound, dy if dy_on_grid else wt, case)
    ref32 = s64.float()
    if act_op is not None:
        ref32 = torch.where(_act_hi(act_op) > 0, ref32, ref32 * 0.0)
    check_exact(dx, ref32, case + " exact")
    parts = _next_operand(nxt, c["out"])
    if parts is not None:
        hi, lo = f32_split(ref32)
        check_exact(parts[0], hi, case + " exact hi")
        check_exact(parts[1], lo, case + " exact lo")


# ------------------------------------------------------------------------------------------------ weight gradients
def wgrad_slices(pixels, cout, n_cols):
    """launch_*_wgrad's split-K slice count: about 264 CTAs over the 64 x 128 tiles, >= 4 K blocks per slice, <= 64."""
    s = cdiv(264, cdiv(cout, 64) * cdiv(n_cols, 128))
    return max(1, min(s, pixels // 256, 64))


def slice_len(pixels, slices):
    return cdiv(cdiv(pixels, slices), 64) * 64


WGRAD = {
    "dis 8->32 pad1 1 slice": dict(kind="dis", cin=8, cout=32, pad=1, b=1, t=2, h=9, w=17, slices=1),
    # N = 75 * 8 = 600 (a 88-column tail), Cout 32 (an M tail), 12 slices of which the last is empty
    "dis 8->32 pad1 37x61 Ntail empty slice": dict(kind="dis", cin=8, cout=32, pad=1, b=2, t=3, h=37, w=61, slices=12,
                                                   empty=1),
    "dis 128->128 pad2 2 M tiles": dict(kind="dis", cin=128, cout=128, pad=2, b=1, t=2, h=60, w=108, slices=2),
    "c2d 8->32 rows 64x64x128 64-slice cap": dict(kind="c2d", cin=8, cout=32, n=64, h=64, w=128, layout="rows",
                                                  slices=64),
    # N = 49 * 16 = 784, Cout 2 padded to 8, 38 slices of 320 pixels: the last 7 are empty
    "c2d 16->2 rows 9x23x47 empty slices": dict(kind="c2d", cin=16, cout=2, n=9, h=23, w=47, layout="rows",
                                                slices=38, empty=7),
    "c2d 64->32 dense 16x13x21": dict(kind="c2d", cin=64, cout=32, n=16, h=13, w=21, layout="split", slices=11,
                                      empty=1),
    "c2d 32->16 rows 1 slice": dict(kind="c2d", cin=32, cout=16, n=2, h=4, w=8, layout="rows", slices=1),
}


def _wgrad_call(c, x, dy, cuda):
    """Run the weight gradient; returns (dW, db, the operand channel count, the kernel's cout, pixels, work elems)."""
    lib = _lib.load()
    if c["kind"] == "dis":
        x_hi, x_lo = ops.split_bf16(x)
        b, t, h, w, cs = x.shape
        elems = lib.e2f_dis_conv3d_wgrad_work_elems(b, t, h, w, cs, c["cout"], c["pad"])
        dw, db = ops.dis_conv3d_wgrad(dy, x_hi, x_lo, c["cin"], c["pad"], True)
        return dw, db, cs, c["cout"], dy.numel() // c["cout"], elems
    xo = ops.pack_rows(x, lead=3) if c["layout"] == "rows" else ops.split_nhwc(x)
    xc = xo.cin if c["layout"] == "rows" else xo.hi.shape[-1]
    n, h, w, cout = dy.shape
    cpad = cdiv(cout, 8) * 8
    elems = lib.e2f_conv2d_wgrad_work_elems(n, h, w, xc, cpad)
    dw, db = ops.conv2d_wgrad(dy, xo, c["cin"], with_bias=True)
    return dw, db, xc, cpad, n * h * w, elems


@reference_math()
def _wgrad_ref(c, x64, dy64):
    """(dW, db, bound of dW, bound of db) in float64."""
    cout = c["cout"]
    if c["kind"] == "dis":
        xc, dyc = x64.permute(0, 4, 1, 2, 3), dy64.permute(0, 4, 1, 2, 3)
        kw = dict(stride=(1, 2, 2), padding=(1, c["pad"], c["pad"]))
        shape = (cout, c["cin"], 3, 5, 5)
        dw = nn_grad.conv3d_weight(xc, shape, dyc, **kw)
        bound = nn_grad.conv3d_weight(xc.abs(), shape, dyc.abs(), **kw)
    else:
        dyc = dy64.permute(0, 3, 1, 2)
        shape = (cout, c["cin"], 7, 7)
        dw = nn_grad.conv2d_weight(x64, shape, dyc, padding=3)
        bound = nn_grad.conv2d_weight(x64.abs(), shape, dyc.abs(), padding=3)
    red = tuple(range(dy64.dim() - 1))
    return dw, dy64.sum(red), bound, dy64.abs().sum(red)


@pytest.mark.parametrize("case", list(WGRAD))
def test_wgrad_slices(cuda, case):
    c = WGRAD[case]
    cin, cout = c["cin"], c["cout"]
    taps = 75 if c["kind"] == "dis" else 49
    if c["kind"] == "dis":
        ho, wo = ops.dis_out_size(c["h"], c["pad"]), ops.dis_out_size(c["w"], c["pad"])
        x_shape, dy_shape = (c["b"], c["t"], c["h"], c["w"], cin), (c["b"], c["t"], ho, wo, cout)
        names = ("wgrad_mma_kernel<3, 5, 2>", "bias_partial_kernel", "reduce_kernel<75>")
    else:
        x_shape, dy_shape = (c["n"], cin, c["h"], c["w"]), (c["n"], c["h"], c["w"], cout)
        names = ("wgrad_mma_kernel<1, 7, 1>", "bias_partial_rows_kernel", "reduce_kernel<49>")
    g = torch.Generator(device=cuda).manual_seed(204)
    # random data
    x = torch.randn(x_shape, device=cuda, generator=g)
    dy = torch.randn(dy_shape, device=cuda, generator=g)
    (dw, db, xc, kcout, pixels, elems), launches = run_traced(lambda: _wgrad_call(c, x, dy, cuda))
    n_cols = taps * xc
    slices = wgrad_slices(pixels, kcout, n_cols)
    assert slices == c["slices"] and elems == slices * (kcout * n_cols + kcout), (slices, elems)
    ln = slice_len(pixels, slices)
    empty = sum(1 for z in range(slices) if z * ln >= pixels)
    assert empty == c.get("empty", 0), empty
    ours = [k for k in launches if k.name in names]
    assert [k.name for k in ours] == list(names), [k.name for k in launches]
    assert ours[0].grid == (cdiv(n_cols, 128), cdiv(kcout, 64), slices), ours[0].grid
    assert ours[1].grid == (slices, 1, 1) and ours[2].grid == (cdiv(kcout * n_cols, 256), 1, 1), (ours[1], ours[2])
    kb = ln // 64
    TABLE.append((case, names[0], "x".join(map(str, ours[0].grid)), f"{slices}sl", f"{kb}kb", ours[0].smem,
                  f"{pixels} px, slice {ln} px, empty slices {empty}, M tiles {cdiv(kcout, 64)}, N {n_cols}"))
    check_same_bits((dw, db), _wgrad_call(c, x, dy, cuda)[:2], case)
    ref_w, ref_b, bound_w, bound_b = _wgrad_ref(c, x.double(), dy.double())
    acc_w = U * (12 * kb + slices) * bound_w
    check_close(dw, ref_w, bound_w, 1e-4, "f32", case + " dW", extra=acc_w)
    check_close(db, ref_b, torch.zeros_like(bound_b), 1e-4, "f32", case + " db",
                extra=U * (ln + 256 + slices) * bound_b)
    # exact-grid data in both directions: dY on the grid with integer X (the kernel splits dY), X on the grid with
    # integer dY (integer dY: the bias gradient is a sum of integers below 2^24, exact).  The grid operand's fine
    # background puts nonzero terms in every K block of every slice: a dropped or repeated block changes the result.
    for dy_on_grid in (True, False):
        if dy_on_grid:
            dy, x = grid_values(dy_shape, g, _density(pixels), fine=True), int_values(x_shape, g, 2)
        else:
            dy, x = int_values(dy_shape, g, 2), grid_values(x_shape, g, _density(pixels), fine=True)
        dw, db, *_ = _wgrad_call(c, x, dy, cuda)
        ref_w, ref_b, bound_w, bound_b = _wgrad_ref(c, x.double(), dy.double())
        what = f"{case} exact ({'dY' if dy_on_grid else 'X'} on the grid)"
        assert_exact_grid(bound_w, dy if dy_on_grid else x, what)
        assert float(bound_b.max()) < (2.0 ** 12 if dy_on_grid else 2.0 ** 24), float(bound_b.max())
        check_exact(dw, ref_w.float(), what + " dW")
        check_exact(db, ref_b.float(), what + " db")


# ------------------------------------------------------------------------------------------------ SoftComp / SoftSplit
SC_TAPS = [len([1 for dy in range((6 - ry) // 3 + 1) for dx in range((6 - rx) // 3 + 1)])
           for ry in range(3) for rx in range(3)]                # taps per phase of the 7 / 3 / 3 transposed conv

SOFT = {
    "soft_comp base 64x 60x108 res + bias map -> f32": dict(op="comp", n=64, h=60, w=108, out="f32"),
    "soft_comp hq ragged 47x83 -> split": dict(op="comp", n=None, h=47, w=83, out="split"),
    "soft_split 128->512 64x 60x108": dict(op="split", n=64, h=60, w=108),
}


@reference_math()
def _soft_comp_ref(tok64, w64, b64, extra64, res64, h, w):
    n, fh, fw, hid = tok64.shape
    lin = F.linear(tok64.view(n, fh * fw, hid), w64, b64).permute(0, 2, 1)
    ref = F.fold(lin, (h, w), 7, padding=3, stride=3)
    lin = F.linear(tok64.abs().view(n, fh * fw, hid), w64.abs(), b64.abs()).permute(0, 2, 1)
    bound = F.fold(lin, (h, w), 7, padding=3, stride=3)
    if extra64 is not None:
        ref, bound = ref + extra64, bound + extra64.abs()
    if res64 is not None:
        ref, bound = ref + res64, bound + res64.abs()
    return ref.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1)


@reference_math()
def _soft_split_ref(x64, w64, b64):
    cols = F.unfold(x64, 7, padding=3, stride=3).permute(0, 2, 1)
    colsa = F.unfold(x64.abs(), 7, padding=3, stride=3).permute(0, 2, 1)
    return F.linear(cols, w64, b64), F.linear(colsa, w64.abs(), b64.abs())


def _sc_operands(gen, n, h, w, fh, fw, exact, cuda):
    if exact:
        tok = grid_values((n, fh, fw, 512), gen, _density(9 * 512))   # <= 9 taps x 512 per output
        return (tok, int_values((128 * 49, 512), gen), int_values((128 * 49,), gen),
                int_values((128, h, w), gen), int_values((n, 128, h, w), gen))
    return (torch.randn(n, fh, fw, 512, device=cuda, generator=gen),
            torch.randn(128 * 49, 512, device=cuda, generator=gen) / 512 ** 0.5,
            torch.randn(128 * 49, device=cuda, generator=gen) * 0.1,
            torch.randn(128, h, w, device=cuda, generator=gen) * 0.3,
            torch.randn(n, 128, h, w, device=cuda, generator=gen))


def _soft_comp_call(tok, wt, bias, extra, res, h, w, out):
    wp, bp = torch.nn.Parameter(wt), torch.nn.Parameter(bias)
    with torch.no_grad():
        if out == "f32":
            return ops.soft_comp(tok, wp, bp, (h, w), 7, 3, 3, bias_map_extra=torch.nn.Parameter(extra),
                                 residual=res.contiguous(memory_format=torch.channels_last)).permute(0, 2, 3, 1)
        return ops.soft_comp(tok, wp, bp, (h, w), 7, 3, 3, out="split")


def gather_tiles_per_image(gh, gw, stride):
    """Tiles per image and phase of the gather convs (SoftComp, SoftSplit): the fewest tile_w x tile_h <= 128 boxes
    (sides <= 256 / stride and within the grid) that cover the gh x gw GEMM grid, the count the tile choice
    minimises first.  Found by enumerating every box, independently of the library's tile search."""
    return min(cdiv(gh, th) * cdiv(gw, tw) for tw in range(1, min(gw, 256 // stride) + 1)
               for th in range(1, min(gh, 256 // stride, 128 // tw) + 1))


@pytest.mark.parametrize("case", list(SOFT))
def test_soft_comp_split_multi_tile(cuda, case):
    c = SOFT[case]
    s, h, w = sms(), c["h"], c["w"]
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    assert gather_tiles_per_image(20, 36, 1) == 6                   # 12 x 10 tiles the 8-clip token grid exactly
    g = torch.Generator(device=cuda).manual_seed(205)
    if c["op"] == "split":
        # SoftSplit: a 7x7 / stride-3 conv, 128 -> 512 channels: one phase, 49 taps x 2 K chunks
        n = c["n"]
        tiles = n * gather_tiles_per_image(fh, fw, 3) * 4
        for exact in (False, True):
            if exact:
                x, wt, bias = grid_values((n, 128, h, w), g, _density(49 * 128)), int_values((512, 128 * 49), g), \
                    int_values((512,), g)
            else:
                x = torch.randn(n, 128, h, w, device=cuda, generator=g)
                wt = torch.randn(512, 128 * 49, device=cuda, generator=g) / (128 * 49) ** 0.5
                bias = torch.randn(512, device=cuda, generator=g) * 0.1
            wp, bp = torch.nn.Parameter(wt), torch.nn.Parameter(bias)
            xin = x.contiguous(memory_format=torch.channels_last)
            with torch.no_grad():
                got, launches = run_traced(lambda: ops.soft_split(xin, wp, bp, 7, 3, 3))
            ref, bound = _soft_split_ref(x.double(), wt.double(), bias.double())
            if exact:
                assert_exact_grid(bound, x, case)
                check_exact(got, ref.float(), case + " exact")
            else:
                expect_schedule(case, persistent_launch(launches), "conv3x3_kernel<128, false>", tiles, "num_kb 98")
                check_close(got, ref, bound, 5e-5, "f32", case)
        return
    # SoftComp: nine phases of 9 / 6 / 4 taps x 8 K chunks of the 512 hidden channels
    assert SC_TAPS == [9, 6, 6, 6, 4, 4, 6, 4, 4]
    per = gather_tiles_per_image(fh, fw, 1) * 9
    n = c["n"] or images_for(lambda k: k * per, 2 * s + 1)
    tiles = n * per                                       # 128 channels: one N tile of 128 (no halving: > S / 2 tiles)
    assert 2 * tiles > s
    kbs, mixed = _phase_regime(tiles, min(tiles, s), lambda i: SC_TAPS[i % 9] * 8)
    assert mixed and len(kbs) >= 2, kbs
    for exact in (False, True):
        tok, wt, bias, extra, res = _sc_operands(g, n, h, w, fh, fw, exact, cuda)
        got, launches = run_traced(lambda: _soft_comp_call(tok, wt, bias, extra, res, h, w, c["out"]))
        base = c["out"] == "f32"
        ref, bound = _soft_comp_ref(tok.double(), wt.double(), bias.double(), extra.double() if base else None,
                                    res.double() if base else None, h, w)
        if not exact:
            expect_schedule(case, persistent_launch(launches), "conv3x3_kernel<128, false>", tiles,
                            f"num_kb per phase {[k * 8 for k in SC_TAPS]}, one CTA's: {kbs}")
            again = _soft_comp_call(tok, wt, bias, extra, res, h, w, c["out"])
            check_same_bits((got,) if base else (got.hi, got.lo), (again,) if base else (again.hi, again.lo), case)
            if base:
                check_close(got, ref, bound, 5e-5, "f32", case)
            else:
                check_close(got.hi.double() + got.lo.double(), ref, bound, 5e-5, "split", case)
            continue
        assert_exact_grid(bound, tok, case)
        ref32 = ref.float()
        if base:
            check_exact(got, ref32, case + " exact")
        else:
            hi, lo = f32_split(ref32)
            check_exact(got.hi, hi, case + " exact hi")
            check_exact(got.lo, lo, case + " exact lo")


# ------------------------------------------------------------------------------------------------ bitwise permutation
def _perm(cuda, n, seed):
    return torch.randperm(n, device=cuda, generator=torch.Generator(device=cuda).manual_seed(seed))


def test_dis_clip_permutation_bitwise(cuda):
    """Discriminator layer 2 (32 -> 64, pad 2) over 8 clips of 5 frames at 120 x 216 (the 432 x 240 input after layer
    1): forward and input gradient (LeakyReLU derivative, split output); permuting the clips permutes the results
    bit for bit."""
    b, t, h, w, cin, cout, pad = 8, 5, 120, 216, 32, 64, 2
    g = torch.Generator(device=cuda).manual_seed(206)
    perm = _perm(cuda, b, 207)
    x = torch.randn(b, t, h, w, cin, device=cuda, generator=g)
    wt = torch.randn(cout, cin, 3, 5, 5, device=cuda, generator=g) / (cin * 75) ** 0.5
    bias = torch.randn(cout, device=cuda, generator=g) * 0.1
    w_hi, w_lo = ops.dis_pack_weight(wt, cin)
    xs = [ops.split_bf16(x), ops.split_bf16(x[perm].contiguous())]
    (oa, la), (ob, lb) = [run_traced(lambda: ops.dis_conv3d(*xp, w_hi, w_lo, bias, cout, pad, True)) for xp in xs]
    ho, wo = ops.dis_out_size(h, pad), ops.dis_out_size(w, pad)
    bn, tiles = dis_tiles(b * t, ho, wo, cout)
    expect_schedule("perm dis fwd 32->64 8 clips", same_launch(la, lb), f"conv3x3_kernel<{bn}, true>", tiles)
    for u, v in zip(oa, ob):
        assert torch.equal(u[perm], v)
    dy = torch.randn(b, t, ho, wo, cout, device=cuda, generator=g)
    act = torch.randn(b, t, h, w, cin, device=cuda, generator=g).bfloat16()
    t_hi, t_lo = ops.dis_pack_weight_t(wt, pad, cin)
    dys = [(ops.split_bf16(dy), act), (ops.split_bf16(dy[perm].contiguous()), act[perm].contiguous())]
    (da, la), (db, lb) = [run_traced(lambda: ops.dis_conv3d_dgrad(*d, t_hi, t_lo, a, h, w, cin, pad, split=True))
                          for d, a in dys]
    bn, tiles = dis_tiles(b * t, (h + 1) // 2, (w + 1) // 2, cin, 4)
    expect_schedule("perm dis dgrad 64->32 act 8 clips", same_launch(la, lb), f"conv3x3_kernel<{bn}, true>", tiles)
    for u, v in zip(da, db):
        assert torch.equal(u[perm], v)


def test_spynet_dgrad_and_soft_comp_image_permutation_bitwise(cuda):
    """SPyNet 32 <- 64 input gradient (dense dY, row-gapped ReLU activation and output) at 64 images of 64 x 128, and
    SoftComp (residual, bias map) at 64 images of 60 x 108: permuting the images permutes the results bit for bit."""
    n, h, w = 64, 64, 128
    g = torch.Generator(device=cuda).manual_seed(208)
    perm = _perm(cuda, n, 209)
    c = SPYNET["32<-64 dense dY, act rows, out split"]
    dy = torch.randn(n, 64, h, w, device=cuda, generator=g)
    act = torch.relu(torch.randn(n, 32, h, w, device=cuda, generator=g))
    wt = torch.randn(64, 32, 7, 7, device=cuda, generator=g) * 0.05
    runs = []
    for d, a in ((dy, act), (dy[perm], act[perm])):
        dy_op, act_op = _spynet_operands(d, a, c)
        runs.append(run_traced(lambda: ops.conv2d_dgrad(dy_op, wt, act=act_op, out="rows")))
    (ra, la), (rb, lb) = runs
    expect_schedule("perm spynet dgrad 32<-64 64x64x128", same_launch(la, lb), c["kernel"],
                    n * cdiv(h, spynet_tile(h, w, False)[1]) * cdiv(w, spynet_tile(h, w, False)[0]))
    assert torch.equal(ra[0][perm], rb[0])
    for part in ("hi", "lo"):
        assert torch.equal(rows_nhwc(getattr(ra[1], part), ra[1])[perm], rows_nhwc(getattr(rb[1], part), rb[1]))
    h, w = 60, 108
    fh, fw = 20, 36
    tok, wsc, bsc, extra, res = _sc_operands(g, n, h, w, fh, fw, False, cuda)
    (sa, la), (sb, lb) = [run_traced(lambda: _soft_comp_call(tk, wsc, bsc, extra, r, h, w, "f32"))
                          for tk, r in ((tok, res), (tok[perm].contiguous(), res[perm].contiguous()))]
    expect_schedule("perm soft_comp 64x 60x108", same_launch(la, lb), "conv3x3_kernel<128, false>",
                    n * gather_tiles_per_image(fh, fw, 1) * 9)
    assert torch.equal(sa[perm], sb)
