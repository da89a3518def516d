"""Helpers shared by the tests that hold the persistent wgmma kernels to float64 references: which kernel a call
reached (torch.profiler), the launchers' tile arithmetic, the per-element error bound and the exact check.

Per-element bound (``check_close``).  C = 2^-14.  Each fp32 operand is a bf16 pair hi + lo: |x - hi| <= 2^-8 |x| and
the rounding of lo leaves at most 2^-16 |x|, typically 2^-17 or less; the dropped lo.lo product is <= 2^-16 |x||w|,
typically 2^-18.  Per product that is at most 3 * 2^-16 of |x||w| (0.75 C) and on average several times less, and
the fp32 accumulation adds a few 2^-24 of A per accumulator update, whose errors largely cancel over long K.  A is the
same operation on |x| and |w| plus |bias| and |residual|.

Exact check (``check_exact``) on exact-grid operands (``grid_values`` with an integer-valued other operand,
``int_values``): every value a + b * 2^-8 with |a| <= 4, |b| < 256 is hi + lo with both parts exact bf16 (at most 12
significant bits), every product with an integer of magnitude < 2^8 is a multiple of 2^-8, and while
A = sum |x||w| < 2^12 (``assert_exact_grid``) every partial sum is a multiple of 2^-8 below 2^12: 20 significant
bits, exact in fp32 in any order of accumulation.  The kernel's fp32 result must then equal the float64 reference.

The last section holds SPyNet's fp32 glue kernels (spynet.cu) to float64 per element, with bounds derived from their
arithmetic (``check_bounded``), and decodes the row-gapped operand slot by slot."""
import json
import math
import os
import re
import tempfile
from collections import namedtuple

import torch
import torch.nn.functional as F

C = 2.0 ** -14
ROUND = {"f32": 0.0, "f16": 2.0 ** -11, "split": 2.0 ** -16}   # relative rounding of the stored output format
GRID = 2.0 ** -8                                                # step of the exact-grid values
EXACT_LIMIT = 2.0 ** 12                                         # A below this: every fp32 partial sum is exact

Launch = namedtuple("Launch", "name grid smem")
PERSISTENT = re.compile(r"^(linear_kernel|conv3x3_kernel|conv3x3_dact_kernel|conv3x3_halo_kernel|conv_kxn_kernel)<")
TABLE = []         # rows of the schedule table: (case, kernel, grid, tiles, tiles per CTA, smem, note)
MARGINS = {}       # check -> worst err / per-element bound over its elements
INCOMPLETE = []    # traces without a record of every library kernel: (launched, recorded, kernel names)


# ------------------------------------------------------------------------------------------------ which kernel ran
_LITERALS = [(re.compile(r"\(bool\)0"), "false"), (re.compile(r"\(bool\)1"), "true"),
             (re.compile(r"\((?:unsigned )?int\)(-?\d+)"), r"\1")]


def short_name(name):
    """'void e2f::conv::conv3x3_kernel<(int)96, (bool)0>(e2f::conv::Maps, ...)' -> 'conv3x3_kernel<96, false>'."""
    for pat, rep in _LITERALS:
        name = pat.sub(rep, name)
    m = re.search(r"(\w+)\s*(<[^()]*>)?\s*\(", name)
    if m is None:
        return name
    return m.group(1) + re.sub(r"\s*,\s*", ", ", m.group(2) or "")


def run_traced(fn, attempts=3):
    """Run ``fn`` under torch.profiler (CUDA activity); return (its result, [Launch(name, grid, smem)] in launch
    order) read from the Kineto trace, which records each kernel's grid and shared memory.

    A trace is complete when it holds one record per kernel this library launched during ``fn`` (the e2f:: kernels,
    counted by ops.launch_count).  CUPTI sometimes delivers a trace that lacks some or all of them (an H100 run gave
    one with no kernel record at all); then ``fn``, a pure op, is traced again, at most ``attempts`` times in all.
    The last trace is returned either way and the caller's assertions decide; every incomplete trace is listed by
    ``print_tables``."""
    from e2fgvi_b200 import ops
    for _ in range(attempts):
        n0 = ops.launch_count()
        result, launches, recorded = _traced(fn)
        launched = ops.launch_count() - n0
        if recorded == launched:
            break
        INCOMPLETE.append((launched, recorded, [k.name for k in launches]))
    return result, launches


def _traced(fn):
    """(result, launches, number of e2f:: kernel records) of one profiled call."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        result = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0))
    recorded = sum(1 for e in kernels if "e2f::" in e["name"])
    return result, [Launch(short_name(e["name"]), tuple(e.get("args", {}).get("grid", ())),
                           e.get("args", {}).get("shared memory")) for e in kernels], recorded


def conv3x3_tanh_nchw_entry(x, weight, bias):
    """tanh(conv2d(x, weight, bias, 1, 1)) as contiguous (N, Cout, H, W) fp32 through the C entry e2f_conv3x3_tanh_nchw
    (the implicit-GEMM conv with the tanh / NCHW epilogue), which the Python wrappers do not call: they run the decoder's
    output conv on the kx-in-N kernel."""
    from e2fgvi_b200 import _lib, ops
    src = ops.split_nhwc(x)
    n, c, h, w = src.shape
    cout = weight.shape[0]
    w_hi, w_lo, _ = ops._conv3x3_operand(weight, [c], 1, 0)
    b32 = bias.detach().float().contiguous()
    out = torch.empty((n, cout, h, w), dtype=torch.float32, device=weight.device)
    st = _lib.load().e2f_conv3x3_tanh_nchw(src.hi.data_ptr(), src.lo.data_ptr(), src.hi.shape[-1], w_hi.data_ptr(),
                                           w_lo.data_ptr(), b32.data_ptr(), out.data_ptr(), n, h, w, cout,
                                           torch.cuda.current_stream().cuda_stream)
    _lib.check(st, "e2f_conv3x3_tanh_nchw")
    return out


def persistent_launch(launches):
    """The one persistent GEMM launch among ``launches`` (split / pack kernels around it are ignored)."""
    hits = [k for k in launches if PERSISTENT.match(k.name)]
    assert len(hits) == 1, [k.name for k in launches]
    return hits[0]


def same_launch(la, lb):
    """Both traces ran the same persistent kernel on the same grid; returns it."""
    a, b = persistent_launch(la), persistent_launch(lb)
    assert (a.name, a.grid) == (b.name, b.grid), (a, b)
    return a


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def expect_schedule(case, launch, kernel, tiles, note=""):
    """Assert the instantiation and grid == min(tiles, SMs); record the row of the schedule table."""
    s = sms()
    assert launch.name == kernel, (launch.name, kernel)
    grid = min(tiles, s)
    assert launch.grid == (grid, 1, 1), (launch.grid, tiles, s)
    TABLE.append((case, kernel, grid, tiles, -(-tiles // grid), launch.smem, note))
    return -(-tiles // grid)


def print_tables():
    """Print (and clear) the schedule table and the worst margin of every per-element check."""
    if TABLE:
        notes = any(row[6] for row in TABLE)
        print(f"\n{'case':44s} {'kernel':34s} {'grid':>5s} {'tiles':>6s} {'tiles/CTA':>9s} {'smem':>7s}"
              + ("  note" if notes else ""))
        for row in TABLE:
            print(f"{row[0]:44s} {row[1]:34s} {str(row[2]):>5s} {str(row[3]):>6s} {str(row[4]):>9s} {str(row[5]):>7s}"
                  + (f"  {row[6]}" if notes else ""))
    if MARGINS:
        print("\nworst |got - ref| / per-element bound, per check")
        for what, ratio in MARGINS.items():
            print(f"{what:44s} {ratio:.3f}")
    for launched, recorded, names in INCOMPLETE:
        print(f"incomplete trace, taken again: {recorded} of {launched} library kernels recorded {names}")
    TABLE.clear()
    MARGINS.clear()
    INCOMPLETE.clear()


# ------------------------------------------------------------------------------------------------ checks
def reference_math():
    """Context for the float64 references: cuDNN off, so convolutions run as im2col / col2im and cuBLAS GEMMs -- the
    same float64 arithmetic on every call, whatever algorithm cuDNN's heuristics would pick for a shape or the free
    memory (some of its algorithms are not exact on exact data, some add with atomics)."""
    return torch.backends.cudnn.flags(enabled=False)


def check_same_bits(got, again, what=""):
    """Two runs of one kernel on the same inputs give the same bits."""
    for a, b in zip(got if isinstance(got, (tuple, list)) else (got,), again if isinstance(again, (tuple, list)) else (again,)):
        if a is None:
            assert b is None, what
            continue
        assert a.dtype == b.dtype and a.shape == b.shape, what
        n = int((a.view(torch.int16 if a.element_size() == 2 else torch.int32)
                 != b.view(torch.int16 if b.element_size() == 2 else torch.int32)).sum())
        assert n == 0, f"{what}: {n} of {a.numel()} elements differ from run to run"


def check_close(got, ref, bound, tol, out_fmt="f32", what="", extra=None):
    """rel-of-max < tol, and per element |got - ref| <= C * bound + ROUND[out_fmt] * |ref| (+ ``extra``, an absolute
    allowance per element, e.g. the accumulation term of a long-K weight gradient)."""
    got = got.double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got - ref).abs()
    lim = C * bound + ROUND[out_fmt] * ref.abs()
    if extra is not None:
        lim = lim + extra
    worst = (err / lim.clamp_min(1e-300)).max().item()
    MARGINS[what] = worst
    assert worst <= 1.0, (what, int((err > lim).sum()), worst)
    rel = (err.max() / ref.abs().max().clamp_min(1e-30)).item()
    assert rel < tol, (what, rel)


def check_bounded(got, ref, bound, what="", rounding=0.0):
    """Per element |got - ref| <= bound + rounding * (|ref| + bound): ``bound`` an fp32 kernel's own error, derived
    from its arithmetic; ``rounding`` the relative rounding of the stored format (ROUND)."""
    got = got.double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    lim = bound + rounding * (ref.abs() + bound)
    worst = (err / lim.clamp_min(1e-300)).max().item()          # NaN in got fails too
    MARGINS[what] = worst
    assert worst <= 1.0, (what, int((err > lim).sum()), worst)


def check_bits(got, want, what=""):
    """got and want hold the same bits element by element."""
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    iv = torch.int16 if got.element_size() == 2 else torch.int32
    diff = got.contiguous().view(iv) != want.contiguous().view(iv)
    n = int(diff.sum())
    if n:
        first = [tuple(int(v) for v in idx) for idx in diff.nonzero()[:4].tolist()]
        raise AssertionError(f"{what}: {n} of {diff.numel()} elements differ in their bits; first at {first}: (got, want) "
                             f"{[(float(got[i]), float(want[i])) for i in first]}")


def check_exact(got, ref, what=""):
    """got == ref element by element (values: +0 and -0 compare equal, NaN never does); on failure report the count,
    the first differing coordinates and both values there."""
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    diff = got.double() != ref.double()
    n = int(diff.sum())
    if n:
        first = [tuple(int(v) for v in idx) for idx in diff.nonzero()[:4].tolist()]
        vals = [(float(got[i]), float(ref[i])) for i in first]
        raise AssertionError(f"{what}: {n} of {diff.numel()} elements differ; first at {first}: (got, ref) {vals}")


# ------------------------------------------------------------------------------------------------ exact-grid data
def grid_values(shape, gen, density=1.0, fine=False, device=None):
    """fp32 values a + b * 2^-8 (a in [-4, 4], b in [-255, 255]) with probability ``density``, else 0, or with
    ``fine`` one of -2^-8, 0, 2^-8: then every 64-pixel K block of a long-K sum (a weight gradient's) contributes,
    for about 2^-8 * 2/3 * E|other operand| of A per term."""
    dev = device if device is not None else gen.device
    a = torch.randint(-4, 5, shape, generator=gen, device=dev).float()
    b = torch.randint(-255, 256, shape, generator=gen, device=dev).float()
    keep = torch.rand(shape, generator=gen, device=dev) < density
    rest = torch.randint(-1, 2, shape, generator=gen, device=dev).float() * GRID if fine else torch.zeros((), device=dev)
    return torch.where(keep, a + b * GRID, rest)


def int_values(shape, gen, m=3, density=1.0, device=None):
    """fp32 integers in [-m, m], each nonzero with probability ``density``."""
    dev = device if device is not None else gen.device
    v = torch.randint(-m, m + 1, shape, generator=gen, device=dev).float()
    keep = torch.rand(shape, generator=gen, device=dev) < density
    return torch.where(keep, v, torch.zeros((), device=dev))


def assert_exact_grid(bound, grid_operand, what=""):
    """The precondition of an exact check: A < 2^12 everywhere, and the grid operand has elements whose bf16 lo part
    is nonzero (so the lo products contribute)."""
    a_max = float(bound.max())
    assert a_max < EXACT_LIMIT, (what, a_max)
    x = grid_operand.float()
    assert torch.any((x - x.bfloat16().float()) != 0), (what, "no element has a nonzero lo part")
    return a_max


def f32_split(v):
    """The (hi, lo) bf16 pair the kernels' epilogues store for the fp32 value v (round to nearest even, twice)."""
    hi = v.float().bfloat16()
    return hi, (v.float() - hi.float()).bfloat16()


# ------------------------------------------------------------------------------------------------ tile arithmetic
def cdiv(a, b):
    return -(-a // b)


def conv_tile(h, w, stride=1):
    """(tile_w, tile_h) that launch_conv3x3 / launch_conv3d pick for an h x w output grid (dense sources)."""
    if w < 16 or h < 8:
        return min(w, 16), min(h, 8)
    best, tw, th = cdiv(h, 8) * cdiv(w, 16), 16, 8
    for t in range(32, 7, -1):
        u = 128 // t
        if u < 4 or u > h or t > w or t * stride > 256 or u * stride > 256:
            continue
        cnt = cdiv(h, u) * cdiv(w, t)
        if cnt < best:
            best, tw, th = cnt, t, u
    return tw, th


def conv_bn(cog):
    return 32 if cog <= 32 else 64 if cog <= 64 else 96 if cog == 96 else 128


def generic_tiles(n, oh, ow, cout, groups=1, stride=1, tile=None, nphase=1, in_rows=False):
    """(BN, tiles) of conv3x3_kernel for an oh x ow GEMM grid (incl. the N-tile halving for launches of few tiles)."""
    tw, th = tile or conv_tile(oh, ow, stride)
    cog = cout // groups
    bn = conv_bn(cog)
    per = n * cdiv(oh, th) * cdiv(ow, tw) * groups * nphase
    if bn == 128 and cog % 64 == 0 and not in_rows and 2 * per * cdiv(cog, 128) <= sms():
        bn = 64
    return bn, per * cdiv(cog, bn)


def halo_tiles(n, h, w):
    return n * cdiv(h, 16) * cdiv(w, 8)


def kxn_tiles(n, h, w, ks, groups=1):
    return n * cdiv(h, 4) * cdiv(w, 32 - 2 * (ks // 2)) * groups


def images_for(tiles_of, want):
    """Smallest image count n with tiles_of(n) >= want."""
    n = 1
    while tiles_of(n) < want:
        n += 1
    return n


def cta_tiles(tiles, grid):
    """Tile indices of each CTA of a persistent launch: CTA b takes b, b + grid, ..."""
    return [range(b, tiles, grid) for b in range(grid)]


# ------------------------------------------------------------------------------------------------ SPyNet glue
# The fp32 glue kernels of csrc/spynet.cu against float64 restatements (oracle/restate_flow.py), per element.  A
# bilinear sample in fp32 differs from the float64 one in two ways:
#   * the blend rounds: with U = 2^-24, a weight l0 = 1 - l1 is within U of its value relative (l1 = src - i0 is
#     exact), and each product and sum rounds once, so a 2-D blend l0y (l0x a + l1x b) + l1y (...) -- two weight
#     roundings and four operations on every term's path -- is within 6 U * sum_i w_i |x_i| (the warp's products of
#     two weights and four fmas: 7 U);
#   * the source coordinate rounds: align_corners=True computes s = fl(scale) * dst (2 U s); align_corners=False
#     s = fl(scale) * (dst + 0.5) - 0.5 (three roundings, each within U of at most scale (dst + 0.5) + 0.5).  The
#     blend is piecewise linear in s, so a coordinate off by ds moves it by at most ds times the largest difference
#     of neighbouring inputs over the intervals next to the sample (``_slopes``).
# Errors the inputs already carry pass through the convex blend unchanged (the larger of the 3 x 3 neighbourhood,
# since a rounded coordinate may pick the neighbouring tap), and move the slope by at most twice that.  Everything
# above is first order; the bounds carry a factor 1 + 2^-20 for the products of two roundings.
U = 2.0 ** -24
SECOND_ORDER = 1.0 + 2.0 ** -20


def src_coords(n_in, n_out, align_corners, device=None):
    """ATen's float64 source coordinate of every output index of a bilinear resize n_in -> n_out, and the bound on
    how far the fp32 kernels' coordinate (spynet.cu src_index) is from it."""
    d = torch.arange(n_out, dtype=torch.float64, device=device)
    if align_corners:
        scale = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
        return scale * d, 2 * U * scale * d
    scale = n_in / n_out
    return (scale * (d + 0.5) - 0.5).clamp_min(0), 3 * U * (scale * (d + 0.5) + 0.5)


def _taps(src, n_in):
    i0 = src.floor().long().clamp(max=n_in - 1)
    return i0, (i0 + 1).clamp(max=n_in - 1), src - i0


def _blend(x, ty, tx):
    """Bilinear samples of x (N, C, h, w) at separable taps ((i0, i1, l1) per output row, per output column)."""
    (y0, y1, ly), (x0, x1, lx) = ty, tx
    ly = ly[:, None]
    r0, r1 = x[..., y0, :], x[..., y1, :]
    return (1 - ly) * ((1 - lx) * r0[..., x0] + lx * r0[..., x1]) + ly * ((1 - lx) * r1[..., x0] + lx * r1[..., x1])


def _slopes(x):
    """(Sy, Sx) of x (N, C, h, w): Sy[r, c] = the largest |x[r' + 1, c'] - x[r', c']| over r' in r-1 .. r+1 and
    c' in c, c+1 -- the y slope of every interval a sample whose top-left tap is (r, c) reaches when its coordinate
    moves by less than a pixel; Sx likewise in x."""
    h, w = x.shape[-2:]
    sy = torch.zeros_like(x) if h == 1 else F.max_pool2d(F.pad((x[..., 1:, :] - x[..., :-1, :]).abs(), (0, 1, 1, 2)), (3, 2), 1)
    sx = torch.zeros_like(x) if w == 1 else F.max_pool2d(F.pad((x[..., 1:] - x[..., :-1]).abs(), (1, 2, 0, 1)), (2, 3), 1)
    return sy, sx


def resize_bound(x, size, align_corners, arith=6, x_err=None):
    """Per output element of an fp32 bilinear resize of x (N, C, h, w) float64 -- the values the kernel reads -- to
    ``size``: arith * U * sum_i w_i |x_i| + (coordinate error) * slope (+ the blend of ``x_err``, the error the
    kernel's inputs carry).  See the section comment for the derivation."""
    h, w = x.shape[-2:]
    (sy, dy), (sx, dx) = src_coords(h, size[0], align_corners, x.device), src_coords(w, size[1], align_corners, x.device)
    ty, tx = _taps(sy, h), _taps(sx, w)
    gy, gx = _slopes(x)
    dy = dy[:, None]
    if x_err is not None:
        near = F.max_pool2d(x_err, 3, 1, 1)
        gy, gx = gy + 2 * near, gx + 2 * near
    b = arith * U * _blend(x.abs(), ty, tx) + dy * gy[..., ty[0], :][..., tx[0]] + dx * gx[..., ty[0], :][..., tx[0]]
    if x_err is not None:
        b = b + _blend(near, ty, tx)
    return b * SECOND_ORDER


def spynet_sizes(H, W):
    """(h, w, h_up, w_up) of a SPyNet estimate on H x W frames: the 1/4 size and its round-up to multiples of 32."""
    h, w = int(H * 0.25), int(W * 0.25)
    return h, w, -(-h // 32) * 32, -(-w // 32) * 32


def spynet_pairs(b, l_t):
    """(ref, supp) indices, into the b * l_t local frames, of the 2 * b * (l_t - 1) pairs: the forward pairs (j, j + 1)
    of every clip, then the backward pairs (j + 1, j)."""
    fwd = [(bi * l_t + j, bi * l_t + j + 1) for bi in range(b) for j in range(l_t - 1)]
    return fwd + [(s, r) for r, s in fwd]


def pyramid_reference(frames, l_t, mean, std, unit):
    """Float64 pyramid of the local frames of ``frames`` (b, t, 3, H, W) fp32 (restate_flow: (x + 1) / 2 unless
    ``unit``, quarter, pyramid) and the per-element bound on the fp32 kernel's level 0:

        e1 = resize_bound(x01 -> (h, w), align_corners=True, x_err = U x01 for the rounding of x + 1)
        e2 = resize_bound(small -> (h_up, w_up), align_corners=False, x_err = e1)
        level 0:  e2 / std + 2 U |ref|   (v - mean and the division each round once)."""
    from oracle import restate_flow
    H, W = frames.shape[-2:]
    x = frames[:, :l_t].reshape(-1, 3, H, W).double()
    x01 = x if unit else (x + 1) / 2
    small = restate_flow.quarter(x01)
    m, s = mean.double().view(1, 3, 1, 1), std.double().view(1, 3, 1, 1)
    levels = restate_flow.pyramid(small, m, s)
    e1 = resize_bound(x01, small.shape[-2:], True, x_err=None if unit else U * x01)
    e2 = resize_bound(small, levels[0].shape[-2:], False, x_err=e1)
    return levels, (e2 / s.abs() + 2 * U * levels[0].abs()) * SECOND_ORDER


def pool32(x):
    """The kernel's 2x2 average pool in fp32: ((a + b) + c) + d, then / 4 -- ATen avg_pool2d's order."""
    return (((x[..., 0::2, 0::2] + x[..., 0::2, 1::2]) + x[..., 1::2, 0::2]) + x[..., 1::2, 1::2]) / 4


def check_pyramid(levels, frames, l_t, mean, std, unit, what):
    """Level 0 per element against float64; every level k >= 1 bit for bit the fp32 pool of the kernel's level k-1."""
    ref, bound = pyramid_reference(frames, l_t, mean, std, unit)
    check_bounded(levels[0], ref[0], bound, f"{what} level 0")
    for k in range(1, 6):
        check_bits(levels[k], pool32(levels[k - 1]), f"{what} level {k}")
    return ref


def exact_pyramid_budget(frames, l_t, mean, std, unit, ref):
    """The precondition of comparing every level with float64 exactly.

    Level 0: the frames are multiples of 1/4 (x01 = (x + 1) / 2 then of 1/8, exact), and every source coordinate of
    both resizes is dyadic, so a blend weight is a multiple of 1 / den (den: the coordinate's denominator) and every
    product and partial sum of either blend is a multiple of g0 = grid / (den1y den1x den2y den2x) in [0, 1]: exact in
    fp32 while 1 / g0 <= 2^24.  mean 0 and std a power of two leave it exact.
    Levels 1..5: each pool's partial sums (a + b), (a + b) + c, ((a + b) + c) + d of the float64 level k-1 must be
    fp32 numbers; then by induction the kernel's fp32 pool of an exact level is exact (/ 4 is).  Returns log2(1 / g0)."""
    from fractions import Fraction
    H, W = frames.shape[-2:]
    h, w, hu, wu = spynet_sizes(H, W)
    x = frames[:, :l_t].double()
    grid = 4 if unit else 8
    assert torch.equal(x * 4, (x * 4).round()) and float(x.abs().max()) <= 1.0, "frames off the 1/4 grid"
    den = 1
    for n_in, n_out in ((H, h), (W, w)):
        den *= Fraction(n_in - 1, n_out - 1).denominator            # s = scale * dst
    for n_in, n_out in ((h, hu), (w, wu)):
        den *= (Fraction(n_in, n_out) * Fraction(1, 2)).denominator   # s = scale * (dst + 1/2) - 1/2
    bits = (grid * den).bit_length() - 1
    assert grid * den == 1 << bits, ("a coordinate is not dyadic", H, W)
    assert bits <= 24, ("level 0 needs more than 24 significant bits", bits)
    assert float(mean.abs().max()) == 0.0, "mean must be 0"
    for v in std.double().view(-1).tolist():
        assert v > 0 and math.log2(v).is_integer(), ("std must be a power of two", v)
    for k in range(1, 6):
        p = ref[k - 1]
        for part in (p[..., 0::2, 0::2] + p[..., 0::2, 1::2],
                     p[..., 0::2, 0::2] + p[..., 0::2, 1::2] + p[..., 1::2, 0::2],
                     p[..., 0::2, 0::2] + p[..., 0::2, 1::2] + p[..., 1::2, 0::2] + p[..., 1::2, 1::2]):
            assert torch.equal(part, part.float().double()), ("a pool partial sum is not an fp32 number", k)
    return bits


def exact_frames(b, t, l_t, H, W, unit, seed):
    """Sparse CPU frames (b, t, 3, H, W) on the 1/4 grid: background -1 (0 with ``unit``; x01 = 0 either way), a few
    random pixels and the four corners and four edge midpoints at x01 = 1/8 or 1/4 (1/4 or 1/2 with ``unit``), so
    that every pool of every level stays within 24 significant bits (exact_pyramid_budget).  Frames j >= l_t, which
    the pyramid must not read, are NaN."""
    g = torch.Generator().manual_seed(seed)
    x01 = torch.zeros(b, t, 3, H, W)
    pick = torch.rand(b, t, 3, H, W, generator=g) < 0.004
    step = 0.25 if unit else 0.125
    x01[pick] = torch.randint(1, 3, (int(pick.sum()),), generator=g).float() * step
    for y, xx in ((0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (0, W // 2), (H - 1, W // 2), (H // 2, 0), (H // 2, W - 1)):
        x01[..., y, xx] = torch.randint(1, 3, (b, t, 3), generator=g).float() * step
    x = x01 if unit else x01 * 2 - 1
    x[:, l_t:] = float("nan")
    return x


def rows_decode(flat, n, h, w, lead, pitch, tail, cin):
    """Slots of a row-gapped buffer (ops.RowsNHWC: [n][h][pitch][cin], then ``tail`` pixels): (the pixels
    (n, h, w, cin), every gap, rounding and tail slot as one flat tensor)."""
    assert flat.numel() == (n * h * pitch + tail) * cin, (flat.numel(), n, h, pitch, tail, cin)
    body = flat[: n * h * pitch * cin].view(n, h, pitch, cin)
    gaps = torch.cat([body[:, :, :lead].reshape(-1), body[:, :, lead + w:].reshape(-1), flat[n * h * pitch * cin:]])
    return body[:, :, lead: lead + w], gaps


def warp_bound(supp, flow_up):
    """Per element bound on the fp32 border-mode warp of supp (P, 3, h, w) float64 at (x + u, y + v), flow_up
    (P, h, w, 2) the kernel's fp32 flow: 7 U * sum_i w_i |s_i| for the weights and the four fmas, plus the coordinate
    term.  The kernel rounds x + u once (U |x + u|); the float64 reference's normalise / unnormalise round trip in
    grid_sample adds a few 2^-53 of (|x + u| + 1), inside the U * 1 that the coordinate bound adds."""
    n, c, h, w = supp.shape
    gy, gx = torch.meshgrid(torch.arange(h, dtype=torch.float64, device=supp.device),
                            torch.arange(w, dtype=torch.float64, device=supp.device), indexing="ij")
    ix, iy = gx + flow_up[..., 0].double(), gy + flow_up[..., 1].double()
    px, py = ix.clamp(0, w - 1), iy.clamp(0, h - 1)
    x0, y0 = px.floor().long().clamp(max=w - 1), py.floor().long().clamp(max=h - 1)
    x1, y1 = (x0 + 1).clamp(max=w - 1), (y0 + 1).clamp(max=h - 1)
    lx, ly = (px - x0)[:, None], (py - y0)[:, None]

    def at(t, yi, xi):
        return t.flatten(2).gather(2, (yi * w + xi).flatten(1)[:, None].expand(-1, t.shape[1], -1)).view(t.shape)

    a = supp.abs()
    blend = (1 - ly) * ((1 - lx) * at(a, y0, x0) + lx * at(a, y0, x1)) + ly * ((1 - lx) * at(a, y1, x0) + lx * at(a, y1, x1))
    sy, sx = _slopes(supp)
    dx, dy = (U * (ix.abs() + 1))[:, None], (U * (iy.abs() + 1))[:, None]
    return (7 * U * blend + dx * at(sx, y0, x0) + dy * at(sy, y0, x0)) * SECOND_ORDER


def check_level_input(hi, lo, pitch, tail, lead, flow_up, img, prev, b, l_t, what):
    """The row-gapped operand (flat bf16 hi, lo) and flow_up (P, hk, wk, 2) of one SPyNet level, img the level's
    pyramid image (b * l_t, 3, hk, wk) fp32 and prev the coarser flow (P, hk/2, wk/2, 2) or None:
      * flow_up per element against float64 2 * up2x(prev) (resize_bound, times 2), or bitwise 0 without prev;
      * every gap and tail slot bitwise 0 in hi and lo;
      * channels 0..2 bitwise the split of the pair's ref frame, 6..7 of flow_up;
      * channels 3..5: hi + lo per element against the float64 border warp of the pair's support frame at the
        kernel's own flow_up (warp_bound, plus 2^-16 for the split); without prev, the split of the support frame."""
    from oracle import restate_flow
    hk, wk = img.shape[-2:]
    P = 2 * b * (l_t - 1)
    assert flow_up.shape == (P, hk, wk, 2), (what, tuple(flow_up.shape))
    if prev is None:
        check_bits(flow_up, torch.zeros_like(flow_up), f"{what} flow_up")
    else:
        p64 = prev.double().permute(0, 3, 1, 2)
        check_bounded(flow_up.permute(0, 3, 1, 2), restate_flow.upsample_flow(p64), 2 * resize_bound(p64, (hk, wk), True),
                      f"{what} flow_up")
    h_px, h_gaps = rows_decode(hi, P, hk, wk, lead, pitch, tail, 8)
    l_px, l_gaps = rows_decode(lo, P, hk, wk, lead, pitch, tail, 8)
    check_bits(h_gaps, torch.zeros_like(h_gaps), f"{what} gaps hi")
    check_bits(l_gaps, torch.zeros_like(l_gaps), f"{what} gaps lo")
    pairs = spynet_pairs(b, l_t)
    ref = img[[r for r, _ in pairs]].permute(0, 2, 3, 1)
    supp = img[[s for _, s in pairs]]
    for (got_h, got_l), v, name in (((h_px[..., 0:3], l_px[..., 0:3]), ref, "ref"),
                                    ((h_px[..., 6:8], l_px[..., 6:8]), flow_up, "flow_up")):
        want_h, want_l = f32_split(v)
        check_bits(got_h.contiguous(), want_h, f"{what} {name} hi")
        check_bits(got_l.contiguous(), want_l, f"{what} {name} lo")
    got = (h_px[..., 3:6].double() + l_px[..., 3:6].double()).permute(0, 3, 1, 2)
    if prev is None:
        want_h, want_l = f32_split(supp)
        check_exact(h_px[..., 3:6].permute(0, 3, 1, 2), want_h, f"{what} identity warp hi")
        check_exact(l_px[..., 3:6].permute(0, 3, 1, 2), want_l, f"{what} identity warp lo")
    s64 = supp.double()
    check_bounded(got, restate_flow.flow_warp(s64, flow_up.double()), warp_bound(s64, flow_up), f"{what} warp",
                  ROUND["split"])


def check_final(fwd, bwd, flow, h, w, what):
    """flows_forward / flows_backward (b, l_t-1, 2, h, w) of spynet_final on the level-0 flow (P, h_up, w_up, 2): the
    first P/2 pairs forward, the rest backward, per element against float64 resize_flow; bound resize_bound times
    the rescale, plus 2 U |ref| for the fp32 rescale factor and product."""
    from oracle import restate_flow
    P, hu, wu, _ = flow.shape
    f64 = flow.double().permute(0, 3, 1, 2)
    ref = restate_flow.resize_flow(f64, h, w)
    rs = torch.tensor([w / wu, h / hu], dtype=torch.float64, device=flow.device).view(1, 2, 1, 1)
    bound = (resize_bound(f64, (h, w), False) * rs + 2 * U * ref.abs()) * SECOND_ORDER
    got = torch.cat([fwd.reshape(-1, 2, h, w), bwd.reshape(-1, 2, h, w)])
    check_bounded(got, ref, bound, what)
