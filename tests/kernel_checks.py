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
bits, exact in fp32 in any order of accumulation.  The kernel's fp32 result must then equal the float64 reference."""
import json
import os
import re
import tempfile
from collections import namedtuple

import torch

C = 2.0 ** -14
ROUND = {"f32": 0.0, "f16": 2.0 ** -11, "split": 2.0 ** -16}   # relative rounding of the stored output format
GRID = 2.0 ** -8                                                # step of the exact-grid values
EXACT_LIMIT = 2.0 ** 12                                         # A below this: every fp32 partial sum is exact

Launch = namedtuple("Launch", "name grid smem")
PERSISTENT = re.compile(r"^(linear_kernel|conv3x3_kernel|conv3x3_dact_kernel|conv3x3_halo_kernel|conv_kxn_kernel)<")
TABLE = []         # rows of the schedule table: (case, kernel, grid, tiles, tiles per CTA, smem, note)
MARGINS = {}       # check -> worst err / (C * A + rounding) over its elements
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
        print("\nworst |got - ref| / (C * A + rounding) per check")
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
