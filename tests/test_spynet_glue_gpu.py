"""SPyNet's fp32 glue kernels (spynet.cu) against float64 restatements of the reference's ops (oracle/restate_flow),
element by element: spynet_pyramid ([-1, 1] and unit frames), spynet_level_input (every level, two leads) and
spynet_final.

* Random data at the model's sizes: level 0 of the pyramid, flow_up, the warp and the final flows are held per element
  to bounds derived from the kernels' fp32 arithmetic (kernel_checks, SPyNet glue section: a few 2^-24 of
  sum |w_i| |x_i| per blend and a coordinate term, the rounded source coordinate times the local slope of the
  input).  Pyramid levels 1..5 are compared bit for bit with the fp32 2x2 pool of the kernel's own level k-1.
* Exact data: sizes whose every scale and sample coordinate is dyadic, frames on the 1/4 grid, mean 0 and std a power
  of two.  Every level of the pyramid then equals float64 exactly (exact_pyramid_budget states why).
* The row-gapped operand is decoded slot by slot: gaps and tail zero, ref and flow_up channels the exact split,
  the pair order direction-major.
* Every kernel runs twice and gives the same bits.
* The frames j >= l_t of a clip are NaN, so a read of them (or a wrong per-clip stride) shows.

With pytest -s the worst err / bound of every per-element check is printed."""
import pytest
import torch

from e2fgvi_b200 import _lib, ops
from kernel_checks import (check_bits, check_exact, check_final, check_level_input, check_pyramid, check_same_bits,
                           exact_frames, exact_pyramid_budget, print_tables, pyramid_reference, reference_math,
                           spynet_sizes)

pytestmark = pytest.mark.gpu

MEAN = (0.485, 0.456, 0.406)                   # SPyNet's normalisation buffers
STD = (0.229, 0.224, 0.225)

# (b, t, l_t, H, W): the base model's 240x432 (60x108 -> 64x128); H and W not multiples of 4 (62x109 -> 64x128) with
# b > 1 and t > l_t; less than one 32x32 block after the 1/4 downsample (22x27 -> 32x32, the resize upsamples); h a
# multiple of 32 (64x130 -> 64x160, the y resize is the identity); the HQ bench sizes 720x1296 (180x324 -> 192x352)
# and 1080x1944 (270x486 -> 288x512)
CASES = [(1, 3, 3, 240, 432), (2, 5, 3, 250, 437), (2, 4, 2, 90, 110), (1, 4, 3, 256, 520), (1, 3, 3, 720, 1296),
         (2, 4, 3, 1080, 1944)]


@pytest.fixture(scope="module", autouse=True)
def margins_table():
    yield
    print_tables()


def _buffers(cuda, mean=MEAN, std=STD):
    return (torch.tensor(mean, device=cuda).view(1, 3, 1, 1), torch.tensor(std, device=cuda).view(1, 3, 1, 1))


def _frames(cuda, b, t, l_t, H, W, unit, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(b, t, 3, H, W, generator=g)
    x = x if unit else x * 2 - 1
    x[:, l_t:] = float("nan")
    return x.to(cuda)


@pytest.mark.parametrize("unit", [False, True])
@pytest.mark.parametrize("b,t,l_t,H,W", CASES)
def test_pyramid_against_float64(cuda, b, t, l_t, H, W, unit):
    x = _frames(cuda, b, t, l_t, H, W, unit, H + W + unit)
    mean, std = _buffers(cuda)
    pyr = ops.spynet_pyramid(x, l_t, mean, std, unit=unit)
    h, w, hu, wu = spynet_sizes(H, W)
    assert (pyr.size, pyr.up) == ((h, w), (hu, wu))
    assert [tuple(v.shape) for v in pyr.levels] == [(b * l_t, 3, hu >> k, wu >> k) for k in range(6)]
    with reference_math():
        check_pyramid(pyr.levels, x, l_t, mean, std, unit, f"pyramid {H}x{W} b{b} unit={int(unit)}")
    check_same_bits(pyr.levels, ops.spynet_pyramid(x, l_t, mean, std, unit=unit).levels, "pyramid")


@pytest.mark.parametrize("unit", [False, True])
@pytest.mark.parametrize("H,W", [(69, 133), (133, 69)])
def test_pyramid_exact(cuda, H, W, unit):
    """h - 1, w - 1 powers of two (17, 33), h / h_up and w / w_up dyadic (17/32, 33/64): every level exact."""
    x = exact_frames(2, 4, 3, H, W, unit, H + unit).to(cuda)
    mean, std = _buffers(cuda, (0.0, 0.0, 0.0), (1.0, 0.5, 2.0))
    pyr = ops.spynet_pyramid(x, 3, mean, std, unit=unit)
    with reference_math():
        ref, _ = pyramid_reference(x, 3, mean, std, unit)
    exact_pyramid_budget(x, 3, mean, std, unit, ref)
    for k in range(6):
        assert float(ref[k].abs().max()) > 0
        check_exact(pyr.levels[k], ref[k].float(), f"exact pyramid {H}x{W} unit={int(unit)} level {k}")


@pytest.fixture(scope="module")
def level_pyramid(cuda):
    """b = 2 clips of t = 4 frames, l_t = 3 local ones, 240x432: levels 64x128 .. 2x4, 8 pairs."""
    mean, std = _buffers(cuda)
    return ops.spynet_pyramid(_frames(cuda, 2, 4, 3, 240, 432, False, 7), 3, mean, std)


@pytest.mark.parametrize("lead", [3, 1])
@pytest.mark.parametrize("k", [5, 4, 3, 2, 1, 0])
def test_level_input_against_float64(cuda, level_pyramid, k, lead):
    pyr = level_pyramid
    img = pyr.levels[k]
    _, _, hk, wk = img.shape
    P = 2 * pyr.b * (pyr.l_t - 1)
    tail = int(_lib.load().e2f_conv_rows_tail(lead, 8))
    g = torch.Generator().manual_seed(31 + k)
    # the model passes no flow at level 5; elsewhere flows of several pixels push samples past every border
    prev = None if k == 5 else (torch.randn(P, hk // 2, wk // 2, 2, generator=g) * 3).to(cuda)
    for p in (prev, None) if prev is not None else (None,):
        rows, flow_up = ops.spynet_level_input(pyr, k, p, lead)
        assert (rows.shape, rows.lead, rows.cin) == ((P, 8, hk, wk), lead, 8)
        with reference_math():
            check_level_input(rows.hi, rows.lo, rows.pitch, tail, lead, flow_up, img, p, pyr.b, pyr.l_t,
                              f"level {k} lead {lead}" + ("" if p is not None else " no flow"))
        rows2, flow_up2 = ops.spynet_level_input(pyr, k, p, lead)
        check_same_bits((rows.hi, rows.lo, flow_up), (rows2.hi, rows2.lo, flow_up2), "level input")


@pytest.mark.parametrize("b,t,l_t,H,W", CASES)
def test_final_against_float64(cuda, b, t, l_t, H, W):
    h, w, hu, wu = spynet_sizes(H, W)
    P = 2 * b * (l_t - 1)
    pyr = ops.FlowPyramid(None, b, l_t, (h, w), (hu, wu))
    flow = (torch.randn(P, hu, wu, 2, generator=torch.Generator().manual_seed(H)) * 4).to(cuda)
    fwd, bwd = ops.spynet_final(flow, pyr)
    assert fwd.shape == bwd.shape == (b, l_t - 1, 2, h, w)
    with reference_math():
        check_final(fwd, bwd, flow, h, w, f"final {H}x{W} b{b}")
    check_same_bits((fwd, bwd), ops.spynet_final(flow, pyr), "final")


@pytest.mark.parametrize("b,l_t,h,w", [(1, 3, 64, 128), (2, 2, 32, 96)])
def test_final_identity(cuda, b, l_t, h, w):
    """h and w multiples of 32: the resize and the rescale are exact, the flows are the level-0 flow as it is."""
    P = 2 * b * (l_t - 1)
    flow = torch.randn(P, h, w, 2, generator=torch.Generator().manual_seed(h + w)).to(cuda)
    fwd, bwd = ops.spynet_final(flow, ops.FlowPyramid(None, b, l_t, (h, w), (h, w)))
    want = flow.permute(0, 3, 1, 2).reshape(2, b, l_t - 1, 2, h, w)
    check_bits(fwd, want[0].contiguous(), "final identity forward")
    check_bits(bwd, want[1].contiguous(), "final identity backward")
