"""The SPyNet glue checks of kernel_checks have teeth: on the CPU, a float32 emulation of the three glue kernels of
spynet.cu (their fp32 source index, lerp, blend order, fma warp and bf16 split) passes the same checks the H100 tests
apply, and each fault such a kernel could carry -- a flipped align_corners, a dropped half-pixel offset or clamp, an
unclamped last tap, zero padding in the warp, a lost factor, a wrong rescale, a wrong pair order, a dirty gap slot, a
lo that is not the remainder of its hi -- fails them."""
import pytest
import torch

from kernel_checks import (check_exact, check_final, check_level_input, check_pyramid, exact_frames, exact_pyramid_budget,
                           pool32, pyramid_reference, spynet_pairs, spynet_sizes)

F32 = torch.float32


def _f(v):
    return torch.tensor(float(v), dtype=F32)


def _src(n_in, n_out, ac, faults):
    """spynet.cu src_index in fp32 ("no_half": without the - 0.5, "no_clamp": without the clamp at 0)."""
    d = torch.arange(n_out, dtype=F32)
    if ac:
        return (_f(n_in - 1) / _f(n_out - 1) if n_out > 1 else _f(0)) * d
    s = _f(n_in) / _f(n_out) * (d + 0.5)
    s = s if "no_half" in faults else s - 0.5
    return s if "no_clamp" in faults else s.clamp_min(0)


def _lerp(src, n_in, clamp_i1=True):
    """make_lerp: i0 by truncation, i1 clamped to the last index, l0 = 1 - l1."""
    i0 = src.to(torch.long)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0) if clamp_i1 else i0 + 1
    l1 = src - i0.to(F32)
    return i0, i1, 1 - l1, l1


def _read(x, yi, xi):
    """x[..., yi, :][..., xi] addressed as the kernels address memory: flat offsets into the whole buffer, so that an
    index one past the last column reads the next row and one past the last row the next plane (zeros past the end)."""
    n, c, h, w = x.shape
    flat = torch.cat([x.reshape(-1), x.new_zeros(2 * h * w)])
    base = torch.arange(n * c).view(n, c, 1, 1) * (h * w)
    return flat[base + yi.view(1, 1, -1, 1) * w + xi.view(1, 1, 1, -1)]


def _resize(x, size, ac, faults=()):
    """A bilinear resize as the kernels blend it: l0y (l0x a + l1x b) + l1y (l0x c + l1x d), in fp32.  Faults: "ac"
    flips align_corners, "i1_row" / "i1_col" leave the last row's / column's second tap unclamped."""
    h, w = x.shape[-2:]
    ac = (not ac) if "ac" in faults else ac
    y0, y1, ly0, ly1 = _lerp(_src(h, size[0], ac, faults), h, "i1_row" not in faults)
    x0, x1, lx0, lx1 = _lerp(_src(w, size[1], ac, faults), w, "i1_col" not in faults)
    ly0, ly1 = ly0.view(-1, 1), ly1.view(-1, 1)
    return ly0 * (lx0 * _read(x, y0, x0) + lx1 * _read(x, y0, x1)) + ly1 * (lx0 * _read(x, y1, x0) + lx1 * _read(x, y1, x1))


def emu_pyramid(frames, l_t, mean, std, unit, down=(), up=(), clip_stride=None):
    """spynet_pyramid_kernel: faults ``down`` / ``up`` on the 1/4 downsample / the resize to multiples of 32;
    ``clip_stride`` reads clip bi's frames at bi * clip_stride instead of bi * t."""
    b, t, _, H, W = frames.shape
    h, w, hu, wu = spynet_sizes(H, W)
    flat = frames.reshape(b * t, 3, H, W)
    x = flat[[bi * (clip_stride or t) + j for bi in range(b) for j in range(l_t)]]
    x01 = x if unit else (x + 1) / 2
    v = _resize(_resize(x01, (h, w), True, down), (hu, wu), False, up)
    levels = [(v - mean.view(1, 3, 1, 1)) / std.view(1, 3, 1, 1)]
    for _ in range(5):
        levels.append(pool32(levels[-1]))
    return levels


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def emu_level_input(img, prev, b, l_t, lead, faults=()):
    """spynet_level_input_kernel -> (hi, lo flat bf16, pitch, tail, flow_up).  Faults: "ac" (the x2 upsample),
    "no_x2" (flow_up without the factor 2), "zeros" (zeros padding in the warp), "clip_major" (pairs ordered clip,
    direction, j), "swap_bwd" (backward pairs with ref and support swapped), "gap" (one gap slot not zeroed), "lo"
    (lo the remainder of a truncated hi, not of the stored one)."""
    n, _, hk, wk = img.shape
    P = 2 * b * (l_t - 1)
    pairs = spynet_pairs(b, l_t)
    if "clip_major" in faults:
        per = b * (l_t - 1)
        pairs = [pairs[d * per + bi * (l_t - 1) + j] for bi in range(b) for d in range(2) for j in range(l_t - 1)]
    if "swap_bwd" in faults:
        pairs = pairs[: P // 2] + [(s, r) for r, s in pairs[P // 2:]]
    ref = img[[r for r, _ in pairs]]
    supp = img[[s for _, s in pairs]]
    if prev is None:
        fu = fv = torch.zeros(P, hk, wk, dtype=F32)
    else:
        up = _resize(prev.permute(0, 3, 1, 2).contiguous(), (hk, wk), True, faults)
        two = 1.0 if "no_x2" in faults else 2.0
        fu, fv = up[:, 0] * two, up[:, 1] * two
    gy, gx = torch.meshgrid(torch.arange(hk, dtype=F32), torch.arange(wk, dtype=F32), indexing="ij")
    px, py = gx + fu, gy + fv
    if "zeros" not in faults:
        px, py = px.clamp(0, wk - 1), py.clamp(0, hk - 1)
    fx0, fy0 = px.floor(), py.floor()
    lx, ly = px - fx0, py - fy0
    x0, y0 = fx0.long(), fy0.long()
    x1 = x0 + 1 if "zeros" in faults else (x0 + 1).clamp(max=wk - 1)
    y1 = y0 + 1 if "zeros" in faults else (y0 + 1).clamp(max=hk - 1)

    def tap(yi, xi):
        ok = ((yi >= 0) & (yi < hk) & (xi >= 0) & (xi < wk))[:, None]
        idx = (yi.clamp(0, hk - 1) * wk + xi.clamp(0, wk - 1)).flatten(1)[:, None].expand(-1, 3, -1)
        return torch.where(ok, supp.flatten(2).gather(2, idx).view(supp.shape), torch.zeros(()))

    acc = torch.zeros_like(supp)
    for wt, v in ((((1 - ly) * (1 - lx)), tap(y0, x0)), ((1 - ly) * lx, tap(y0, x1)), (ly * (1 - lx), tap(y1, x0)),
                  (ly * lx, tap(y1, x1))):
        acc = _fma(wt[:, None], v, acc)
    pitch, tail = lead + wk, lead + 8
    body = torch.zeros(P, hk, pitch, 8)
    body[:, :, lead:lead + wk] = torch.cat([ref, acc, torch.stack((fu, fv), 1)], 1).permute(0, 2, 3, 1)
    f = torch.cat([body.reshape(-1), torch.zeros(tail * 8)])
    hi = f.bfloat16()
    base = (f.view(torch.int32) & -65536).view(F32) if "lo" in faults else hi.float()
    lo = (f - base).bfloat16()
    if "gap" in faults:
        hi[(P * hk - 1) * pitch * 8 + 1] = 1.0          # a lead slot of the last row
    return hi, lo, pitch, tail, torch.stack((fu, fv), -1)


def emu_final(flow, b, l_t, h, w, faults=()):
    """spynet_final_kernel.  Faults: "ac", "no_half" (on the resize), "u_by_h" (u rescaled by h / h_up)."""
    P, hu, wu, _ = flow.shape
    r = _resize(flow.permute(0, 3, 1, 2).contiguous(), (h, w), False, faults)
    sv = _f(h) / _f(hu)
    su = sv if "u_by_h" in faults else _f(w) / _f(wu)
    out = torch.stack((r[:, 0] * su, r[:, 1] * sv), 1)
    return out[: P // 2].reshape(b, l_t - 1, 2, h, w), out[P // 2:].reshape(b, l_t - 1, 2, h, w)


# ------------------------------------------------------------------------------------------------ cases
MEAN = torch.tensor([0.485, 0.456, 0.406])
STD = torch.tensor([0.229, 0.224, 0.225])


def _frames(b, t, l_t, H, W, unit, seed):
    """Random frames; the frames j >= l_t, which the glue must not read, are NaN."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(b, t, 3, H, W, generator=g)
    x = x if unit else x * 2 - 1
    x[:, l_t:] = float("nan")
    return x


EXACT_MEAN = torch.zeros(3)
EXACT_STD = torch.tensor([1.0, 0.5, 2.0])


@pytest.mark.parametrize("unit", [False, True])
def test_pyramid_emulation_passes(unit):
    x = _frames(2, 4, 3, 50, 70, unit, 1)
    check_pyramid(emu_pyramid(x, 3, MEAN, STD, unit), x, 3, MEAN, STD, unit, "host pyramid")


@pytest.mark.parametrize("H,W", [(69, 133), (133, 69)])
@pytest.mark.parametrize("unit", [False, True])
def test_exact_pyramid_emulation(H, W, unit):
    x = exact_frames(2, 4, 3, H, W, unit, H + unit)
    ref, _ = pyramid_reference(x, 3, EXACT_MEAN, EXACT_STD, unit)
    assert exact_pyramid_budget(x, 3, EXACT_MEAN, EXACT_STD, unit, ref) <= 24
    got = emu_pyramid(x, 3, EXACT_MEAN, EXACT_STD, unit)
    for k in range(6):
        check_exact(got[k], ref[k].float(), f"host exact level {k}")
    with pytest.raises(AssertionError):
        exact_pyramid_budget(x, 3, EXACT_MEAN, torch.tensor([1.0, 0.3, 2.0]), unit, ref)
    with pytest.raises(AssertionError):             # (H - 6) / 4 - 1 is odd: the exact case must refuse this size
        exact_pyramid_budget(x[..., :-5, :-5], 3, EXACT_MEAN, EXACT_STD, unit, ref)


@pytest.mark.parametrize("down,up,stride", [(("ac",), (), None), ((), ("ac",), None), ((), ("no_half",), None),
                                            ((), ("no_clamp",), None), ((), ("i1_row",), None),
                                            ((), ("i1_col",), None), ((), (), 3)])
def test_pyramid_fault_fails(down, up, stride):
    x = _frames(2, 4, 3, 50, 70, False, 2)
    x[:, 3:] = torch.rand(2, 1, 3, 50, 70)           # readable, so that a wrong clip stride gives numbers, not NaN
    got = emu_pyramid(x, 3, MEAN, STD, False, down, up, stride)
    with pytest.raises(AssertionError):
        check_pyramid(got, x, 3, MEAN, STD, False, "host pyramid fault")


def _level_case(k, seed=3):
    """Level k of a b = 2, l_t = 3 pyramid of 64 x 96 and a coarser flow of several pixels (None at level 5)."""
    x = _frames(2, 3, 3, 250, 380, False, seed)
    img = emu_pyramid(x, 3, MEAN, STD, False)[k]
    hk, wk = img.shape[-2:]
    g = torch.Generator().manual_seed(seed + k)
    prev = None if k == 5 else torch.randn(8, hk // 2, wk // 2, 2, generator=g) * 3
    return img, prev


@pytest.mark.parametrize("k", range(6))
@pytest.mark.parametrize("lead", [3, 1])
def test_level_input_emulation_passes(k, lead):
    img, prev = _level_case(k)
    hi, lo, pitch, tail, flow_up = emu_level_input(img, prev, 2, 3, lead)
    check_level_input(hi, lo, pitch, tail, lead, flow_up, img, prev, 2, 3, "host level input")
    hi, lo, pitch, tail, flow_up = emu_level_input(img, None, 2, 3, lead)
    check_level_input(hi, lo, pitch, tail, lead, flow_up, img, None, 2, 3, "host level input identity")


@pytest.mark.parametrize("fault", ["ac", "no_x2", "zeros", "clip_major", "swap_bwd", "gap", "lo"])
def test_level_input_fault_fails(fault):
    img, prev = _level_case(1)
    hi, lo, pitch, tail, flow_up = emu_level_input(img, prev, 2, 3, 3, (fault,))
    with pytest.raises(AssertionError):
        check_level_input(hi, lo, pitch, tail, 3, flow_up, img, prev, 2, 3, f"host level input {fault}")


@pytest.mark.parametrize("H,W", [(250, 380), (128, 256), (90, 110)])
def test_final_emulation_passes(H, W):
    h, w, hu, wu = spynet_sizes(H, W)
    flow = torch.randn(8, hu, wu, 2, generator=torch.Generator().manual_seed(H)) * 4
    fwd, bwd = emu_final(flow, 2, 3, h, w)
    check_final(fwd, bwd, flow, h, w, "host final")


@pytest.mark.parametrize("fault", ["ac", "no_half", "u_by_h", "swap_directions"])
def test_final_fault_fails(fault):
    h, w, hu, wu = spynet_sizes(250, 380)
    flow = torch.randn(8, hu, wu, 2, generator=torch.Generator().manual_seed(4)) * 4
    fwd, bwd = emu_final(flow, 2, 3, h, w, (fault,))
    if fault == "swap_directions":
        fwd, bwd = bwd, fwd
    with pytest.raises(AssertionError):
        check_final(fwd, bwd, flow, h, w, f"host final {fault}")
