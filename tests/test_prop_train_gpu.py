"""H100: the feature propagation's backward against float64.

* The flow-warp backward (``ops.flow_warp_backward``: d flow and the sorted dx scatter) against float64 autograd of
  ``oracle.restate.flow_warp``, element by element, on NHWC C = 128 features and on 2-channel flow planes read in place
  from a (b, t-1, 2, h, w) tensor.  The float64 side samples at the kernel's fp32 positions (x + u rounded to fp32, with
  the derivative of the unrounded sum), so both take the same cells and the difference is the kernels' fp32 arithmetic:
  - dx: each term w_k dout is 3 roundings off (the weight is a product of two differences), and a destination's run of r
    terms plus the residual adds r + 1: |e| <= (r + 4) u (sum |w_k dout| + |residual|), u = 2^-24, r counted per case;
  - d flow: each channel's slope takes 6 roundings, and the channel sum adds 4 ceil(C / 128) + 5 (NHWC: 4-channel
    vectors per lane, then a 5-level shuffle tree) or C (NCHW: one thread's loop), the residual 1 more:
    |e| <= (12 + chain) u (sum_c |dout_c| sum_k |x at corner k| + |residual|).
  Exact-grid (dyadic) data give gradients equal to float64; a second run gives the same bits.
* The module (``BidirectionalPropagation.forward`` on the fused path) against float64 autograd of
  ``oracle.restate.bidirectional_propagation``, with the DCN's x and weight read through fp16 and LeakyReLU's decisions
  taken from the GPU forward (as test_align_train_gpu.py does for the alignment): every parameter, x and flow gradient
  within 1e-3 of the gradient's largest value; three Adam steps within 1e-3 of float64.
* Behaviour: the tracked output has the untracked call's bits, a second backward raises, an in-place parameter change
  raises autograd's version error, and the derived-weight caches follow optimizer steps.  Launch sets:
  test_gpu_schedules_prop.py."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.feat_prop import BidirectionalPropagation
from kernel_checks import check_same_bits
from oracle import restate

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


# ------------------------------------------------------------------------------------------------------------- warp
def _positions(flow):
    """float64 sample positions (py, px) whose values are the kernel's fp32 sums and whose derivative is the sum's."""
    n, h, w, _ = flow.shape
    f64 = flow.double().cpu()
    gy, gx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    f32 = flow.float().cpu()
    px32 = (gx.float()[None] + f32[..., 0]).double()
    py32 = (gy.float()[None] + f32[..., 1]).double()
    return gx[None], gy[None], f64, px32, py32


def _ref_warp(x, flow, dout, residual, flow_residual):
    gx, gy, f64, px32, py32 = _positions(flow)
    xl = x.detach().double().cpu().requires_grad_()
    fl = f64.clone().requires_grad_()
    px = gx + fl[..., 0]
    py = gy + fl[..., 1]
    px = px + (px32 - px).detach()
    py = py + (py32 - py).detach()
    out = restate.bilinear_gather(xl, py, px)
    out.backward(dout.detach().double().cpu())
    dx, dfl = xl.grad, fl.grad
    if residual is not None:
        dx = dx + residual.double().cpu()
    if flow_residual is not None:
        dfl = dfl + flow_residual.double().cpu()
    return dx, dfl, py32, px32


def _magnitudes(x, dout, py, px, residual, flow_residual):
    """(sum of |w_k dout| per dx element, sum_c |dout_c| sum_k |x at corner k| per pixel, the longest run) in float64."""
    n, c, h, w = x.shape
    xa, da = x.detach().double().cpu().abs(), dout.detach().double().cpu().abs()
    y0, x0 = torch.floor(py), torch.floor(px)
    ly, lx = py - y0, px - x0
    y0, x0 = y0.long(), x0.long()
    mag_x = torch.zeros(n, c, h * w, dtype=torch.float64)
    corner_abs = torch.zeros(n, c, h, w, dtype=torch.float64)
    count = torch.zeros(n, h * w, dtype=torch.float64)
    for dy, wy in ((0, 1 - ly), (1, ly)):
        for dx_, wx in ((0, 1 - lx), (1, lx)):
            yy, xx = y0 + dy, x0 + dx_
            inside = ((yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)).double()
            idx = (yy.clamp(0, h - 1) * w + xx.clamp(0, w - 1)).reshape(n, -1)
            wgt = (wy * wx * inside).reshape(n, 1, -1)
            mag_x.scatter_add_(2, idx[:, None].expand(n, c, -1), wgt * da.reshape(n, c, -1))
            count.scatter_add_(1, idx, inside.reshape(n, -1))
            corner_abs += torch.gather(xa.reshape(n, c, -1), 2, idx[:, None].expand(n, c, -1)).reshape(n, c, h, w) * \
                inside[:, None]
    mag_x = mag_x.view(n, c, h, w)
    if residual is not None:
        mag_x = mag_x + residual.double().cpu().abs()
    mag_f = (da * corner_abs).sum(1)[..., None].expand(n, h, w, 2)
    if flow_residual is not None:
        mag_f = mag_f + flow_residual.double().cpu().abs()
    return mag_x, mag_f, int(count.max())


def _warp_inputs(layout, n, c, h, w, flows, seed, dev, residuals=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    if layout == "nhwc":
        x = torch.randn(n, c, h, w, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    else:      # a slice flows[:, 1] of a (n, 3, 2, h, w) tensor: planes read in place with a batch stride
        x = (3 * torch.randn(n, 3, c, h, w, device=dev, generator=g))[:, 1]
    flow = 2 * torch.randn(n, h, w, 2, device=dev, generator=g)
    if flows == "outside":          # some samples partly, some wholly, outside the image
        flow = flow + torch.tensor([0.7 * w, -0.5 * h], device=dev)
        flow[0, : h // 2] += torch.tensor([-2.0 * w, 0.0], device=dev)
    elif flows == "integer":        # samples on integer coordinates
        flow = flow.round()
    dout = torch.randn(n, c, h, w, device=dev, generator=g)
    res = fres = None
    if residuals:
        res = torch.randn(n, c, h, w, device=dev, generator=g)
        fres = torch.randn(n, h, w, 2, device=dev, generator=g)
    return x, flow, dout, res, fres


@pytest.mark.parametrize("layout,n,c,h,w,flows", [
    ("nhwc", 1, 128, 60, 108, "random"),
    ("nhwc", 3, 128, 13, 19, "outside"),
    ("nhwc", 2, 128, 13, 19, "integer"),
    ("nchw", 1, 2, 60, 108, "random"),
    ("nchw", 2, 2, 13, 19, "outside"),
    ("nchw", 3, 2, 13, 19, "integer"),
])
def test_warp_backward_against_float64(cuda, layout, n, c, h, w, flows):
    x, flow, dout, res, fres = _warp_inputs(layout, n, c, h, w, flows, n * 31 + h, cuda)
    dx, dflow = ops.flow_warp_backward(x, flow, dout, residual=res, flow_residual=fres)
    torch.cuda.synchronize()
    rdx, rdf, py, px = _ref_warp(x, flow, dout, res, fres)
    mag_x, mag_f, r = _magnitudes(x, dout, py, px, res, fres)
    if flows == "outside":
        assert ((px <= -1) | (px >= w) | (py <= -1) | (py >= h)).any()
        part = lambda p, size: ((p > -1) & (p < 0)) | ((p > size - 1) & (p < size))      # noqa: E731
        assert (part(px, w) | part(py, h)).any()                                            # some partly outside
    if flows == "integer":
        assert ((px == px.round()) & (py == py.round())).all()
    chain = 4 * math.ceil(c / 128) + 5 if layout == "nhwc" else c
    for what, got, ref, bound in (("dx", dx, rdx, (r + 4) * U * mag_x), ("dflow", dflow, rdf, (12 + chain) * U * mag_f)):
        err = (got.double().cpu() - ref).abs()
        bad = err > bound
        assert not bad.any(), (what, int(bad.sum()), float((err / bound.clamp_min(1e-300)).max()))


@pytest.mark.parametrize("layout,c", [("nhwc", 128), ("nchw", 2)])
def test_warp_backward_exact_grid(cuda, layout, c):
    """Flows on a 1/4 grid (exact positions, weights on a 1/16 grid), x and dout on a 1/8 grid: every product and sum is
    exact in fp32, so both gradients equal float64.  Some samples fall outside the image, some on integer coordinates."""
    n, h, w = 2, 9, 11
    g = torch.Generator(device=cuda).manual_seed(5)
    x = torch.randint(-8, 9, (n, c, h, w), device=cuda, generator=g) / 8
    if layout == "nhwc":
        x = x.contiguous(memory_format=torch.channels_last)
    flow = torch.randint(-16, 17, (n, h, w, 2), device=cuda, generator=g) / 4
    dout = torch.randint(-8, 9, (n, c, h, w), device=cuda, generator=g) / 8
    dx, dflow = ops.flow_warp_backward(x, flow, dout)
    rdx, rdf, py, px = _ref_warp(x, flow, dout, None, None)
    assert ((px < 0) | (px > w - 1)).any() and (px == px.round()).any()
    assert torch.equal(dx.double().cpu(), rdx), float((dx.double().cpu() - rdx).abs().max())
    assert torch.equal(dflow.double().cpu(), rdf), float((dflow.double().cpu() - rdf).abs().max())


@pytest.mark.parametrize("layout,c", [("nhwc", 128), ("nchw", 2)])
def test_warp_backward_same_bits(cuda, layout, c):
    x, flow, dout, res, fres = _warp_inputs(layout, 4, c, 30, 54, "random", 3, cuda)
    flow[:, :, :20] = 0.25 * flow[:, :, :20].round()        # many samples sharing corners: long runs
    a = ops.flow_warp_backward(x, flow, dout, residual=res, flow_residual=fres)
    b = ops.flow_warp_backward(x, flow, dout, residual=res, flow_residual=fres)
    check_same_bits(a[0], b[0], "dx")
    check_same_bits(a[1], b[1], "dflow")
    only_x, none = ops.flow_warp_backward(x, flow, dout, need_flow=False, residual=res)
    assert none is None
    check_same_bits(only_x, a[0], "dx without dflow")


# ----------------------------------------------------------------------------------------------------------- module
C = 128


def _module(dev, seed, random_last):
    torch.manual_seed(seed)
    m = BidirectionalPropagation(C)
    for name in m.DIRECTIONS:
        for k in (0, 2):
            torch.nn.init.normal_(m.backbone[name][k].bias, std=0.1)
        if random_last:
            torch.nn.init.normal_(m.deform_align[name].conv_offset[-1].weight, std=0.01)
            torch.nn.init.normal_(m.deform_align[name].conv_offset[-1].bias, std=0.1)
    torch.nn.init.normal_(m.fusion.bias, std=0.1)
    return m.to(dev)


def _module_inputs(b, t, h, w, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(b, t, C, h, w, device=dev, generator=g)
    fb, ff = [2 * torch.randn(b, t - 1, 2, h, w, device=dev, generator=g) for _ in range(2)]
    return x, fb, ff


class _GpuDecisions:
    """``torch.nn.functional`` for the restatement with LeakyReLU's decisions taken from the GPU forward, in call
    order (the gradients are those of the function the GPU evaluated)."""

    def __init__(self, masks):
        self.masks, self.i = masks, 0

    def __getattr__(self, name):
        return getattr(F, name)

    def leaky_relu(self, v, slope):
        mask = self.masks[self.i % len(self.masks)]
        self.i += 1
        return torch.where(mask, v, slope * v)


def _gpu_decisions(m, x, fb, ff):
    keep = {}
    with torch.no_grad():
        x32 = x.permute(0, 1, 3, 4, 2).contiguous().float()
        m._propagate_keep(x32, *ops.split_bf16(x32), fb, ff, keep)
    masks = []
    for name in m.DIRECTIONS:
        for st in keep["steps"][name]:
            if "acts" in st:
                masks += [(a > 0).cpu() for a in st["acts"][1:]]
            masks.append((st["y32"] > 0).cpu())
    return _GpuDecisions(masks)


def _fp16(t):
    return t + (t.detach().half().double() - t.detach())


def _patch_restate(monkeypatch, m, x, fb, ff):
    """The restatement with the DCN's x and weight read through fp16 (identity derivative) and the GPU's LeakyReLU
    decisions."""
    dcn = restate.modulated_deform_conv2d
    monkeypatch.setattr(restate, "modulated_deform_conv2d",
                        lambda xx, off, mask, wt, *a, **k: dcn(_fp16(xx), off, mask, _fp16(wt), *a, **k))
    monkeypatch.setattr(restate, "F", _gpu_decisions(m, x, fb, ff))


def _ref_module(monkeypatch, m, x, fb, ff, dy):
    sd = {f"m.{k}": v.detach().double().cpu().requires_grad_() for k, v in m.state_dict().items()}
    leaves = [t.detach().double().cpu().requires_grad_() for t in (x, fb, ff)]
    _patch_restate(monkeypatch, m, x, fb, ff)
    out = restate.bidirectional_propagation(sd, "m", *leaves)
    out.backward(dy.double().cpu())
    monkeypatch.undo()
    return out.detach(), [t.grad for t in leaves], {k[2:]: v.grad for k, v in sd.items()}


@pytest.mark.parametrize("b,t,random_last", [(1, 2, False), (2, 3, True), (1, 5, True), (2, 5, False)])
def test_module_against_float64(cuda, monkeypatch, b, t, random_last):
    m = _module(cuda, 3 + t, random_last)
    x, fb, ff = _module_inputs(b, t, 6, 10, cuda, 4 + b)
    leaves = [v.clone().requires_grad_() for v in (x, fb, ff)]
    out = m(*leaves)
    assert out.grad_fn is not None
    dy = torch.randn(out.shape, device=cuda, generator=torch.Generator(device=cuda).manual_seed(9))
    out.backward(dy)
    ref_out, ref_in, ref_p = _ref_module(monkeypatch, m, x, fb, ff, dy)
    assert float((out.detach().double().cpu() - ref_out).abs().max()) <= 1e-3 * float(ref_out.abs().max())
    pairs = [(what, v.grad, r) for what, v, r in zip(("x", "flows_backward", "flows_forward"), leaves, ref_in)]
    pairs += [(k, p.grad, ref_p[k]) for k, p in m.named_parameters()]
    for what, gk, r in pairs:
        assert gk is not None, what
        gk = gk.double().cpu()
        scale = float(r.abs().max())
        err = float((gk - r).abs().max())
        assert err <= 1e-3 * scale, (what, err, scale)


def test_tracked_output_same_bits_and_second_backward(cuda):
    m = _module(cuda, 5, True)
    x, fb, ff = _module_inputs(2, 4, 8, 12, cuda, 6)
    with torch.no_grad():
        want = m(x, fb, ff)
    xg = x.clone().requires_grad_()
    out = m(xg, fb, ff)
    assert out.grad_fn is not None
    check_same_bits(out, want, "tracked output")
    out1 = m(x[:1], fb[:1], ff[:1])
    with torch.no_grad():
        check_same_bits(out1, m(x[:1], fb[:1], ff[:1]), "tracked output, one clip")
    out.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second time"):
        out.sum().backward()
    out = m(x, fb, ff)
    with torch.no_grad():
        m.fusion.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.sum().backward()


@pytest.mark.parametrize("b", [1, 2])
def test_backward_leaves_the_incoming_gradient_alone(cuda, b):
    """The output also feeds a sibling branch (out + 2 y, as the generator adds the propagation's output to other
    features), and the incoming gradient has the output's own memory layout, so that for one clip its (t, b, h, w, c)
    view is contiguous: the backward must not write into it, and the sibling's gradient is exactly 2 x it."""
    m = _module(cuda, 21, True)
    x, fb, ff = _module_inputs(b, 3, 6, 10, cuda, 22)
    xg = x.clone().requires_grad_()
    y = torch.zeros_like(x, requires_grad=True)
    dy = torch.randn(b, 3, 6, 10, C, device=cuda).permute(0, 1, 4, 2, 3)
    keep = dy.clone()
    (m(xg, fb, ff) + 2 * y).backward(dy)
    check_same_bits(dy, keep, "incoming gradient after the backward")
    check_same_bits(y.grad, 2 * keep, "the sibling branch's gradient")
    ref = x.clone().requires_grad_()
    m(ref, fb, ff).backward(keep.clone())
    check_same_bits(xg.grad, ref.grad, "x's gradient")


def test_caches_follow_optimizer_steps(cuda):
    """After optimizer steps the tracked forward and backward give the bits of a fresh copy of the module, whose
    derived operands (packed / split / transposed weights) are built from scratch."""
    m = _module(cuda, 8, True)
    x, fb, ff = _module_inputs(1, 3, 6, 8, cuda, 2)
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    for _ in range(2):
        opt.zero_grad()
        m(x, fb, ff).square().mean().backward()
        opt.step()
    fresh = copy.deepcopy(m)           # new parameter objects: every derived operand is built from scratch
    for mod in (m, fresh):
        mod.zero_grad()
    a, b = m(x, fb, ff), fresh(x, fb, ff)
    check_same_bits(a, b, "output after optimizer steps")
    a.square().mean().backward()
    b.square().mean().backward()
    for (k, p), q in zip(m.named_parameters(), fresh.parameters()):
        check_same_bits(p.grad, q.grad, k)


def test_adam_steps_track_float64(cuda, monkeypatch):
    """Three Adam steps on a linear loss (the inner product with a fixed random tensor) next to the same steps in float64
    autograd of the restatement (the DCN's x and weight read through fp16): every parameter's total update is within
    1e-3 (L2, relative).  Each parameter's Adam eps is 10x its largest first gradient (as in test_align_train_gpu.py),
    so that near-zero gradient elements do not turn into full-size updates; each float64 step takes LeakyReLU's
    decisions from the GPU forward at that step's parameters."""
    m = _module(cuda, 13, True)
    x, fb, ff = _module_inputs(1, 3, 6, 10, cuda, 14)
    target = torch.randn(1, 3, C, 6, 10, device=cuda)
    xg = x.clone().requires_grad_()
    named = dict(m.named_parameters())
    p0 = {k: v.detach().clone() for k, v in named.items()}
    (m(xg, fb, ff) * target).mean().backward()
    eps = {k: 10 * float(v.grad.abs().max()) + 1e-30 for k, v in named.items()}
    m.zero_grad()
    opt = torch.optim.Adam([{"params": [named[k]], "eps": eps[k]} for k in named], lr=1e-3)
    gpu_params = []
    for _ in range(3):
        gpu_params.append({k: v.detach().clone() for k, v in named.items()})
        opt.zero_grad()
        (m(xg, fb, ff) * target).mean().backward()
        opt.step()
    final = {k: v.detach().clone() for k, v in named.items()}
    ref = {k: v.detach().double().cpu().clone().requires_grad_() for k, v in p0.items()}
    ropt = torch.optim.Adam([{"params": [ref[k]], "eps": eps[k]} for k in named], lr=1e-3)
    xs = [v.double().cpu() for v in (x, fb, ff)]
    for step in range(3):
        with torch.no_grad():
            for k, v in named.items():
                v.copy_(gpu_params[step][k])
        _patch_restate(monkeypatch, m, x, fb, ff)
        ropt.zero_grad()
        out = restate.bidirectional_propagation({f"m.{k}": v for k, v in ref.items()}, "m", *xs)
        (out * target.double().cpu()).mean().backward()
        monkeypatch.undo()
        ropt.step()
    for k in named:
        d_gpu = final[k].double().cpu() - p0[k].double().cpu()
        d_ref = ref[k].detach() - p0[k].double().cpu()
        rel = float((d_gpu - d_ref).norm() / d_ref.norm().clamp_min(1e-30))
        assert rel <= 1e-3, (k, rel)
