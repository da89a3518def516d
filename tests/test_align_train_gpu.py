"""H100: the deformable alignment's backward against float64.

* The core (``ops.deform_align_backward``: dA = dY . W16, the sampler's adjoint, dW = dY^T A, the sorted dx gather)
  given head, flows, the fp16 x and W16 and dY, against float64 autograd of the restated DCN epilogue +
  ``oracle.restate.modulated_deform_conv2d``, element by element.  The float64 side reads the same fp16 x and W16 and the
  same raw head, so the only differences are the kernels' fp32 / bf16x3 arithmetic (and fast_tanh / fast_sigmoid, 1e-7
  absolute): the bound of every element is 1e-5 x (its float64 value + the same gradient of the all-positive problem
  |x|, |W|, |dY|) + 1e-6 x the largest value of that gradient; 1e-4 and 1e-5 for d head and d flow, whose bilinear
  slopes move with the kernels' offsets, 1e-6 px from the float64 ones (fast_tanh).  Sample points within 1e-4 of an
  integer coordinate (but not on it) are left out of d offset and d flow, where the floor-based slope changes, and so
  are points on the `inside` boundary (h_im or w_im = -1): the kernel treats such a sample as outside the image.
* Exact-grid data (head 0: tanh' = 1, mask = 1/2; dyadic flows, x, W and dY) give gradients equal to float64.
* The same bits on a second run.
* The module (``SecondOrderDeformableAlignment.forward``) against float64 autograd of ``oracle.restate.deform_align``
  with x and ``weight`` rounded to fp16; its behaviour (bits, second backward, the W16^T cache, Adam steps).  Launch sets: test_gpu_schedules_align.py.
"""
import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.feat_prop import SecondOrderDeformableAlignment
from kernel_checks import check_same_bits
from oracle import restate

pytestmark = pytest.mark.gpu

DG, CIN, COUT = 16, 256, 128


def _epilogue(head, f1, f2, max_res=10.0):
    o1, o2, mask = torch.chunk(head, 3, dim=1)
    offset = max_res * torch.tanh(torch.cat((o1, o2), dim=1))
    off1, off2 = torch.chunk(offset, 2, dim=1)
    off1 = off1 + f1.flip(1).repeat(1, off1.size(1) // 2, 1, 1)
    off2 = off2 + f2.flip(1).repeat(1, off2.size(1) // 2, 1, 1)
    return torch.cat([off1, off2], dim=1), torch.sigmoid(mask)


def _ref_core(x16, head, f1, f2, w16, bias, dy):
    """float64 gradients of restate.modulated_deform_conv2d after the restated epilogue, and the sample coordinates."""
    leaf = [t.detach().double().cpu().requires_grad_() for t in (x16, head, f1, f2, w16, bias)]
    x, hd, a, b, w, bb = leaf
    offset, mask = _epilogue(hd, a, b)
    out = restate.modulated_deform_conv2d(x, offset, mask, w, bb, 1, 1, 1, 1, DG)
    out.backward(dy.detach().double().cpu())
    n, _, h, wd = x.shape
    gy, gx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(wd, dtype=torch.float64), indexing="ij")
    tap = torch.arange(DG * 9) % 9
    hy = gy + (tap // 3 - 1).view(1, -1, 1, 1).double() + offset[:, 0::2].detach()
    wx = gx + (tap % 3 - 1).view(1, -1, 1, 1).double() + offset[:, 1::2].detach()
    return dict(x=x.grad, head=hd.grad, flow_1=a.grad, flow_2=b.grad, weight=w.grad, bias=bb.grad), (hy, wx)


def _unpack(w_packed):
    """fp16 (Cout, 9*Cin) in the sampler's K order -> (Cout, Cin, 3, 3)."""
    return w_packed.view(COUT, DG, 9, CIN // DG).transpose(2, 3).reshape(COUT, CIN, 3, 3)


def _got(x16, head, f1, f2, w_packed, dy, **need):
    dx, dhead, dflow, dw, db = ops.deform_align_backward(x16, head, f1, f2, w_packed, dy, DG, 10.0, **need)
    torch.cuda.synchronize()
    return dict(x=dx, head=dhead, flow_1=dflow[..., 0:2].permute(0, 3, 1, 2), flow_2=dflow[..., 2:4].permute(0, 3, 1, 2),
                weight=dw, bias=db)


def _inputs(n, h, w, flows, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    x16 = torch.randn(n, CIN, h, w, device=dev, generator=g).half().contiguous(memory_format=torch.channels_last)
    head = (0.3 * torch.randn(n, 27 * DG, h, w, device=dev, generator=g)).contiguous(memory_format=torch.channels_last)
    fl = [torch.randn(n, 2, h, w, device=dev, generator=g) * 2 for _ in range(2)]
    if flows == "outside":        # half the flows push samples partly, some wholly, out of the image
        fl[0] = fl[0] + torch.tensor([1.5 * w, -0.6 * h], device=dev).view(1, 2, 1, 1)
        fl[1] = fl[1] * 0 + torch.tensor([-3.0 * w, 0.0], device=dev).view(1, 2, 1, 1)
    elif flows == "integer":      # head 0 on one flow's groups: their sample points lie on integer coordinates
        fl = [f.round() for f in fl]
        head[:, : 72 * 2] = 0
        head[:, 144: 144 + 72 * 2] = 0
    elif flows == "one_point":    # every pixel's flow points at (2, 3): a few very long destination runs
        gy, gx = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        fl = [torch.stack([3 - gx, 2 - gy]).float().expand(n, 2, h, w).contiguous() for _ in range(2)]
        head.zero_()
    weight = torch.randn(COUT, CIN, 3, 3, device=dev, generator=g) / 48
    w_packed = ops.pack_dcn_weight(weight, DG)
    bias = torch.randn(COUT, device=dev, generator=g)
    dy = torch.randn(n, COUT, h, w, device=dev, generator=g)
    return x16, head, fl[0], fl[1], w_packed, bias, dy


def _excluded(hy, wx):
    """(n, 144, h, w): sample points within 1e-4 of an integer coordinate but not on it, and points on the `inside`
    boundary (h_im = -1 or w_im = -1, where the kernel takes the whole sample as outside and gives it no offset
    gradient, while the restatement's corner rule gives x[0]'s row or column a weight of zero and a slope)."""
    h, w = hy.shape[-2:]
    fy, fx = (hy - hy.round()).abs(), (wx - wx.round()).abs()
    near = ((fy > 0) & (fy < 1e-4)) | ((fx > 0) & (fx < 1e-4))
    edge = (hy == -1) | (hy == h) | (wx == -1) | (wx == w)
    return near | edge


def _check_core(got, ref, mag, near, what):
    keep = {k: torch.ones_like(v, dtype=torch.bool) for k, v in ref.items()}
    keep["head"][:, 0:288:2] &= ~near
    keep["head"][:, 1:288:2] &= ~near
    for half, k in ((0, "flow_1"), (1, "flow_2")):
        keep[k] &= ~near[:, 72 * half: 72 * (half + 1)].any(1, keepdim=True)
    for k, r in ref.items():
        gk = got[k].double().cpu()
        rel = 1e-4 if k in ("head", "flow_1", "flow_2") else 1e-5
        bound = rel * (r.abs() + mag[k].abs()) + 0.1 * rel * r.abs().max()
        err = (gk - r).abs()
        bad = (err > bound) & keep[k]
        assert not bad.any(), (what, k, int(bad.sum()), float((err / bound)[keep[k]].max()))


@pytest.mark.parametrize("n,h,w,flows", [
    (1, 60, 108, "random"),      # M = 6480, not a multiple of 128
    (2, 8, 16, "random"),        # M = 256, a multiple of 128
    (3, 5, 7, "random"),
    (2, 7, 9, "outside"),
    (1, 11, 13, "integer"),
    (1, 12, 10, "one_point"),
])
def test_core_against_float64(cuda, n, h, w, flows):
    x16, head, f1, f2, w_packed, bias, dy = _inputs(n, h, w, flows, n * 100 + h, cuda)
    got = _got(x16, head, f1, f2, w_packed, dy)
    w16 = _unpack(w_packed)
    ref, (hy, wx) = _ref_core(x16, head, f1, f2, w16, bias, dy)
    mag, _ = _ref_core(x16.abs(), head, f1, f2, w16.abs(), bias, dy.abs())
    if flows == "outside":
        assert ((hy <= -1) | (hy >= h) | (wx <= -1) | (wx >= w)).any()          # some samples wholly outside
    if flows == "integer":
        assert ((hy == hy.round()) & (wx == wx.round())).any()
    _check_core(got, ref, mag, _excluded(hy, wx), f"{n}x{h}x{w} {flows}")


def test_core_exact_grid(cuda):
    """head = 0 (tanh' = 1, mask = 1/2 exactly), flows on a 1/4 grid, x on a 1/8 grid, W on a 1/64 grid and dY on a 1/8
    grid: every product and sum is exact in fp32, so every gradient equals float64."""
    n, h, w = 2, 9, 11
    g = torch.Generator(device=cuda).manual_seed(7)
    x16 = (torch.randint(-8, 9, (n, CIN, h, w), device=cuda, generator=g) / 8).half().contiguous(
        memory_format=torch.channels_last)
    head = torch.zeros(n, 27 * DG, h, w, device=cuda).contiguous(memory_format=torch.channels_last)
    f1, f2 = [torch.randint(-12, 13, (n, 2, h, w), device=cuda, generator=g) / 4 for _ in range(2)]
    weight = torch.randint(-4, 5, (COUT, CIN, 3, 3), device=cuda, generator=g) / 64
    w_packed = ops.pack_dcn_weight(weight, DG)
    dy = torch.randint(-2, 3, (n, COUT, h, w), device=cuda, generator=g) / 8
    got = _got(x16, head, f1, f2, w_packed, dy)
    ref, (hy, wx) = _ref_core(x16, head, f1, f2, _unpack(w_packed), torch.zeros(COUT), dy)
    edge = _excluded(hy, wx)
    assert edge.any() and not edge.all()
    keep = {k: torch.ones_like(v, dtype=torch.bool) for k, v in ref.items()}
    keep["head"][:, 0:288:2] &= ~edge
    keep["head"][:, 1:288:2] &= ~edge
    keep["flow_1"] &= ~edge[:, :72].any(1, keepdim=True)
    keep["flow_2"] &= ~edge[:, 72:].any(1, keepdim=True)
    for k, r in ref.items():
        gk = got[k].double().cpu()
        assert torch.equal(gk[keep[k]], r[keep[k]]), (k, float((gk - r)[keep[k]].abs().max()))


def test_core_same_bits(cuda):
    x16, head, f1, f2, w_packed, bias, dy = _inputs(2, 30, 54, "random", 5, cuda)
    a = _got(x16, head, f1, f2, w_packed, dy)
    b = _got(x16, head, f1, f2, w_packed, dy)
    for k in a:
        check_same_bits(a[k], b[k], k)


# ------------------------------------------------------------------------------------------------------------ module
def _module(dev, seed, random_last):
    torch.manual_seed(seed)
    m = SecondOrderDeformableAlignment(2 * COUT, COUT, 3, padding=1, deform_groups=DG)
    if random_last:
        torch.nn.init.normal_(m.conv_offset[-1].weight, std=0.01)
        torch.nn.init.normal_(m.conv_offset[-1].bias, std=0.1)
    return m.to(dev)


def _module_inputs(n, h, w, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(n, 2 * COUT, h, w, device=dev, generator=g)
    extra = torch.randn(n, 3 * COUT, h, w, device=dev, generator=g)
    f1, f2 = [torch.randn(n, 2, h, w, device=dev, generator=g) * 3 for _ in range(2)]
    return x, extra, f1, f2


class _GpuDecisions:
    """``torch.nn.functional`` for the restatement with LeakyReLU's decisions taken from the GPU forward: the offset
    head's three activations, in call order (the accuracy convention: the gradients are those of the function the
    GPU evaluated, and a pre-activation within rounding of 0 may fall on either side)."""

    def __init__(self, masks):
        self.masks, self.i = masks, 0

    def __getattr__(self, name):
        return getattr(F, name)

    def leaky_relu(self, v, slope):
        mask = self.masks[self.i % len(self.masks)]
        self.i += 1
        return torch.where(mask, v, slope * v)


def _gpu_decisions(m, x, extra, f1, f2):
    keep = {}
    with torch.no_grad():
        m._forward_keep(x, extra, f1, f2, keep)
    return _GpuDecisions([(a > 0).cpu() for a in keep["acts"][1:]])


def _ref_module(m, x, extra, f1, f2, dy):
    sd = {f"m.{k}": v.detach().double().cpu().requires_grad_() for k, v in m.state_dict().items()}
    w16 = sd["m.weight"]
    use = dict(sd)
    use["m.weight"] = w16 + (w16.detach().half().double() - w16.detach())      # the kernel reads fp16 W
    leaves = [t.detach().double().cpu().requires_grad_() for t in (x, extra, f1, f2)]
    xr = leaves[0] + (leaves[0].detach().half().double() - leaves[0].detach())  # and fp16 x
    restate.F = _gpu_decisions(m, x, extra, f1, f2)
    try:
        out = restate.deform_align(use, "m", xr, leaves[1], leaves[2], leaves[3])
    finally:
        restate.F = F
    out.backward(dy.double().cpu())
    return out.detach(), [t.grad for t in leaves], {k[2:]: v.grad for k, v in sd.items()}


@pytest.mark.parametrize("random_last", [False, True])
def test_module_against_float64(cuda, random_last):
    m = _module(cuda, 3, random_last)
    x, extra, f1, f2 = _module_inputs(2, 12, 20, cuda, 4)
    leaves = [t.clone().requires_grad_() for t in (x, extra, f1, f2)]
    out = m(*leaves)
    assert out.grad_fn is not None
    dy = torch.randn(out.shape, device=cuda, generator=torch.Generator(device=cuda).manual_seed(9))
    out.backward(dy)
    ref_out, ref_in, ref_p = _ref_module(m, x, extra, f1, f2, dy)
    pairs = [(f"input {i}", t.grad, r) for i, (t, r) in enumerate(zip(leaves, ref_in))]
    pairs += [(k, p.grad, ref_p[k]) for k, p in m.named_parameters()]
    for what, gk, r in pairs:
        gk = gk.double().cpu()
        scale = float(r.abs().max())
        if scale == 0:
            assert float(gk.abs().max()) == 0, what
            continue
        err = (gk - r).abs()
        assert float(err.max()) <= 1e-3 * scale, (what, float(err.max()), scale)


def test_tracked_output_same_bits_and_second_backward(cuda):
    m = _module(cuda, 5, True)
    x, extra, f1, f2 = _module_inputs(1, 10, 14, cuda, 6)
    with torch.no_grad():
        want = m(x, extra, f1, f2)
    out = m(x, extra, f1, f2)
    assert out.grad_fn is not None
    check_same_bits(out, want, "tracked output")
    out.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second time"):
        out.sum().backward()
    out = m(x, extra, f1, f2)
    with torch.no_grad():
        m.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.sum().backward()


def test_transposed_weight_cache_follows_updates(cuda):
    m = _module(cuda, 8, True)
    a = m.transposed_weight()
    assert m.transposed_weight() is a
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    x, extra, f1, f2 = _module_inputs(1, 6, 8, cuda, 2)
    m(x, extra, f1, f2).sum().backward()
    opt.step()
    b = m.transposed_weight()
    assert b is not a
    check_same_bits(b[0], ops.dcn_transposed_split(m.weight, DG)[0], "rebuilt after optimizer.step()")
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    sd["weight"] = sd["weight"] * 2
    m.load_state_dict(sd)
    ops.invalidate_weight_caches()
    check_same_bits(m.transposed_weight()[1], ops.dcn_transposed_split(m.weight, DG)[1], "after load_state_dict")


def test_adam_steps_track_float64(cuda, monkeypatch):
    """Three Adam steps on a linear loss (the inner product with a fixed random tensor) next to the same steps in float64
    autograd of the restatement (x and ``weight`` read through fp16): every parameter's total update is within 1e-3
    (L2, relative).  The loss's output gradient is the fixed tensor on both sides, so the forward's fp16 GEMM operands,
    which the float64 side does not round, do not enter the steps.  Each parameter's Adam eps is 10x its largest first
    gradient (as in test_block_train_gpu.py), so that the steps do not turn the sign of near-zero gradient elements into
    full-size updates.  Each float64 step takes LeakyReLU's decisions from the GPU forward at that step's parameters."""
    m = _module(cuda, 13, True)
    x, extra, f1, f2 = _module_inputs(1, 10, 12, cuda, 14)
    target = torch.randn(1, COUT, 10, 12, device=cuda)
    named = dict(m.named_parameters())
    p0 = {k: v.detach().clone() for k, v in named.items()}
    (m(x, extra, f1, f2) * target).mean().backward()
    eps = {k: 10 * float(v.grad.abs().max()) for k, v in named.items()}
    m.zero_grad()
    opt = torch.optim.Adam([{"params": [named[k]], "eps": eps[k]} for k in named], lr=1e-3)
    gpu_params = []
    for _ in range(3):
        gpu_params.append({k: v.detach().clone() for k, v in named.items()})
        opt.zero_grad()
        (m(x, extra, f1, f2) * target).mean().backward()
        opt.step()
    final = {k: v.detach().clone() for k, v in named.items()}
    ref = {k: v.detach().double().cpu().clone().requires_grad_() for k, v in p0.items()}
    ropt = torch.optim.Adam([{"params": [ref[k]], "eps": eps[k]} for k in named], lr=1e-3)
    xs = [t.double().cpu() for t in (x, extra, f1, f2)]
    for step in range(3):
        with torch.no_grad():
            for k, v in named.items():
                v.copy_(gpu_params[step][k])
        monkeypatch.setattr(restate, "F", _gpu_decisions(m, x, extra, f1, f2))
        ropt.zero_grad()
        sd = {f"m.{k}": v for k, v in ref.items()}
        w = sd["m.weight"]
        sd["m.weight"] = w + (w.detach().half().double() - w.detach())
        out = restate.deform_align(sd, "m", xs[0].half().double(), *xs[1:])
        (out * target.double().cpu()).mean().backward()
        ropt.step()
    for k in named:
        d_gpu = final[k].double().cpu() - p0[k].double().cpu()
        d_ref = ref[k].detach() - p0[k].double().cpu()
        rel = float((d_gpu - d_ref).norm() / d_ref.norm().clamp_min(1e-30))
        assert rel <= 1e-3, (k, rel)