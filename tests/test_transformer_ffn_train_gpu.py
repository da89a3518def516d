"""H100: the transformer's token path in training — the Linear weight gradient (``e2f_linear_wgrad_bf16x3``), the
fold/normalise/unfold + GELU adjoint of ``e2f_t2t_fold_unfold_train`` and the differentiable SoftSplit, SoftComp and
FusionFeedForward — against float64 torch, element by element.

Bounds (kernel_checks): C * A for the bf16 three-term split, A the same operation on absolute values.  Weight
gradients add the fixed-order accumulation term U * (12 kb + slices) * A (kb = 64-token blocks per slice, three split
terms and four k16 steps each) and the bias gradient U * (2 * 64 kb + slices) * A (tokens summed one by one, hi + lo).
A module's gradient passes through up to three such stages, each within C * A of its own input's A, so the module
checks hold each result to 3 C A, A restated on absolute values along the whole chain (|GELU'(u)| for GELU')."""
import math

import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.tfocal_transformer import FusionFeedForward, SoftComp, SoftSplit
from kernel_checks import (assert_exact_grid, cdiv, check_close, check_exact, check_same_bits, grid_values, int_values,
                           reference_math)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T2T = dict(kernel_size=(7, 7), stride=(3, 3), padding=(3, 3))


def _slices(m, n, k):
    """linear_wgrad_slices (linear_wgrad.cu)."""
    s = cdiv(264, cdiv(n, 128) * cdiv(k, 128))
    return max(1, min(s, m // 256, 64))


def _wgrad_extra(m, n, k):
    sl = _slices(m, n, k)
    kb = cdiv(cdiv(m, sl), 64)
    return U * (12 * kb + sl), U * (128 * kb + sl)


def _check_wgrad(dw, db, dy, x, what, n=None, k=None):
    dy64, x64 = dy.double(), x.double()
    n = n or dy.shape[1]
    k = k or x.shape[1]
    dy64, x64 = dy64[:, :n], x64[:, :k]
    ref_w, ref_b = dy64.t() @ x64, dy64.sum(0)
    bw, bb = dy64.abs().t() @ x64.abs(), dy64.abs().sum(0)
    ew, eb = _wgrad_extra(dy.shape[0], n, k)
    check_close(dw, ref_w, bw, 1e-4, "f32", what + " dW", extra=ew * bw)
    check_close(db, ref_b, bb, 1e-4, "f32", what + " db", extra=eb * bb)


# (m, n, k, ldy, ldx): tiny; m not a multiple of 64; several slices with several items per CTA; the four layers
WGRAD = [(40, 24, 16, 24, 16), (1000, 200, 136, 200, 136), (5000, 512, 1960, 512, 1984), (4600, 1960, 512, 1984, 512),
         (3000, 512, 6272, 512, 6272), (3000, 6272, 512, 6272, 512), (20000, 256, 384, 256, 384)]


@pytest.mark.parametrize("m,n,k,ldy,ldx", WGRAD)
def test_linear_wgrad_against_float64(cuda, m, n, k, ldy, ldx):
    g = torch.Generator(device=cuda).manual_seed(m + n + k)
    dy = torch.randn(m, ldy, device=cuda, generator=g)
    x = torch.randn(m, ldx, device=cuda, generator=g)
    dy[:, n:] = 0
    x[:, k:] = 0
    dys, xs = ops.SplitMat(*ops.split_bf16(dy)), ops.SplitMat(*ops.split_bf16(x))
    dw, db = ops.linear_wgrad(dys, xs, shape=(n, k))
    _check_wgrad(dw, db, dy, x, f"linear_wgrad {m}x{n}x{k}", n, k)
    again = ops.linear_wgrad(dys, xs, shape=(n, k))
    check_same_bits((dw, db), again, "linear_wgrad run to run")
    dw2, db2 = ops.linear_wgrad(dys, xs, with_bias=False, shape=(n, k))
    assert db2 is None
    check_same_bits(dw2, dw, "linear_wgrad without the bias")


@pytest.mark.parametrize("m,n,k", [(777, 200, 136), (4600, 512, 1960)])
def test_linear_wgrad_exact_grid(cuda, m, n, k):
    g = torch.Generator(device=cuda).manual_seed(n)
    dy = int_values((m, n), g, m=2, density=0.3)
    x = grid_values((m, k), g, density=0.05, fine=True)
    dw, db = ops.linear_wgrad(dy, x)
    ref_w = dy.double().t() @ x.double()
    assert_exact_grid(dy.double().abs().t() @ x.double().abs(), x, "linear_wgrad")
    check_exact(dw, ref_w, "linear_wgrad exact dW")
    check_exact(db, dy.double().sum(0), "linear_wgrad exact db")


def _ffn_mid64(h, output_size):
    """u = unfold(fold(h) / fold(ones)), z = GELU(u) in float64 (tfocal_transformer.py:89-96)."""
    bt, n, ck = h.shape
    fold = F.fold(h.transpose(1, 2), output_size, **T2T)
    ones = F.fold(torch.ones_like(h).transpose(1, 2), output_size, **T2T)
    u = F.unfold(fold / ones, **T2T).transpose(1, 2)
    return u


def _dgelu(u):
    return 0.5 * (1 + torch.erf(u / math.sqrt(2))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)


@pytest.mark.parametrize("bt,h,w,c", [(2, 60, 108, 40), (1, 90, 162, 8), (1, 20, 36, 40)])
def test_fold_unfold_adjoint_against_float64(cuda, bt, h, w, c):
    """Training forward: the same bits as the inference kernel and u; adjoint: float64 autograd of F.fold / F.unfold /
    F.gelu (90 x 162 is wider than one x tile of the tiled kernel, 60 x 108 and 20 x 36 run the full-width one)."""
    g = torch.Generator(device=cuda).manual_seed(h + c)
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    ck = c * 49
    pitch = (ck + 63) // 64 * 64
    tok = torch.randn(bt, fh * fw, ck, device=cuda, generator=g)
    want = ops.t2t_fold_unfold(tok, (h, w), **T2T, gelu=True, out="split", pitch=pitch)
    z, u = ops.t2t_fold_unfold_train(tok, (h, w), **T2T, out="split", pitch=pitch)
    check_same_bits((z.hi, z.lo), (want.hi, want.lo), "training forward vs inference")
    with reference_math():
        t64 = tok.double().requires_grad_()
        u64 = _ffn_mid64(t64, (h, w))
        dz = torch.randn(bt, fh * fw, ck, device=cuda, generator=g)
        F.gelu(u64).backward(dz.double())
        ua = _ffn_mid64(dz.double().abs() * _dgelu(u64.detach()).abs(), (h, w))
    check_close(u, u64.detach(), _ffn_mid64(tok.double().abs(), (h, w)), 1e-5, "f32", "fold_unfold u")
    dh = ops.t2t_fold_unfold_train(dz, (h, w), **T2T, u=u, out="split", pitch=pitch)
    got = dh.hi.float()[..., :ck] + dh.lo.float()[..., :ck]
    assert torch.all(dh.hi[..., ck:] == 0) and torch.all(dh.lo[..., ck:] == 0)
    # GELU'(u) = Phi(u) + u phi(u) in fp32 (erff, __expf, the kernel's u) is off by a few 2^-24 absolute, not relative:
    # near its zero (u ~ -0.75) the two terms cancel, so the allowance is 2^-20 |dz| (1 + |u|) through U D F
    ex = _ffn_mid64(dz.double().abs() * (1 + u64.detach().abs()), (h, w))
    check_close(got, t64.grad, ua, 1e-4, "split", "fold_unfold adjoint", extra=2.0 ** -20 * ex)
    again = ops.t2t_fold_unfold_train(dz, (h, w), **T2T, u=u, out="split", pitch=pitch)
    check_same_bits((dh.hi, dh.lo), (again.hi, again.lo), "adjoint run to run")


# ------------------------------------------------------------------------------------------------ modules
def _t2t(size):
    return dict(T2T, output_size=size)


def _modules(cuda, hq, size, seed):
    torch.manual_seed(seed)
    ss = SoftSplit(128, 512, **T2T).to(cuda)
    sc = SoftComp(128, 512, None if hq else size, hq=hq).to(cuda)
    ffn = FusionFeedForward(512, t2t_params=_t2t(size)).to(cuda)
    with torch.no_grad():
        if not hq:
            sc.bias.normal_(0, 0.1)
        for lin in (ss.embedding, sc.embedding, ffn.conv1[0], ffn.conv2[1]):
            lin.bias.normal_(0, 0.1)
    return ss, sc, ffn


def _step64(p, feat, b, size, hq):
    """sc(ffn(ss(feat)), residual=feat) in float64 on the restated operations; p: float64 parameters by name."""
    bt, c, h, w = feat.shape
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    tok = F.linear(F.unfold(feat, **T2T).transpose(1, 2), p["ss.w"], p["ss.b"])            # (bt, L, 512)
    x = tok.reshape(b, -1, 512)
    hmid = F.linear(x, p["ffn.w1"], p["ffn.b1"]).reshape(bt, fh * fw, -1)
    zz = F.gelu(_ffn_mid64(hmid, size)).reshape(b, -1, hmid.shape[-1])
    y = F.linear(zz, p["ffn.w2"], p["ffn.b2"]) + x
    cols = F.linear(y.reshape(bt, fh * fw, 512), p["sc.w"], p["sc.b"])
    img = F.fold(cols.transpose(1, 2), size, **T2T)
    if hq:
        return F.conv2d(img, p["sc.bcw"], p["sc.bcb"], padding=1) + feat
    return img + p["sc.bias"] + feat


def _names(ss, sc, ffn, hq):
    named = {"ss.w": ss.embedding.weight, "ss.b": ss.embedding.bias, "sc.w": sc.embedding.weight,
             "sc.b": sc.embedding.bias, "ffn.w1": ffn.conv1[0].weight, "ffn.b1": ffn.conv1[0].bias,
             "ffn.w2": ffn.conv2[1].weight, "ffn.b2": ffn.conv2[1].bias}
    if hq:
        named.update({"sc.bcw": sc.bias_conv.weight, "sc.bcb": sc.bias_conv.bias})
    else:
        named["sc.bias"] = sc.bias
    return named


def _run(ss, sc, ffn, feat, b, size, hq):
    t = feat.shape[0] // b
    tok = ss(feat, b, size)
    y = ffn(tok.reshape(b, -1, 512), size, residual=tok.reshape(b, -1, 512))
    return sc(y.reshape(tok.shape), t, size, residual=feat)


@pytest.mark.parametrize("hq,b,t,h,w", [(False, 1, 2, 60, 108), (True, 1, 2, 36, 84)])
def test_modules_against_float64(cuda, hq, b, t, h, w):
    """Every parameter, the features (through SoftSplit and as SoftComp's residual) against float64 autograd of the
    restatement; the tracked forward is the same bits as the untracked one."""
    size = (h, w)
    ss, sc, ffn = _modules(cuda, hq, size, 7)
    g = torch.Generator(device=cuda).manual_seed(11)
    feat = torch.randn(b * t, 128, h, w, device=cuda, generator=g).contiguous(memory_format=torch.channels_last)
    dout = torch.randn(b * t, 128, h, w, device=cuda, generator=g)
    with torch.no_grad():
        want = _run(ss, sc, ffn, feat, b, size, hq)
    x = feat.clone().requires_grad_()
    out = _run(ss, sc, ffn, x, b, size, hq)
    assert out.grad_fn is not None
    check_same_bits(out.contiguous(), want.contiguous(), "tracked forward")
    out.backward(dout)
    named = _names(ss, sc, ffn, hq)
    with reference_math():
        p64 = {k: v.detach().double().requires_grad_() for k, v in named.items()}
        x64 = feat.double().requires_grad_()
        _step64(p64, x64, b, size, hq).backward(dout.double())
        # A: the same chain on absolute values (a float64 restatement with |parameters|, |features|, |GELU'|)
        pa = {k: v.detach().double().abs().requires_grad_() for k, v in named.items()}
        xa = feat.double().abs().requires_grad_()
        _step64_abs(pa, xa, b, size, hq).backward(dout.double().abs())
    for k, v in named.items():
        check_close(v.grad, p64[k].grad, 3 * pa[k].grad, 1e-3, "f32", f"{'hq' if hq else 'base'} {k}")
    check_close(x.grad, x64.grad, 3 * xa.grad, 1e-3, "f32", f"{'hq' if hq else 'base'} features")


def _step64_abs(p, feat, b, size, hq):
    """``_step64`` on absolute values with GELU replaced by a function whose derivative is |GELU'| and every bias
    dropped from the forward values (they enter A only through their own gradients)."""
    class AbsGelu(torch.autograd.Function):
        @staticmethod
        def forward(ctx, u):
            ctx.save_for_backward(u)
            return u
        @staticmethod
        def backward(ctx, gr):
            (u,) = ctx.saved_tensors
            return gr * _dgelu(u).abs()
    bt, c, h, w = feat.shape
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    tok = F.linear(F.unfold(feat, **T2T).transpose(1, 2), p["ss.w"], p["ss.b"])
    x = tok.reshape(b, -1, 512)
    hmid = F.linear(x, p["ffn.w1"], p["ffn.b1"]).reshape(bt, fh * fw, -1)
    zz = AbsGelu.apply(_ffn_mid64(hmid, size)).reshape(b, -1, hmid.shape[-1])
    y = F.linear(zz, p["ffn.w2"], p["ffn.b2"]) + x
    cols = F.linear(y.reshape(bt, fh * fw, 512), p["sc.w"], p["sc.b"])
    img = F.fold(cols.transpose(1, 2), size, **T2T)
    if hq:
        return F.conv2d(img, p["sc.bcw"], p["sc.bcb"], padding=1) + feat
    return img + p["sc.bias"] + feat


def _launched(fn):
    """Names of the library launches (``ops._timed`` records) of fn()."""
    rec = ops.profile_kernels(True)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        ops.profile_kernels(False)
    return set(rec)


def test_frozen_parts_launch_nothing_and_second_backward_raises(cuda):
    """A frozen Linear launches no weight-gradient kernel and an input that needs no gradient no input-gradient
    kernel; each module's second backward raises."""
    size = (60, 108)
    ss, sc, ffn = _modules(cuda, False, size, 3)
    g = torch.Generator(device=cuda).manual_seed(5)
    x = torch.randn(1, 720, 512, device=cuda, generator=g)
    for p_ in ffn.parameters():
        p_.requires_grad_(False)
    ffn.conv2[1].weight.requires_grad_(True)
    out = ffn(x, size)
    assert _launched(lambda: out.sum().backward()) == {"linear_wgrad_bf16x3"}     # no adjoint, no input gradient
    assert ffn.conv2[1].weight.grad is not None and ffn.conv1[0].weight.grad is None
    out = ffn(x.clone().requires_grad_(), size)
    out.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="backpropagated a second time"):
        out.sum().backward()
    for p_ in ss.parameters():
        p_.requires_grad_(False)
    feat = torch.randn(1, 128, 60, 108, device=cuda, generator=g, requires_grad=True)
    tok = ss(feat, 1, size)
    got = _launched(lambda: tok.sum().backward())
    assert "linear_wgrad_bf16x3" not in got and "t2t_unfold" not in got and "conv3x3_bf16x3" in got, sorted(got)
    for p_ in sc.parameters():
        p_.requires_grad_(False)
    out = sc(torch.randn(1, 1, 20, 36, 512, device=cuda, generator=g, requires_grad=True), 1, size)
    got = _launched(lambda: out.sum().backward(retain_graph=True))
    assert "linear_wgrad_bf16x3" not in got and "t2t_unfold" not in got and "conv3x3_bf16x3" in got, sorted(got)
    with pytest.raises(RuntimeError, match="backpropagated a second time"):
        out.sum().backward()
    sc.embedding.weight.requires_grad_(True)
    out = sc(torch.randn(1, 1, 20, 36, 512, device=cuda, generator=g), 1, size)
    assert _launched(lambda: out.sum().backward()) == {"t2t_unfold", "linear_wgrad_bf16x3"}


def test_adam_steps_track_float64(cuda):
    """Four Adam steps of sc(ffn(ss(feat))) on the mean squared error against a target, next to the same steps on the
    float64 restatement: each parameter's total update is within 1e-3 (L2, relative) of the float64 one.  Each
    parameter's eps is ten times its largest first-step gradient: Adam's step is then close to linear in the gradient,
    instead of lr * sign for gradient elements near zero, whose GPU and float64 values may differ in sign within the
    gradients' tolerance (test_encdec_train_gpu.py sets eps above the gradients' scale for the same reason).  The loss
    is smooth: with L1, an output within rounding of its target takes the other sign of the derivative, and one such
    pixel alone moves the bias map's update by 3e-3."""
    size = (30, 54)
    b, t = 1, 2
    ss, sc, ffn = _modules(cuda, False, size, 9)
    named = _names(ss, sc, ffn, False)
    start = {k: v.detach().double().clone() for k, v in named.items()}
    p64 = {k: v.clone().requires_grad_() for k, v in start.items()}
    g = torch.Generator(device=cuda).manual_seed(2)
    feat = torch.randn(b * t, 128, *size, device=cuda, generator=g)
    target = torch.randn(b * t, 128, *size, device=cuda, generator=g)

    def loss64():
        with reference_math():
            (_step64(p64, feat.double(), b, size, False) - target.double()).pow(2).mean().backward()

    loss64()
    eps = {k: 10 * p64[k].grad.abs().max().item() for k in named}
    opt = torch.optim.Adam([{"params": [named[k]], "eps": eps[k]} for k in named], lr=1e-3)
    opt64 = torch.optim.Adam([{"params": [p64[k]], "eps": eps[k]} for k in named], lr=1e-3)
    for _ in range(4):
        opt.zero_grad()
        (_run(ss, sc, ffn, feat, b, size, False) - target).pow(2).mean().backward()
        opt.step()
        opt64.zero_grad()
        loss64()
        opt64.step()
    for k, v in named.items():
        ours, ref = v.detach().double() - start[k], p64[k].detach() - start[k]
        assert (ours - ref).norm() <= 1e-3 * ref.norm(), (k, ((ours - ref).norm() / ref.norm()).item())
