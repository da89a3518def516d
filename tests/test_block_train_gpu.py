"""H100: the temporal focal transformer blocks in training — the LayerNorm backward (``e2f_layernorm_backward``), the
LayerNorm + focal pooling backward (``e2f_layernorm_pool_backward``) and the differentiable
``TemporalFocalTransformerBlock`` — against float64 torch, element by element.

Bounds.
* The LayerNorm kernels (fp32 arithmetic, ``check_bounded``), per row with U = 2^-24, x^ and g = gamma * dy in float64:
  the mean has at most 21 U mean|x| of error (16 sequential adds per lane, then five butterfly levels) and rstd 16 U
  relative (the variance sum likewise, rsqrtf 2 ulp), so x^ is off by at most e = 24 U (|x^| + rstd mean|x|).
  mean(g) is off by 21 U mean|g|, mean(g x^) by 22 U mean|g x^| + mean(|g| e), and the last line rounds 3 times:
    |dx - ref| <= 2 [rstd (21 U mean|g| + |x^| (22 U mean|g x^| + mean(|g| e)) + |mean(g x^)| e) + 3 U rstd S + 16 U |ref|]
  with S = |g| + mean|g| + |x^| mean|g x^| (+ U |residual|).  dgamma and dbeta add one term per row, each off by
  |dy| e (+ U of its size), in at most 8 (per lane) + 8 (warps) + P / 8 + 8 (the fixed-order column sum over P partial
  rows) = n additions: |err| <= 2 (sum |dy| e + (n + 2) U sum |dy x^|).  The pooling backward alike, with
  dy = dxn + w dpooled (one more rounding) and d w_pool = sum dpooled LN(x) (LN(x) off by |gamma| e + 2 U |LN(x)|,
  21 more additions in the warp sum).  Split outputs add the 2^-16 rounding of the pair.
* The block (``check_close``, C = 2^-14): 6 C A.  A is the last product of each gradient on absolute values at the
  float64 intermediate gradients, as in test_attention_train_gpu.py: |dY|^T |X| and sum |dY| for each Linear, sum |dy|
  |x^| and sum |dy| for each LayerNorm, sum |dpooled| |LN(x)| for the pooling weight, and for x the LayerNorms' input
  gradients restated on absolute values (rstd (|gamma| a + mean(|gamma| a) + |x^| mean(|gamma| a |x^|)), a = the
  absolute product that feeds them).  Each gradient passes through at most two bf16x3 stages after the attention core
  (3 C A each in the neighbouring files, and their errors add); 6 covers both.  The attention is evaluated at the fp16
  qkv the kernels compute, with the gradient passed straight through that rounding, as the backward does.
* The trunk of eight blocks: the same A per block; a block's incoming gradient carries the errors of the blocks above it,
  which add along the residual stream, so the bound is 8 x 6 C A."""
import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.tfocal_transformer import SoftComp, SoftSplit, TemporalFocalTransformerBlock
from kernel_checks import check_bounded, check_close, check_same_bits, reference_math
from oracle import restate

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T2T = dict(kernel_size=(7, 7), stride=(3, 3), padding=(3, 3))


# ---------------------------------------------------------------------------------------------------- kernel bounds
def _ln64(x, eps=1e-5):
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    rstd = ((x - mu) ** 2).mean(-1, keepdim=True).add(eps).rsqrt()
    return (x - mu) * rstd, rstd, x.abs().mean(-1, keepdim=True)


def _ln_bound(xh, rstd, xabs, g):
    """The per-element bound of the LayerNorm input gradient (module docstring) at x^, rstd, mean|x| and g."""
    e = 24 * U * (xh.abs() + rstd * xabs)
    ga = g.abs()
    m2 = (g * xh).mean(-1, keepdim=True)
    s = ga + ga.mean(-1, keepdim=True) + xh.abs() * (ga * xh.abs()).mean(-1, keepdim=True)
    core = rstd * (21 * U * ga.mean(-1, keepdim=True) + xh.abs() * (22 * U * (ga * xh.abs()).mean(-1, keepdim=True)
                                                                    + (ga * e).mean(-1, keepdim=True)) + m2.abs() * e)
    return 2 * (core + 3 * U * rstd * s), e


def _ln_backward64(x, dy, gamma, res=None):
    xh, rstd, xabs = _ln64(x)
    g = dy.double() * gamma.double()
    dx = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    bound, e = _ln_bound(xh, rstd, xabs, g)
    if res is not None:
        dx = dx + res.double()
        bound = bound + U * res.double().abs()
    return dx, bound + 32 * U * dx.abs(), xh, e


@pytest.mark.parametrize("rows", [1, 3, 64 * 5 + 17, 46080])
def test_layernorm_backward_against_float64(cuda, rows):
    g_ = torch.Generator(device=cuda).manual_seed(rows)
    x = torch.randn(rows, 512, device=cuda, generator=g_) * 2 + 0.5
    dy = torch.randn(rows, 512, device=cuda, generator=g_)
    gamma = 1 + 0.2 * torch.randn(512, device=cuda, generator=g_)
    res = torch.randn(rows, 512, device=cuda, generator=g_)
    parts = (rows + 63) // 64
    n_add = 8 + 8 + parts // 8 + 8
    for with_res in (False, True):
        r = res if with_res else None
        (dx32, dxs), dg, db = ops.layer_norm_backward(x, dy, gamma, residual=r, out="both")
        (dx32b, dxsb), dgb, dbb = ops.layer_norm_backward(x, dy, gamma, residual=r, out="both")
        for a, b_, what in ((dx32, dx32b, "dx"), (dxs.hi, dxsb.hi, "hi"), (dxs.lo, dxsb.lo, "lo"), (dg, dgb, "dgamma"),
                            (db, dbb, "dbeta")):
            check_same_bits(a, b_, f"layernorm backward {rows} {what} repeat")
        ref, bound, xh, e = _ln_backward64(x, dy, gamma, r)
        case = f"layernorm backward rows={rows} res={with_res}"
        check_bounded(dx32.cpu(), ref.cpu(), bound.cpu(), case + " dx")
        check_bounded((dxs.hi.double() + dxs.lo.double()).cpu(), ref.cpu(), bound.cpu(), case + " split", 2.0 ** -16)
        dyd = dy.double()
        check_bounded(dg.cpu(), (dyd * xh).sum(0).cpu(),
                      (2 * ((dyd.abs() * e).sum(0) + (n_add + 2) * U * (dyd * xh).abs().sum(0))).cpu(), case + " dgamma")
        check_bounded(db.cpu(), dyd.sum(0).cpu(), (2 * (n_add + 2) * U * dyd.abs().sum(0)).cpu(), case + " dbeta")
    # the split alone, and the fp32 output alone without partial sums: the same bits as with them
    dxs_only, none_g, none_b = ops.layer_norm_backward(x, dy, gamma, out="split", need_weight=False, need_bias=False)
    assert none_g is None and none_b is None
    (dx_ref, dxs_ref), _, _ = ops.layer_norm_backward(x, dy, gamma, out="both")
    check_same_bits(dxs_only.hi, dxs_ref.hi, "split only")
    before = ops.launch_count()
    ops.layer_norm_backward(x, dy, gamma, need_weight=False, need_bias=False)
    torch.cuda.synchronize()
    assert ops.launch_count() - before == 1                      # no partial rows, no column sum


@pytest.mark.parametrize("B,T,H,W", [(1, 1, 20, 36), (2, 8, 20, 36), (1, 1, 5, 9), (3, 2, 5, 9), (1, 8, 40, 72),
                                     (2, 1, 40, 72)])
def test_layernorm_pool_backward_against_float64(cuda, B, T, H, W):
    g_ = torch.Generator(device=cuda).manual_seed(B * 1000 + T * 100 + H)
    C, nW = 512, (H // 5) * (W // 9)
    x = torch.randn(B, T, H, W, C, device=cuda, generator=g_) * 2 + 0.5
    n_tok, n_pool = B * T * H * W, B * T * nW
    drows = torch.randn(n_tok + n_pool, C, device=cuda, generator=g_)
    dx1 = torch.randn(B, T, H, W, C, device=cuda, generator=g_)
    gamma = 1 + 0.2 * torch.randn(C, device=cuda, generator=g_)
    beta = 0.2 * torch.randn(C, device=cuda, generator=g_)
    pw = torch.randn(1, 45, device=cuda, generator=g_) / 45
    got = ops.layer_norm_pool_backward(x, drows, dx1, gamma, beta, 1e-5, pw, (5, 9))
    again = ops.layer_norm_pool_backward(x, drows, dx1, gamma, beta, 1e-5, pw, (5, 9))
    for a, b_, what in zip(got, again, ("dx", "dgamma", "dbeta", "dpool_w", "dpool_b")):
        check_same_bits(a, b_, f"pool backward {what} repeat")
    dx, dg, db, dpw, dpb = got
    # float64: dy = dxn + w[token] dpooled[window], per token of each window
    dp = drows[n_tok:].double().view(B, T, H // 5, 1, W // 9, 1, C)
    w64 = pw.double().view(1, 1, 1, 5, 1, 9, 1)
    dxn = drows[:n_tok].double().view(B, T, H // 5, 5, W // 9, 9, C)
    dy = (dxn + w64 * dp).view(B, T, H, W, C)
    xh, rstd, xabs = _ln64(x)
    g = dy * gamma.double()
    ref = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True)) + dx1.double()
    bound, e = _ln_bound(xh, rstd, xabs, g)
    bound = bound + 2 * U * rstd * gamma.double().abs() * dy.abs() + U * dx1.double().abs() + 32 * U * ref.abs()
    case = f"pool backward {B}x{T}x{H}x{W}"
    check_bounded(dx.cpu(), ref.cpu(), bound.cpu(), case + " dx")
    n_add = 8 + 8 + (B * T * nW) // 8 + 8
    check_bounded(dg.cpu(), (dy * xh).sum((0, 1, 2, 3)).cpu(),
                  (2 * ((dy.abs() * (e + U * xh.abs())).sum((0, 1, 2, 3))
                        + (n_add + 2) * U * (dy * xh).abs().sum((0, 1, 2, 3)))).cpu(), case + " dgamma")
    check_bounded(db.cpu(), dy.sum((0, 1, 2, 3)).cpu(), (2 * (n_add + 2) * U * dy.abs().sum((0, 1, 2, 3))).cpu(),
                  case + " dbeta")
    xn = (xh * gamma.double() + beta.double()).view(B, T, H // 5, 5, W // 9, 9, C)
    xn_err = gamma.double().abs() * e.view(xn.shape) + 2 * U * xn.abs()
    dpv = dp.expand(B, T, H // 5, 5, W // 9, 9, C)
    ref_w = (dpv * xn).sum((0, 1, 2, 4, 6)).reshape(1, 45)
    b_w = 2 * ((dpv.abs() * xn_err).sum((0, 1, 2, 4, 6)) + (n_add + 23) * U * (dpv * xn).abs().sum((0, 1, 2, 4, 6)))
    check_bounded(dpw.cpu(), ref_w.cpu(), b_w.reshape(1, 45).cpu(), case + " dpool_w")
    check_bounded(dpb.cpu(), dp.sum().view(1).cpu(), (2 * (n_add + 23) * U * dp.abs().sum()).view(1).cpu(),
                  case + " dpool_b")
    # parts left out: no dx, or the pooling's gradients alone (the norm's partial columns are not written)
    _, dg2, _, dpw2, _ = ops.layer_norm_pool_backward(x, drows, None, gamma, beta, 1e-5, pw, (5, 9), need_x=False)
    check_same_bits(dg2, dg, "no dx: dgamma")
    check_same_bits(dpw2, dpw, "no dx: dpool_w")
    _, n1, n2, dpw3, dpb3 = ops.layer_norm_pool_backward(x, drows, None, gamma, beta, 1e-5, pw, (5, 9), need_x=False,
                                                         need_norm=False)
    assert n1 is None and n2 is None
    check_same_bits(dpw3, dpw, "pool only: dpool_w")
    check_same_bits(dpb3, dpb, "pool only: dpool_b")


# ---------------------------------------------------------------------------------------------------- the block
def _block(cuda, hq, seed, focal_level=2):
    torch.manual_seed(seed)
    t2t = dict(T2T) if hq else dict(T2T, output_size=(60, 108))
    blk = TemporalFocalTransformerBlock(512, 4, (5, 9), focal_level=focal_level, focal_window=(5, 9), t2t_params=t2t,
                                        pool_method="fc", hq=hq).to(cuda)
    with torch.no_grad():
        for name, p_ in blk.named_parameters():
            if name.startswith("norm"):
                p_.add_(0.1 * torch.randn_like(p_))
            elif name.startswith("pool"):
                p_.add_(0.02 * torch.randn_like(p_))
            else:
                p_.normal_(0, 0.05 if name.endswith("weight") else 0.1)
    return blk


class _Linear64:
    """restate._linear with the attention's qkv evaluated at the kernels' fp16 values (passed straight through) and
    every Linear's input and output kept, with their gradients, for the bounds."""

    def __init__(self, qkvs):
        self.qkvs, self.calls = list(qkvs), []

    def __call__(self, sd, prefix, x):
        y = F.linear(x, sd[prefix + ".weight"], sd.get(prefix + ".bias"))
        if prefix.endswith(".attn.qkv"):
            kern = self.qkvs.pop(0)
            y = y + (kern.double().cpu().view(y.shape) - y).detach()
        for t in (x, y):
            if t.requires_grad:
                t.retain_grad()
        self.calls.append((prefix, x, y))
        return y


def _kernel_qkvs(blocks, x, output_size):
    """The fp16 qkv (and qkv_pooled) each block's kernels compute, in the order the restatement asks for them."""
    out = []
    with torch.no_grad():
        for blk in blocks:
            keep = {}
            x = blk._forward(x, output_size, keep)
            out.append(keep["attn"]["qkv"])
            if keep["attn"]["qkv_pooled"] is not None:
                out.append(keep["attn"]["qkv_pooled"])
    return out


def _block64_nopool(sd, prefix, x, output_size):
    """transformer_block without the pooled keys (focal_level=1: no pool_layers), restated alike."""
    B, T, H, W, C = x.shape
    xn = F.layer_norm(x, (C,), sd[prefix + ".norm1.weight"], sd[prefix + ".norm1.bias"])
    qkv = restate._linear(sd, prefix + ".attn.qkv", xn)
    att = restate.focal_window_attention(qkv, None, 4, (5, 9), (2, 4), (5, 9), 128 ** -0.5,
                                         sd[prefix + ".attn.valid_ind_rolled"])
    x = x + restate._linear(sd, prefix + ".attn.proj", att)
    y = F.layer_norm(x, (C,), sd[prefix + ".norm2.weight"], sd[prefix + ".norm2.bias"])
    y = restate._linear(sd, prefix + ".mlp.conv1.0", y.view(B, T * H * W, C))
    y = restate._fold_average(None, y, output_size, H * W)
    y = restate._linear(sd, prefix + ".mlp.conv2.1", F.gelu(y))
    return x + y.view(B, T, H, W, C)


def _sd64(blk, prefix):
    sd = {f"{prefix}.{k}": v.detach().double().cpu().requires_grad_() for k, v in blk.named_parameters()}
    sd.update({f"{prefix}.{k}": v.cpu() for k, v in blk.named_buffers()})
    return sd


def _ln_abs(x, gamma, a):
    """A LayerNorm's input gradient restated on absolute values: a = the absolute gradient of its output."""
    xh, rstd, _ = _ln64(x)
    ga = gamma.detach().double().abs() * a
    return rstd * (ga + ga.mean(-1, keepdim=True) + xh.abs() * (ga * xh.abs()).mean(-1, keepdim=True))


def _block_bounds(prefix, calls, sd, x_in, pooled_block):
    """A (module docstring) for every parameter of one restated block and for its input, from its Linear calls."""
    by = {}
    for p, xx, yy in calls:
        if p.startswith(prefix + "."):
            by.setdefault(p[len(prefix) + 1:], []).append((xx, yy))
    C = 512
    bound = {}
    for name, uses in by.items():
        dy = torch.cat([yy.grad.reshape(-1, yy.shape[-1]).abs() for _, yy in uses])
        xs = torch.cat([xx.detach().reshape(-1, xx.shape[-1]).abs() for xx, _ in uses])
        bound[name + ".weight"] = dy.t() @ xs
        bound[name + ".bias"] = dy.sum(0)
    (xn, qkv), = by["attn.qkv"][:1]
    (att, proj), = by["attn.proj"]
    (y2, h1), = by["mlp.conv1.0"]
    x_in = x_in.detach()
    B, T, H, W, _ = x_in.shape
    x1 = x_in + proj.detach()
    xh2, _, _ = _ln64(x1)
    xh1, _, _ = _ln64(x_in)
    dy2 = y2.grad.view(x_in.shape).abs()
    dxn = xn.grad.abs()
    bound["norm2.weight"], bound["norm2.bias"] = (dy2 * xh2.abs()).sum((0, 1, 2, 3)), dy2.sum((0, 1, 2, 3))
    bound["norm1.weight"], bound["norm1.bias"] = (dxn * xh1.abs()).sum((0, 1, 2, 3)), dxn.sum((0, 1, 2, 3))
    w1 = sd[prefix + ".mlp.conv1.0.weight"].detach().abs()
    wq = sd[prefix + ".attn.qkv.weight"].detach().abs()
    a_dx1 = proj.grad.abs() + _ln_abs(x1, sd[prefix + ".norm2.weight"], (h1.grad.abs() @ w1).view(x_in.shape))
    a_xn = (qkv.grad.abs() @ wq).view(x_in.shape)
    if pooled_block:
        (pooled, qkv_p) = by["attn.qkv"][1]
        dp = pooled.grad.abs()                                                     # (B,T,nWh,nWw,C)
        xn6 = xn.detach().abs().view(B, T, H // 5, 5, W // 9, 9, C)
        dp6 = dp.view(B, T, H // 5, 1, W // 9, 1, C)
        bound["pool_layers.0.weight"] = (dp6 * xn6).sum((0, 1, 2, 4, 6)).reshape(1, 45)
        bound["pool_layers.0.bias"] = dp.sum().view(1)
        wp = sd[prefix + ".pool_layers.0.weight"].detach().abs().view(1, 1, 1, 5, 1, 9, 1)
        a_p = (qkv_p.grad.abs() @ wq).view(B, T, H // 5, 1, W // 9, 1, C)
        a_xn = a_xn + (wp * a_p).expand(B, T, H // 5, 5, W // 9, 9, C).reshape(B, T, H, W, C)
    bound["x"] = a_dx1 + _ln_abs(x_in, sd[prefix + ".norm1.weight"], a_xn)
    return bound


def _run_block(blk, x, output_size):
    out = blk([x, output_size]) if blk.hq else blk(x)
    return out[0] if blk.hq else out


@pytest.mark.parametrize("case,hq,B,T,H,W,level", [("base", False, 1, 2, 20, 36, 2), ("hq", True, 1, 1, 40, 72, 2),
                                                   ("base-l1", False, 1, 2, 20, 36, 1)])
def test_block_against_float64(cuda, monkeypatch, case, hq, B, T, H, W, level):
    """Every parameter and x of one block against float64 autograd of the restated block; the tracked output is the
    same bits as the untracked one, and a repeat gives the same gradient bits."""
    blk = _block(cuda, hq, 17, level)
    size = (3 * H, 3 * W)
    g_ = torch.Generator(device=cuda).manual_seed(5)
    x = torch.randn(B, T, H, W, 512, device=cuda, generator=g_)
    dout = torch.randn(B, T, H, W, 512, device=cuda, generator=g_)
    with torch.no_grad():
        want = _run_block(blk, x, size)
    grads = []
    for _ in range(2):
        blk.zero_grad()
        xs = x.clone().requires_grad_()
        out = _run_block(blk, xs, size)
        assert out.grad_fn is not None
        check_same_bits(out, want, f"{case} tracked output")
        out.backward(dout)
        grads.append([xs.grad] + [p_.grad.clone() for p_ in blk.parameters()])
    for a, b_ in zip(*grads):
        check_same_bits(a, b_, f"{case} gradient repeat")
    lin = _Linear64(_kernel_qkvs([blk], x, size))
    monkeypatch.setattr(restate, "_linear", lin)
    sd = _sd64(blk, "blk")
    with reference_math():
        x64 = x.double().cpu().requires_grad_()
        if level == 2:
            out64 = restate.transformer_block(sd, "blk", x64, size)
        else:
            out64 = _block64_nopool(sd, "blk", x64, size)
        out64.backward(dout.double().cpu())
        bound = _block_bounds("blk", lin.calls, sd, x64, level == 2)
    for k, p_ in blk.named_parameters():
        check_close(p_.grad.cpu(), sd["blk." + k].grad, 6 * bound[k].view(p_.shape), 1e-3, "f32", f"{case} {k}")
    check_close(xs.grad.cpu(), x64.grad, 6 * bound["x"], 1e-3, "f32", f"{case} x")


@pytest.mark.parametrize("hq,b,t,h,w", [(False, 1, 2, 60, 108), (True, 1, 2, 30, 54)])
def test_trunk_against_float64(cuda, monkeypatch, hq, b, t, h, w):
    """sc(transformer(ss(feat)), t, residual=feat) of the generators' trunk: all eight blocks, every block parameter
    and feat against float64 autograd of the restatement (bound: module docstring)."""
    torch.manual_seed(23)
    size = (h, w)
    ss = SoftSplit(128, 512, **T2T, t2t_param=None if hq else dict(T2T, output_size=size)).to(cuda)
    sc = SoftComp(128, 512, None if hq else size, hq=hq).to(cuda)
    blocks = torch.nn.Sequential(*[_block(cuda, hq, 100 + i) for i in range(8)])
    if not hq:
        for blk in blocks:
            blk.mlp.t2t_params["output_size"] = size
    g_ = torch.Generator(device=cuda).manual_seed(8)
    feat = torch.randn(b * t, 128, h, w, device=cuda, generator=g_).contiguous(memory_format=torch.channels_last)
    dout = torch.randn(b * t, 128, h, w, device=cuda, generator=g_)

    def run(f):
        tok = ss(f, b, size)
        tok = blocks([tok, size])[0] if hq else blocks(tok)
        return sc(tok, t, size, residual=f)
    with torch.no_grad():
        want = run(feat)
    fs = feat.clone().requires_grad_()
    out = run(fs)
    check_same_bits(out.contiguous(), want.contiguous(), "trunk tracked output")
    out.backward(dout)
    with torch.no_grad():
        tok0 = ss(feat, b, size)
    lin = _Linear64(_kernel_qkvs(blocks, tok0, size))
    monkeypatch.setattr(restate, "_linear", lin)
    sd = {}
    for i, blk in enumerate(blocks):
        sd.update(_sd64(blk, f"transformer.{i}"))
    with reference_math():
        f64 = feat.double().cpu().requires_grad_()
        fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
        tok = F.linear(F.unfold(f64, **T2T).transpose(1, 2), ss.embedding.weight.double().cpu(),
                       ss.embedding.bias.double().cpu()).reshape(b, t, fh, fw, 512)
        ins = []
        for i in range(8):
            tok.retain_grad()
            ins.append(tok)
            tok = restate.transformer_block(sd, f"transformer.{i}", tok, size)
        cols = F.linear(tok.reshape(b * t, fh * fw, 512), sc.embedding.weight.double().cpu(),
                        sc.embedding.bias.double().cpu())
        img = F.fold(cols.transpose(1, 2), size, **T2T)
        if hq:
            img = F.conv2d(img, sc.bias_conv.weight.double().cpu(), sc.bias_conv.bias.double().cpu(), padding=1)
        else:
            img = img + sc.bias.double().cpu()
        (img + f64).backward(dout.double().cpu())
        bounds = [_block_bounds(f"transformer.{i}", lin.calls, sd, ins[i], True) for i in range(8)]
    case = "hq" if hq else "base"
    for i, blk in enumerate(blocks):
        for k, p_ in blk.named_parameters():
            check_close(p_.grad.cpu(), sd[f"transformer.{i}.{k}"].grad, 48 * bounds[i][k].view(p_.shape), 1e-3, "f32",
                        f"trunk {case} block {i} {k}")
    # feat: through SoftSplit (its input gradient sums 49 token gradients per pixel) and as SoftComp's residual
    a_tok = bounds[0]["x"].reshape(b * t, fh * fw, 512) @ ss.embedding.weight.double().cpu().abs()
    a_feat = F.fold(a_tok.transpose(1, 2), size, **T2T) + dout.double().cpu().abs()
    check_close(fs.grad.cpu(), f64.grad, 48 * a_feat, 1e-3, "f32", f"trunk {case} feat")


# ---------------------------------------------------------------------------------------------------- launches
def _launched(fn):
    rec = ops.profile_kernels(True)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        ops.profile_kernels(False)
    return {k: len(v) for k, v in rec.items()}


def test_launch_sets_and_second_backward(cuda):
    """Frozen norms launch no partial sums; with only mlp trainable and tokens without grad only the feed-forward's
    kernels run; no_grad gives no grad_fn; a second backward raises."""
    blk = _block(cuda, False, 3)
    g_ = torch.Generator(device=cuda).manual_seed(1)
    x = torch.randn(1, 2, 20, 36, 512, device=cuda, generator=g_)
    for n in (blk.norm1, blk.norm2):
        n.weight.requires_grad_(False)
        n.bias.requires_grad_(False)
    blk.pool_layers.requires_grad_(False)
    out = blk(x.clone().requires_grad_())
    got = _launched(lambda: out.sum().backward())
    # the LayerNorm backwards still run for dx1 and dx, without partial sums (test_layernorm_backward_against_float64
    # counts their kernels)
    assert got == {"linear_wgrad_bf16x3": 4, "linear_bf16x3": 4, "t2t_fold_unfold_adjoint": 1, "layernorm_backward": 1,
                   "focal_window_attention_backward": 1, "layernorm_pool_backward": 1}, got
    assert blk.norm1.weight.grad is None and blk.norm2.bias.grad is None and blk.pool_layers[0].weight.grad is None
    blk.requires_grad_(False)
    blk.mlp.requires_grad_(True)
    out = blk(x)
    got = _launched(lambda: out.sum().backward(retain_graph=True))
    assert got == {"linear_wgrad_bf16x3": 2, "linear_bf16x3": 1, "t2t_fold_unfold_adjoint": 1}, got
    with pytest.raises(RuntimeError, match="backpropagated a second time"):
        out.sum().backward()
    with torch.no_grad():
        assert blk(x.clone().requires_grad_()).grad_fn is None
    out = blk(x)
    with torch.no_grad():
        blk.mlp.conv2[1].weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.sum().backward()


@pytest.mark.parametrize("hq", [False, True])
def test_generator_forward_stays_untracked(cuda, hq):
    """InpaintGenerator.forward with trainable parameters under grad mode launches the same kernels, the same number of
    times, as under no_grad, and predicts the same bits."""
    import importlib
    import warnings
    from e2fgvi_b200.synth import synth_frames, synth_state_dict
    net = importlib.import_module("model." + ("e2fgvi_hq" if hq else "e2fgvi"))
    m = net.InpaintGenerator().eval()
    m.load_state_dict(synth_state_dict(m, "stress", 3), strict=True)
    m = m.to(cuda)
    x = synth_frames(1, 5, 240, 432, seed=2).to(cuda)
    with torch.no_grad():
        m(x, 3)
        want = _launched(lambda: m(x, 3))
        pred0, _ = m(x, 3)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        got = _launched(lambda: m(x, 3))
        pred, _ = m(x, 3)
    assert pred.grad_fn is None
    assert got == want, (got, want)
    check_same_bits(pred, pred0, "prediction under grad mode")


def test_adam_steps_track_float64(cuda, monkeypatch):
    """Three Adam steps of one block on the mean squared error against a target next to the same steps in float64: each
    parameter's total update is within 1e-3 (L2, relative) of the float64 one."""
    blk = _block(cuda, False, 29)
    size = (60, 108)
    g_ = torch.Generator(device=cuda).manual_seed(4)
    x = torch.randn(1, 2, 20, 36, 512, device=cuda, generator=g_)
    target = torch.randn(1, 2, 20, 36, 512, device=cuda, generator=g_)
    named = dict(blk.named_parameters())
    start = {k: v.detach().clone() for k, v in named.items()}
    F.mse_loss(blk(x), target).backward()
    eps = {k: 10 * float(v.grad.abs().max()) for k, v in named.items()}
    blk.zero_grad()
    sd = _sd64(blk, "blk")
    opt = torch.optim.Adam([{"params": [named[k]], "eps": eps[k]} for k in named], lr=1e-3)
    opt64 = torch.optim.Adam([{"params": [sd["blk." + k]], "eps": eps[k]} for k in named], lr=1e-3)
    for _ in range(3):
        # float64 first: its attention is evaluated at the fp16 qkv of the block's weights before this step
        monkeypatch.setattr(restate, "_linear", _Linear64(_kernel_qkvs([blk], x, None)))
        opt64.zero_grad()
        with reference_math():
            F.mse_loss(restate.transformer_block(sd, "blk", x.double().cpu(), size), target.double().cpu()).backward()
        opt64.step()
        opt.zero_grad()
        F.mse_loss(blk(x), target).backward()
        opt.step()
    for k, v in named.items():
        d, d64 = (v.detach() - start[k]).double().cpu(), sd["blk." + k].detach() - start[k].double().cpu()
        assert ((d - d64).norm() / d64.norm()).item() < 1e-3, k
