"""H100: the focal window attention in training — the attention backward (``e2f_focal_window_attention_backward``) and
the differentiable ``WindowAttention`` — against float64 torch autograd of the restatement, element by element.

Bounds (kernel_checks.check_close, C = 2^-14):
* the attention backward: C * A with A the largest magnitude of the float64 gradient of the checked part (the q, k or v
  columns).  Its products run on wgmma with the bf16 three-term split and fp32 accumulation (fp16 operands exact as
  two terms; dO, P and dS split to 2^-17).
* the module: 3 C A as for the transformer's other Linears, A the gradient's last product on absolute values at the
  float64 intermediate gradients (|dqkv|^T |x; pooled|, |dqkv| |W_qkv|, |g|^T |O|).  The reference evaluates the
  attention at the fp16 qkv the kernels read (the qkv Linear's own rounding), passing the gradient straight through
  that rounding, as the backward does."""
import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.tfocal_transformer import WindowAttention, rolled_valid_indices
from kernel_checks import check_close, check_same_bits
from oracle import restate

pytestmark = pytest.mark.gpu

WIN, EXP, FOC, HEADS = (5, 9), (2, 4), (5, 9), 4
SCALE = 128 ** -0.5


def _check_parts(got, ref, what):
    for i, part in enumerate("qkv"):
        r = ref[..., 512 * i:512 * (i + 1)]
        if part == "q" and what.endswith("pooled"):
            assert int((got[..., :512] != 0).sum()) == 0, what
            continue
        check_close(got[..., 512 * i:512 * (i + 1)], r, r.abs().max().expand_as(r), 1e-4, "f32", f"{what} d{part}")


def _inputs(cuda, B, T, H, W, use_pooled, seed):
    g = torch.Generator(device=cuda).manual_seed(seed)
    qkv = (torch.randn(B, T, H, W, 3 * 512, device=cuda, generator=g) * 1.5).half()
    qkv_p = None
    if use_pooled:
        qkv_p = (torch.randn(B, T, H // 5, W // 9, 3 * 512, device=cuda, generator=g) * 1.5).half()
    dout = torch.randn(B, T, H, W, 512, device=cuda, generator=g)
    return qkv, qkv_p, dout


# (B, T, H, W, use_pooled): the training grid, a one-window grid (rolls wrap onto the window), 10x18 and 15x27 (pooled
# grids smaller than the 5x9 neighbourhood), an HQ-style grid; T = 1 and 8, B > 1
CORE = [(2, 8, 20, 36, 1), (1, 8, 20, 36, 0), (1, 1, 5, 9, 1), (2, 8, 5, 9, 1), (1, 8, 5, 9, 0), (1, 8, 10, 18, 1),
        (2, 1, 10, 18, 0), (1, 2, 15, 27, 1), (1, 2, 40, 72, 1), (1, 1, 40, 72, 0)]


@pytest.mark.parametrize("B,T,H,W,use_pooled", CORE)
def test_core_against_float64(cuda, B, T, H, W, use_pooled):
    qkv, qkv_p, dout = _inputs(cuda, B, T, H, W, use_pooled, B * 100 + T * 10 + H + use_pooled)
    d = ops.focal_window_attention_backward(qkv, qkv_p, dout, HEADS, WIN, EXP, FOC, SCALE)
    again = ops.focal_window_attention_backward(qkv, qkv_p, dout, HEADS, WIN, EXP, FOC, SCALE)
    check_same_bits(d, again, "attention backward")
    q64 = qkv.cpu().double().requires_grad_()
    p64 = qkv_p.cpu().double().requires_grad_() if use_pooled else None
    out = restate.focal_window_attention(q64, p64, HEADS, WIN, EXP, FOC, SCALE, rolled_valid_indices(WIN, EXP))
    out.backward(dout.cpu().double())
    n_tok = B * T * H * W
    d = d.cpu()
    case = f"core {B}x{T}x{H}x{W} p{use_pooled}"
    _check_parts(d[:n_tok], q64.grad.reshape(n_tok, -1), case)
    if use_pooled:
        _check_parts(d[n_tok:], p64.grad.reshape(d.shape[0] - n_tok, -1), case + " pooled")
    else:
        assert d.shape[0] == n_tok


def _module(cuda, seed, use_pooled=True):
    torch.manual_seed(seed)
    mod = WindowAttention(512, EXP, WIN, FOC, 2 if use_pooled else 1, HEADS, True, "fc").to(cuda)
    with torch.no_grad():
        for p_ in mod.parameters():
            p_.normal_(0, 0.05)
    return mod


def _module64(mod, p, x, pooled, residual, keep=None):
    """WindowAttention.attend in float64 on the CPU on the restated attention (p, x, pooled, residual: CPU float64),
    the attention evaluated at the fp16 qkv the kernels compute from the module's weights."""
    dev = mod.qkv.weight.device

    def qkv_at(rows):
        y = F.linear(rows, p["qkv.weight"], p["qkv.bias"])
        kern = ops.linear(rows.detach().float().contiguous().to(dev), mod.qkv.weight, mod.qkv.bias,
                          out_dtype=torch.float16)
        return y + (kern.double().cpu().view(y.shape) - y).detach()
    qkv = qkv_at(x)
    qkv_p = qkv_at(pooled.permute(0, 3, 1, 2, 4)) if pooled is not None else None
    att = restate.focal_window_attention(qkv, qkv_p, HEADS, WIN, EXP, FOC, SCALE, rolled_valid_indices(WIN, EXP))
    out = F.linear(att, p["proj.weight"], p["proj.bias"])
    if keep is not None:
        for t in (qkv, qkv_p, att):
            if t is not None:
                t.retain_grad()
        keep.update(qkv=qkv, qkv_p=qkv_p, att=att)
    return out + residual if residual is not None else out


@pytest.mark.parametrize("case,B,T,H,W,use_pooled", [("base", 1, 2, 20, 36, True), ("base-l1", 2, 2, 10, 18, False),
                                                     ("hq", 1, 1, 40, 72, True)])
def test_module_against_float64(cuda, case, B, T, H, W, use_pooled):
    """Every parameter, x, pooled and the residual of WindowAttention against float64 autograd of the restated module;
    the tracked output is the same bits as the untracked one."""
    mod = _module(cuda, 11, use_pooled)
    g = torch.Generator(device=cuda).manual_seed(3)
    x = torch.randn(B, T, H, W, 512, device=cuda, generator=g)
    pooled = torch.randn(B, H // 5, W // 9, T, 512, device=cuda, generator=g) if use_pooled else None
    res = torch.randn(B, T, H, W, 512, device=cuda, generator=g)
    dout = torch.randn(B, T, H, W, 512, device=cuda, generator=g)
    with torch.no_grad():
        want = mod.attend(x, pooled, residual=res)
    xs = x.clone().requires_grad_()
    ps = pooled.clone().requires_grad_() if use_pooled else None
    rs = res.clone().requires_grad_()
    out = mod.attend(xs, ps, residual=rs)
    assert out.grad_fn is not None
    check_same_bits(out, want, "tracked output")
    out.backward(dout)
    p64 = {k: v.detach().cpu().double().requires_grad_() for k, v in mod.named_parameters()}
    x64 = x.cpu().double().requires_grad_()
    pool64 = pooled.cpu().double().requires_grad_() if use_pooled else None
    r64 = res.cpu().double().requires_grad_()
    keep = {}
    g64 = dout.cpu().double()
    _module64(mod, p64, x64, pool64, r64, keep).backward(g64)
    # A: the last product of each gradient on absolute values, at the float64 intermediate gradients
    C = 512
    dq_tok = keep["qkv"].grad.reshape(-1, 3 * C).abs()
    dq_all, rows = dq_tok, x64.detach().reshape(-1, C).abs()
    if use_pooled:
        dq_all = torch.cat([dq_tok, keep["qkv_p"].grad.reshape(-1, 3 * C).abs()])
        rows = torch.cat([rows, pool64.detach().permute(0, 3, 1, 2, 4).reshape(-1, C).abs()])
    g_abs, att_abs = g64.reshape(-1, C).abs(), keep["att"].detach().reshape(-1, C).abs()
    wq_abs = p64["qkv.weight"].detach().abs()
    bound = {"qkv.weight": dq_all.t() @ rows, "qkv.bias": dq_all.sum(0), "proj.weight": g_abs.t() @ att_abs,
             "proj.bias": g_abs.sum(0)}
    for k, v in mod.named_parameters():
        check_close(v.grad.cpu(), p64[k].grad, 3 * bound[k], 1e-3, "f32", f"{case} {k}")
    check_close(xs.grad.cpu(), x64.grad, 3 * (dq_tok @ wq_abs).view(x64.shape), 1e-3, "f32", f"{case} x")
    check_close(rs.grad.cpu(), r64.grad, g64.abs(), 1e-6, "f32", f"{case} residual")
    if use_pooled:
        dq_p = keep["qkv_p"].grad.abs() @ wq_abs                  # (B,T,nWh,nWw,C)
        check_close(ps.grad.cpu(), pool64.grad, 3 * dq_p.permute(0, 2, 3, 1, 4), 1e-3, "f32", f"{case} pooled")
    # the reference boundary: forward(x_all) is tracked too and partitions the same result
    got = mod([xs, ps] if use_pooled else [xs])
    assert got.grad_fn is not None and got.shape == (B * (H // 5) * (W // 9), T * 45, 512)


def _launched(fn):
    rec = ops.profile_kernels(True)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        ops.profile_kernels(False)
    return {k: len(v) for k, v in rec.items()}


def test_launch_sets_and_second_backward(cuda):
    """A frozen qkv or proj launches no weight gradient; x and pooled without grad launch no qkv input gradient; a
    second backward raises."""
    mod = _module(cuda, 5)
    g = torch.Generator(device=cuda).manual_seed(9)
    x = torch.randn(1, 2, 20, 36, 512, device=cuda, generator=g)
    pooled = torch.randn(1, 4, 4, 2, 512, device=cuda, generator=g)
    mod.qkv.weight.requires_grad_(False)
    mod.qkv.bias.requires_grad_(False)
    out = mod.attend(x, pooled)
    got = _launched(lambda: out.sum().backward())
    # proj's weight gradient only; dO, the attention backward and qkv's input gradient are not needed
    assert got == {"linear_wgrad_bf16x3": 1}, got
    mod.qkv.weight.requires_grad_(True)
    for p_ in mod.proj.parameters():
        p_.requires_grad_(False)
    out = mod.attend(x, pooled)
    got = _launched(lambda: out.sum().backward())
    # dO (proj input gradient), the attention backward, qkv's weight gradient; no qkv input gradient
    assert got == {"linear_bf16x3": 1, "focal_window_attention_backward": 1, "linear_wgrad_bf16x3": 1}, got
    mod.qkv.weight.requires_grad_(False)
    mod.qkv.bias.requires_grad_(False)
    out = mod.attend(x.clone().requires_grad_(), pooled)
    got = _launched(lambda: out.sum().backward(retain_graph=True))
    assert got == {"linear_bf16x3": 2, "focal_window_attention_backward": 1}, got
    with pytest.raises(RuntimeError, match="backpropagated a second time"):
        out.sum().backward()
    with torch.no_grad():
        assert mod.attend(x.clone().requires_grad_(), pooled).grad_fn is None


def test_adam_steps_track_float64(cuda):
    """Three Adam steps on the mean squared error against a target next to the same steps in float64: each parameter's
    total update is within 1e-3 (L2, relative) of the float64 one.  Later steps read the transposed weights the cache
    rebuilds after each step; a stale W^T would move dO and the input gradients."""
    mod = _module(cuda, 21)
    g = torch.Generator(device=cuda).manual_seed(4)
    x = torch.randn(1, 2, 20, 36, 512, device=cuda, generator=g, requires_grad=True)
    pooled = torch.randn(1, 4, 4, 2, 512, device=cuda, generator=g)
    target = torch.randn(1, 2, 20, 36, 512, device=cuda, generator=g)
    p64 = {k: v.detach().cpu().double().requires_grad_() for k, v in mod.named_parameters()}
    named = dict(mod.named_parameters())
    start = {k: v.detach().clone() for k, v in named.items()}
    F.mse_loss(mod.attend(x, pooled), target).backward()
    eps = {k: 10 * float(v.grad.abs().max()) for k, v in named.items()}
    mod.zero_grad()
    opt = torch.optim.Adam([{"params": [named[k]], "eps": eps[k]} for k in named], lr=1e-3)
    opt64 = torch.optim.Adam([{"params": [p64[k]], "eps": eps[k]} for k in named], lr=1e-3)
    for _ in range(3):
        # float64 first: its attention is evaluated at the fp16 qkv of the module's weights before this step
        opt64.zero_grad()
        F.mse_loss(_module64(mod, p64, x.detach().cpu().double(), pooled.cpu().double(), None),
                   target.cpu().double()).backward()
        opt64.step()
        opt.zero_grad()
        F.mse_loss(mod.attend(x, pooled), target).backward()
        opt.step()
    for k, v in named.items():
        d, d64 = (v.detach() - start[k]).double().cpu(), p64[k].detach() - start[k].double().cpu()
        assert ((d - d64).norm() / d64.norm()).item() < 1e-3, k
