"""H100: the encoder / decoder backward — the 3x3 input and weight gradients (stride 1 and 2, groups, two sources, the
residual-then-derivative epilogue, the row-gapped output conv), the upsample adjoint, the tanh prologue, and the
differentiable ``Encoder`` / ``decode`` — against float64 torch (cuDNN off) element by element.  The schedules of the
input gradient past one tile per CTA are checked under torch.profiler in test_gpu_schedules_encdec.py, which runs
after every test that calls backward: on the H100, a profiler session followed in the same process by autograd
backward passes left later profiler sessions with no kernel records.

Per-element bounds as in kernel_checks: C * A for the bf16x3 split, A the same operation on absolute values.  Weight
gradients also carry the accumulation term of their fixed-order split-K sum, 2^-24 * (12 * K blocks per slice +
slices) * A (test_gpu_train_schedules documents it)."""
import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.generator import _ENC
from kernel_checks import (assert_exact_grid, cdiv, check_close, check_exact, check_same_bits, grid_values, int_values,
                           reference_math)
from oracle import restate

pytestmark = pytest.mark.gpu


U = 2.0 ** -24
SLOPE = 0.2


def _rel(got, want):
    return ((got.double() - want.double()).abs().max() / want.double().abs().max().clamp_min(1e-30)).item()


def _cat(xs, groups):
    """The group-wise concatenation of e2fgvi.py:103-108."""
    if len(xs) == 1:
        return xs[0]
    n, _, h, w = xs[0].shape
    return torch.cat([x.reshape(n, groups, -1, h, w) for x in xs], 2).reshape(n, -1, h, w)


def _dleaky(act_hi):
    return torch.where(act_hi.double() > 0, 1.0, float(torch.tensor(SLOPE, dtype=torch.float32)))


# (name, forward source channels, cout, stride, groups): every encoder conv that has an input gradient, and the decoder's
ENC = [(f"enc{k}", [cin] if k <= 4 else [256, cin - 256], cout, s, g) for k, (cin, cout, s, g) in enumerate(_ENC) if k > 0]
DEC = [("dec0", [128], 128, 1, 1), ("dec2", [128], 64, 1, 1), ("dec4", [64], 64, 1, 1)]
CONVS = ENC + DEC
SIZES = [(1, 6, 10), (2, 13, 19)]


def _dgrad_case(cuda, chans, cout, stride, groups, source, n, h, w, act, res, exact, seed):
    g = torch.Generator(device=cuda).manual_seed(seed)
    cs = chans[source]
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    cin_g = sum(chans) // groups
    if exact:
        dy = grid_values((n, cout, ho, wo), g, density=0.3)
        wt = int_values((cout, cin_g, 3, 3), g, density=0.5)
    else:
        dy = torch.randn(n, cout, ho, wo, device=cuda, generator=g)
        wt = torch.randn(cout, cin_g, 3, 3, device=cuda, generator=g) * 0.05
    act_op = ops.split_nhwc(F.leaky_relu(torch.randn(n, cs, h, w, device=cuda, generator=g), SLOPE)) if act else None
    resid = (int_values if exact else lambda s, gg: torch.randn(*s, device=cuda, generator=gg))((n, h, w, cs), g) if res else None
    return dy, wt, act_op, resid


def _dgrad_ref(dy, wt, chans, groups, stride, source, h, w, act_op, resid):
    """float64 input gradient of the forward conv by autograd, and its bound A (same on absolute values)."""
    outs = []
    for d, ww in ((dy.double(), wt.double()), (dy.double().abs(), wt.double().abs())):
        xs = [torch.zeros(d.shape[0], c, h, w, dtype=torch.float64, device=d.device, requires_grad=True) for c in chans]
        with reference_math():
            F.conv2d(_cat(xs, groups), ww, None, stride, 1, 1, groups).backward(d)
        outs.append(xs[source].grad.permute(0, 2, 3, 1))
    ref, bound = outs
    if resid is not None:
        ref, bound = ref + resid.double(), bound + resid.double().abs()
    if act_op is not None:
        dl = _dleaky(act_op.hi.float())
        ref, bound = ref * dl, bound * dl
    return ref, bound


@pytest.mark.parametrize("name,chans,cout,stride,groups", CONVS, ids=[c[0] for c in CONVS])
@pytest.mark.parametrize("n,h,w", SIZES)
def test_dgrad_against_float64(cuda, name, chans, cout, stride, groups, n, h, w):
    for source in range(len(chans)):
        for act, res in ((False, False), (True, False), (False, True), (True, True)):
            dy, wt, act_op, resid = _dgrad_case(cuda, chans, cout, stride, groups, source, n, h, w, act, res, False,
                                                n * h + source)
            call = lambda: ops.conv_dgrad(ops.split_nhwc(dy), wt, groups=groups, stride=stride, in_size=(h, w),
                                          src_channels=chans, source=source, act=act_op, residual=resid, out="both")
            dx, sp = call()
            ref, bound = _dgrad_ref(dy, wt, chans, groups, stride, source, h, w, act_op, resid)
            what = f"{name} src{source} act{int(act)} res{int(res)} {n}x{h}x{w}"
            check_close(dx, ref, bound, 1e-4, "f32", what)
            assert _rel(sp.hi.float() + sp.lo.float(), dx) < 1e-5, what
            check_same_bits(dx, call()[0], what)


@pytest.mark.parametrize("name,chans,cout,stride,groups", CONVS, ids=[c[0] for c in CONVS])
def test_dgrad_exact_grid(cuda, name, chans, cout, stride, groups):
    n, h, w = 2, 13, 19
    for source in range(len(chans)):
        dy, wt, act_op, resid = _dgrad_case(cuda, chans, cout, stride, groups, source, n, h, w, False, True, True, 7)
        dx = ops.conv_dgrad(ops.split_nhwc(dy), wt, groups=groups, stride=stride, in_size=(h, w), src_channels=chans,
                            source=source, residual=resid)
        ref, bound = _dgrad_ref(dy, wt, chans, groups, stride, source, h, w, None, resid)
        assert_exact_grid(bound, dy, name)
        check_exact(dx, ref, f"{name} src{source} exact")


# the training size of a 240x432 frame: encoder convs 1 (120x216), 2 (stride 2 into 120x216), 3..8 (60x108), decoder
TRAIN = [("enc1", 120, 216), ("enc2", 120, 216), ("enc4", 60, 108), ("enc5", 60, 108), ("enc6", 60, 108),
         ("enc7", 60, 108), ("enc8", 60, 108), ("dec0", 120, 216), ("dec2", 120, 216), ("dec4", 240, 432)]


@pytest.mark.parametrize("name,h,w", TRAIN, ids=[t[0] for t in TRAIN])
def test_dgrad_training_size(cuda, name, h, w):
    _, chans, cout, stride, groups = next(c for c in CONVS if c[0] == name)
    source = len(chans) - 1
    dy, wt, act_op, resid = _dgrad_case(cuda, chans, cout, stride, groups, source, 1, h, w, True, True, False, h)
    dx = ops.conv_dgrad(ops.split_nhwc(dy), wt, groups=groups, stride=stride, in_size=(h, w), src_channels=chans,
                        source=source, act=act_op, residual=resid)
    ref, bound = _dgrad_ref(dy, wt, chans, groups, stride, source, h, w, act_op, resid)
    check_close(dx, ref, bound, 1e-4, "f32", f"{name} {h}x{w}")


@pytest.mark.parametrize("n,h,w", SIZES + [(1, 240, 432)])
def test_output_conv_dgrad_rows(cuda, n, h, w):
    """The 64 -> 3 output conv: dY row-gapped (lead 1, 8 channels) from the tanh prologue."""
    g = torch.Generator(device=cuda).manual_seed(h)
    wt = torch.randn(3, 64, 3, 3, device=cuda, generator=g) * 0.05
    pred = torch.tanh(torch.randn(n, 3, h, w, device=cuda, generator=g))
    dout = torch.randn(n, 3, h, w, device=cuda, generator=g)
    act_op = ops.split_nhwc(F.leaky_relu(torch.randn(n, 64, h, w, device=cuda, generator=g), SLOPE))
    dy32, rows = ops.tanh_backward_rows(dout, pred, lead=1)
    want = dout.double() * (1 - pred.double() ** 2)
    assert _rel(dy32[..., :3].permute(0, 3, 1, 2), want) < 1e-6
    assert torch.count_nonzero(dy32[..., 3:]) == 0
    assert _rel(rows.dense(), want) < 1e-5
    dx = ops.conv_dgrad(rows, wt, act=act_op)
    ref, bound = _dgrad_ref(dy32[..., :3].permute(0, 3, 1, 2).contiguous(), wt, [64], 1, 1, 0, h, w, act_op, None)
    check_close(dx, ref, bound, 1e-4, "f32", f"out conv rows {n}x{h}x{w}")


def _wgrad_ref(x64s, dy64, groups, stride):
    outs = []
    for xs, d in ((x64s, dy64), ([x.abs() for x in x64s], dy64.abs())):
        xc = _cat(xs, groups)
        w = torch.zeros(d.shape[1], xc.shape[1] // groups, 3, 3, dtype=torch.float64, device=d.device, requires_grad=True)
        b = torch.zeros(d.shape[1], dtype=torch.float64, device=d.device, requires_grad=True)
        with reference_math():
            F.conv2d(xc, w, b, stride, 1, 1, groups).backward(d)
        outs += [w.grad, b.grad]
    return outs


def _slices(pixels, cout, n_cols, groups):
    s = cdiv(264, groups * cdiv(cout // groups, 64) * cdiv(n_cols, 128))
    return max(1, min(s, pixels // 256, 64))


@pytest.mark.parametrize("name,chans,cout,stride,groups", CONVS, ids=[c[0] for c in CONVS])
@pytest.mark.parametrize("n,h,w", SIZES + [(1, 60, 108)])
def test_wgrad_against_float64(cuda, name, chans, cout, stride, groups, n, h, w):
    g = torch.Generator(device=cuda).manual_seed(n * w + cout)
    xs = [torch.randn(n, c, h, w, device=cuda, generator=g) for c in chans]
    ops_ = [ops.split_nhwc(x) for x in xs]
    x64 = [(o.hi.double() + o.lo.double()).permute(0, 3, 1, 2) for o in ops_]
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    dy = torch.randn(n, ho, wo, cout, device=cuda, generator=g)
    dw, db = ops.conv3x3_wgrad(dy, ops_, groups=groups, stride=stride)
    ref_w, ref_b, bw, bb = _wgrad_ref(x64, dy.double().permute(0, 3, 1, 2), groups, stride)
    pixels = n * ho * wo
    sl = _slices(pixels, cout, 9 * sum(chans) // groups, groups)
    kb = cdiv(cdiv(cdiv(pixels, sl), 64) * 64, 64)
    what = f"{name} {n}x{h}x{w}"
    check_close(dw, ref_w, bw, 1e-4, "f32", what + " dW", extra=U * (12 * kb + sl) * bw)
    check_close(db, ref_b, torch.zeros_like(bb), 1e-4, "f32", what + " db", extra=U * (kb * 64 + 256 + sl) * bb)
    check_same_bits((dw, db), ops.conv3x3_wgrad(dy, ops_, groups=groups, stride=stride), what)
    # exact-grid: X on the grid, integer dY
    xs = [grid_values((n, c, h, w), g, density=0.2) for c in chans]
    ops_ = [ops.split_nhwc(x) for x in xs]
    dyi = int_values((n, ho, wo, cout), g, density=0.2)
    dw, db = ops.conv3x3_wgrad(dyi, ops_, groups=groups, stride=stride)
    ref_w, ref_b, bw, _ = _wgrad_ref([x.double() for x in xs], dyi.double().permute(0, 3, 1, 2), groups, stride)
    assert_exact_grid(bw, torch.cat([x.flatten() for x in xs]), what)
    check_exact(dw, ref_w, what + " dW exact")
    check_exact(db, ref_b, what + " db exact")


@pytest.mark.parametrize("n,h,w", [(2, 12, 20), (1, 240, 432)])
def test_stem_wgrad_rows(cuda, n, h, w):
    """Encoder conv 0 (3 -> 64, stride 2) on its own 8-channel row-gapped packing of the frames."""
    g = torch.Generator(device=cuda).manual_seed(w)
    x = torch.rand(n, 3, h, w, device=cuda, generator=g) * 2 - 1
    rows = ops.pack_rows(x, lead=1, cin=8)
    dy = torch.randn(n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, 64, device=cuda, generator=g)
    dw, db = ops.conv3x3_wgrad(dy, [rows], stride=2, cin=3)
    assert dw.shape == (64, 3, 3, 3)
    ref_w, ref_b, _, _ = _wgrad_ref([rows.dense().double()], dy.double().permute(0, 3, 1, 2), 1, 2)
    assert _rel(dw, ref_w) < 1e-4 and _rel(db, ref_b) < 1e-4


@pytest.mark.parametrize("n,h,w,c", [(2, 5, 9, 64), (1, 60, 108, 128), (1, 120, 216, 64)])
@pytest.mark.parametrize("act", [False, True])
def test_upsample_backward_against_float64(cuda, n, h, w, c, act):
    g = torch.Generator(device=cuda).manual_seed(h + c)
    dy = torch.randn(n, 2 * h, 2 * w, c, device=cuda, generator=g)
    a = F.leaky_relu(torch.randn(n, c, h, w, device=cuda, generator=g), SLOPE) if act else None
    dx, sp = ops.upsample2x_backward(dy, act=a, out="both")
    x64 = torch.zeros(n, c, h, w, dtype=torch.float64, device=cuda, requires_grad=True)
    F.interpolate(x64, scale_factor=2, mode="bilinear", align_corners=True).backward(dy.double().permute(0, 3, 1, 2))
    want = x64.grad.permute(0, 2, 3, 1)
    a64 = torch.zeros_like(x64, requires_grad=True)
    F.interpolate(a64, scale_factor=2, mode="bilinear", align_corners=True).backward(dy.double().abs().permute(0, 3, 1, 2))
    bound = a64.grad.permute(0, 2, 3, 1)
    if act:
        dl = _dleaky(a.permute(0, 2, 3, 1))
        want, bound = want * dl, bound * dl
    # the kernel takes the forward's fp32 source coordinates s = r * o (r = (h - 1) / (2h - 1) rounded to fp32, then the
    # product rounded): each blend weight is off by <= 2 U (s + 1) absolutely, so with <= 16 products, their sum and the
    # weights' product, |err| <= (2 U (max(h, w) + 1) * 2 + 24 U) * A
    err = (dx.double() - want).abs()
    lim = (4 * U * (max(h, w) + 1) + 24 * U) * bound
    assert bool((err <= lim + 1e-30).all()), (err / lim.clamp_min(1e-30)).max().item()
    assert _rel(dx, want) < 1e-4
    assert _rel(sp.hi.float() + sp.lo.float(), dx) < 1e-5
    assert torch.equal(dx, ops.upsample2x_backward(dy, act=a))


# ---------------------------------------------------------------------------------------------- modules
def _generator(cuda, hq, seed):
    import importlib
    net = importlib.import_module("model.e2fgvi_hq" if hq else "model.e2fgvi")
    gen = net.InpaintGenerator(init_weights=False).to(cuda)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in gen.named_parameters():
            if name.startswith(("encoder.", "decoder.")):
                # He-scaled weights: activations stay O(1) through the 13 convs
                fan_in = p[0].numel() if p.dim() == 4 else 1
                p.copy_(torch.randn(p.shape, generator=g) * ((2.0 / fan_in) ** 0.5 if p.dim() == 4 else 0.02))
    ops.invalidate_weight_caches()
    return gen


def _sd64(gen):
    return {k: v.detach().double().requires_grad_(True) for k, v in gen.state_dict().items()
            if k.startswith(("encoder.", "decoder.")) and v.dtype == torch.float32}


def _leaky_at(pre, act):
    return pre * torch.where(act > 0, 1.0, float(torch.tensor(SLOPE, dtype=torch.float32)))


def _decoder64(sd, x, dacts):
    """oracle/restate.decoder + tanh in float64 with the GPU forward's LeakyReLU decisions (``dacts``: the three
    LeakyReLU outputs of ``_decode``)."""
    up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=True)  # noqa: E731
    y = _leaky_at(F.conv2d(up(x), sd["decoder.0.conv.weight"], sd["decoder.0.conv.bias"], 1, 1), dacts[0])
    y = _leaky_at(F.conv2d(y, sd["decoder.2.weight"], sd["decoder.2.bias"], 1, 1), dacts[1])
    y = _leaky_at(F.conv2d(up(y), sd["decoder.4.conv.weight"], sd["decoder.4.conv.bias"], 1, 1), dacts[2])
    return torch.tanh(F.conv2d(y, sd["decoder.6.weight"], sd["decoder.6.bias"], 1, 1))


def _decisions(gen, x):
    """The GPU forward's LeakyReLU outputs (their signs are its decisions): encoder convs 0-8, decoder convs 0-2."""
    keep, keep_d = [], []
    with torch.no_grad():
        feat = gen.encoder._forward(x, "f32", keep)
        pred = gen._decode(feat, keep_d)
    enc = [keep[k + 1][-1].hi.float().permute(0, 3, 1, 2) for k in range(len(_ENC) - 1)] + [feat]
    u0, y1, y2, u1, y3 = keep_d
    return feat, pred, enc, [y1.hi.float().permute(0, 3, 1, 2), y2, y3.hi.float().permute(0, 3, 1, 2)]


def _encoder64(sd, x, gen_acts):
    """oracle/restate.encoder in float64 with the GPU forward's LeakyReLU decisions (``gen_acts``: each conv's output
    from the GPU, whose sign selects the slope)."""
    bt = x.size(0)
    out, x0 = x, None
    for k, (stride, groups) in enumerate(restate._ENC):
        if k == 4:
            x0 = out
        if k > 4:
            out = _cat([x0, out], groups)
        out = _leaky_at(F.conv2d(out, sd[f"encoder.layers.{2 * k}.weight"], sd[f"encoder.layers.{2 * k}.bias"], stride,
                                 1, 1, groups), gen_acts[k])
    return out


@pytest.mark.parametrize("hq", [False, True])
def test_encoder_decode_against_float64(cuda, hq):
    gen = _generator(cuda, hq, 5)
    g = torch.Generator().manual_seed(11)
    n, H, W = 2, 48, 80
    x = (torch.rand(n, 3, H, W, generator=g) * 2 - 1).to(cuda)
    target = (torch.rand(n, 3, H, W, generator=g) * 2 - 1).to(cuda)
    feat_ng, pred_ng, acts, dacts = _decisions(gen, x)
    feat = gen.encoder(x)
    assert feat.grad_fn is not None
    check_same_bits(feat, feat_ng, "encoder forward under grad")
    pred = gen.decode(feat)
    check_same_bits(pred, pred_ng, "decode forward under grad")
    loss = (pred - target).abs().mean()
    gen.zero_grad()
    loss.backward()
    sd = _sd64(gen)
    with reference_math():
        p64 = _decoder64(sd, _encoder64(sd, x.double(), acts), dacts)
        (p64 - target.double()).abs().mean().backward()
    assert _rel(pred, p64) < 1e-4
    params = dict(gen.named_parameters())
    for k, v in sd.items():
        assert params[k].grad is not None, k
        assert _rel(params[k].grad, v.grad) < 1e-4, (k, _rel(params[k].grad, v.grad))


def test_frozen_parameters_and_frames(cuda):
    """Only the weights of convs 6, 7, 8 train: the backward is the output's LeakyReLU derivative, per conv one weight
    gradient (GEMM + ordered reduction, no bias kernel) and, above conv 6, one input gradient — 9 launches; no input
    gradient reaches x0 or below, and no frozen parameter gets a weight-gradient kernel."""
    gen = _generator(cuda, False, 6)
    x = (torch.rand(1, 3, 32, 48, device=cuda) * 2 - 1)
    for p in gen.encoder.parameters():
        p.requires_grad_(False)
    for k in (6, 7, 8):
        gen.encoder.layers[2 * k].weight.requires_grad_(True)
    gen.encoder(x).sum().backward()                 # packs the input gradients' weights (cached from here on)
    feat = gen.encoder(x)
    before = ops.launch_count()
    feat.sum().backward()
    assert ops.launch_count() - before == 1 + 3 * 2 + 2, ops.launch_count() - before
    assert all(gen.encoder.layers[2 * k].weight.grad is None for k in range(6))
    assert all(gen.encoder.layers[2 * k].weight.grad is not None for k in (6, 7, 8))
    assert all(gen.encoder.layers[2 * k].bias.grad is None for k in range(9))
    with pytest.raises(ValueError, match="frames"):
        gen.encoder(x.clone().requires_grad_(True))
    # the generator's internal call (last_out="both") stays on the untracked inference path
    out, _ = gen.encoder(x, last_out="both")
    assert out.grad_fn is None


def test_adam_steps_track_float64(cuda):
    gen = _generator(cuda, False, 9)
    g = torch.Generator().manual_seed(2)
    x = (torch.rand(2, 3, 32, 48, generator=g) * 2 - 1).to(cuda)
    target = (torch.rand(2, 3, 32, 48, generator=g) * 2 - 1).to(cuda)
    names = [k for k, _ in gen.named_parameters() if k.startswith(("encoder.", "decoder."))]
    params = dict(gen.named_parameters())
    sd = {k: params[k].detach().double().clone().requires_grad_(True) for k in names}
    # eps above the gradients' scale: Adam's step is then close to linear in the gradient, instead of lr * sign for
    # gradient elements near zero, whose float64 and GPU values may differ in sign within the gradients' tolerance
    opt = torch.optim.Adam([params[k] for k in names], lr=1e-3, eps=1e-2)
    opt64 = torch.optim.Adam(list(sd.values()), lr=1e-3, eps=1e-2)
    for _ in range(3):
        opt.zero_grad()
        _, _, acts, dacts = _decisions(gen, x)
        (gen.decode(gen.encoder(x)) - target).abs().mean().backward()
        opt.step()
        opt64.zero_grad()
        with reference_math():
            (_decoder64(sd, _encoder64(sd, x.double(), acts), dacts) - target.double()).abs().mean().backward()
        opt64.step()
    for k in names:
        assert _rel(params[k], sd[k]) < 1e-4, k
