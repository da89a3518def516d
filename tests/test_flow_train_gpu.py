"""H100: the flow-completion backward — SPyNet's 7x7 conv input / weight gradients, the glue's adjoints, the
differentiable ``forward_bidirect_flow`` and ``FlowCompletionLoss`` — against float64 torch autograd."""
import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.synth import synth_frames, synth_spynet_state_dict
from oracle import restate_flow

pytestmark = pytest.mark.gpu


def _rel(got, want):
    return ((got.double() - want.double()).abs().max() / want.double().abs().max().clamp_min(1e-30)).item()


def _l2rel(got, want):
    return ((got.double() - want.double()).norm() / want.double().norm().clamp_min(1e-30)).item()


def _operand(x, layout):
    """(N,C,H,W) fp32 -> the operand layout a SPyNet conv reads: row-gapped with lead 3, or dense split."""
    return ops.pack_rows(x, lead=3) if layout == "rows" else ops.split_nhwc(x)


# (cin, cout) of the forward conv; the input gradient runs cout -> cin
CONVS = [(8, 32), (32, 64), (64, 32), (32, 16), (16, 2)]
SIZES = [(2, 4, 8), (3, 13, 21), (1, 64, 128)]          # (n, h, w): coarsest level, partial tiles, the training size


@pytest.mark.parametrize("cin,cout", CONVS)
@pytest.mark.parametrize("n,h,w", SIZES)
@pytest.mark.parametrize("masked", [False, True])
def test_dgrad_against_float64(cuda, cin, cout, n, h, w, masked):
    g = torch.Generator().manual_seed(cin * 100 + cout + h)
    wt = (torch.randn(cout, cin, 7, 7, generator=g) * 0.05).to(cuda)
    dy = torch.randn(n, cout, h, w, generator=g).to(cuda)
    act = torch.relu(torch.randn(n, cin, h, w, generator=g)).to(cuda) if masked else None
    dy_op = ops.pack_rows(dy, lead=3, cin=max(8, ops.rows_channels(cout))) if cout <= 32 else ops.split_nhwc(dy)
    act_op = None if act is None else _operand(act, "rows" if cin <= 32 else "split")
    out = "rows" if cin <= 32 else "split"
    dx, nxt = ops.conv2d_dgrad(dy_op, wt, act=act_op, out=out)
    want = F.conv_transpose2d(dy.double(), wt.double(), padding=3).permute(0, 2, 3, 1)
    if act is not None:                                  # ReLU's derivative at the saved activation's hi part
        act_hi = act_op.dense().permute(0, 2, 3, 1) if out == "rows" else act_op.hi.float()
        want = want * (act_hi > 0).double()
    assert _rel(dx, want) < 1e-4
    # the bf16 split / row-gapped operand holds dx
    dense = nxt.dense() if out == "rows" else (nxt.hi.float() + nxt.lo.float()).permute(0, 3, 1, 2)
    assert _rel(dense.permute(0, 2, 3, 1), dx) < 1e-5


@pytest.mark.parametrize("cin,cout", CONVS)
@pytest.mark.parametrize("n,h,w", SIZES)
@pytest.mark.parametrize("layout", ["rows", "split"])
def test_wgrad_against_float64(cuda, cin, cout, n, h, w, layout):
    if layout == "rows" and cin > 32:
        pytest.skip("row-gapped operands hold <= 32 channels")
    g = torch.Generator().manual_seed(cin + 7 * cout + w)
    x = torch.randn(n, cin, h, w, generator=g).to(cuda)
    dy = torch.randn(n, h, w, cout, generator=g).to(cuda)
    xo = _operand(x, layout)
    xd = (xo.dense() if layout == "rows" else (xo.hi.float() + xo.lo.float()).permute(0, 3, 1, 2)).double()
    wref = torch.zeros(cout, cin, 7, 7, dtype=torch.float64, device=cuda, requires_grad=True)
    bref = torch.zeros(cout, dtype=torch.float64, device=cuda, requires_grad=True)
    F.conv2d(xd, wref, bref, 1, 3).backward(dy.double().permute(0, 3, 1, 2))
    dw, db = ops.conv2d_wgrad(dy, xo, cin, with_bias=True)
    assert dw.shape == (cout, cin, 7, 7) and db.shape == (cout,)
    assert _rel(dw, wref.grad) < 1e-4
    assert _rel(db, bref.grad) < 1e-4
    dw2, db2 = ops.conv2d_wgrad(dy, xo, cin, with_bias=True)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


def _glue_pyramid(cuda, b, l_t, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    frames = torch.rand(b, l_t, 3, H, W, generator=g).to(cuda)
    mean = torch.tensor([0.485, 0.456, 0.406], device=cuda).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], device=cuda).view(1, 3, 1, 1)
    return ops.spynet_pyramid(frames, l_t, mean, std, unit=True), g


@pytest.mark.parametrize("b,l_t,H,W,k", [(1, 3, 240, 432, 0), (2, 2, 120, 200, 1), (1, 3, 240, 432, 3), (1, 2, 128, 256, 4)])
def test_level_input_backward_against_float64(cuda, b, l_t, H, W, k):
    pyr, g = _glue_pyramid(cuda, b, l_t, H, W, k + H)
    img = pyr.levels[k]
    _, _, hk, wk = img.shape
    P = 2 * b * (l_t - 1)
    # flows of a few pixels: many samples clamp at the border
    prev = (torch.randn(P, hk // 2, wk // 2, 2, generator=g) * 3).to(cuda)
    _, flow_up = ops.spynet_level_input(pyr, k, prev.contiguous())
    d_in = torch.randn(P, hk, wk, 8, generator=g).to(cuda)
    dflow = torch.randn(P, hk, wk, 2, generator=g).to(cuda)
    got = ops.spynet_level_input_backward(d_in, dflow, pyr, k, flow_up)
    # float64 autograd of flow_up = 2 * upsample(prev), warped = flow_warp(supp, flow_up) at the same sample points
    p64 = prev.double().permute(0, 3, 1, 2).requires_grad_(True)
    up = F.interpolate(p64, scale_factor=2, mode="bilinear", align_corners=True) * 2.0
    sup = []
    for p in range(P):
        per_dir = b * (l_t - 1)
        d, q = divmod(p, per_dir)
        bi, j = divmod(q, l_t - 1)
        sup.append(bi * l_t + (j if d else j + 1))
    s = img.double()[sup]
    warped = restate_flow.flow_warp(s, up.permute(0, 2, 3, 1))
    loss = (warped * d_in[..., 3:6].double().permute(0, 3, 1, 2)).sum() + \
        (up * (d_in[..., 6:8] + dflow).double().permute(0, 3, 1, 2)).sum()
    loss.backward()
    want = p64.grad.permute(0, 2, 3, 1)
    # A sample within rounding of an integer coordinate or of the border may legitimately take the other side of the
    # warp's kink in fp32.  Coarse pixels whose gather window (fine rows / columns 2p-3 .. 2p+4) holds no such sample
    # are held to the max-relative bar, elementwise; all of them to an L2 bar.
    gy, gx = torch.meshgrid(torch.arange(hk, device=cuda), torch.arange(wk, device=cuda), indexing="ij")
    iy, ix = gy[None].double() + flow_up[..., 1].double(), gx[None].double() + flow_up[..., 0].double()
    eps = 1e-4
    near = ((ix - ix.round()).abs() < eps) | ((iy - iy.round()).abs() < eps)
    near |= ((ix.abs() < eps) | ((ix - (wk - 1)).abs() < eps) | (iy.abs() < eps) | ((iy - (hk - 1)).abs() < eps))
    near_c = F.max_pool2d(near[:, None].float(), 8, 2, 3)[:, 0] > 0             # (P, hk/2, wk/2)
    far = ~near_c
    assert far.float().mean().item() > 0.9
    err = (got.double() - want).abs().amax(-1)
    assert (err[far].max() / want.abs().max()).item() < 1e-4
    assert _l2rel(got, want) < 1e-4, _l2rel(got, want)
    assert torch.equal(got, ops.spynet_level_input_backward(d_in, dflow, pyr, k, flow_up))


@pytest.mark.parametrize("b,l_t,H,W", [(1, 3, 240, 432), (2, 2, 120, 200), (1, 2, 128, 256)])
def test_final_backward_against_float64(cuda, b, l_t, H, W):
    pyr, g = _glue_pyramid(cuda, b, l_t, H, W, W)
    h, w = pyr.size
    hu, wu = pyr.up
    P = 2 * b * (l_t - 1)
    flow = torch.randn(P, hu, wu, 2, generator=g).to(cuda)
    gf = torch.randn(b, l_t - 1, 2, h, w, generator=g).to(cuda)
    gb = torch.randn(b, l_t - 1, 2, h, w, generator=g).to(cuda)
    got = ops.spynet_final_backward(gf, gb, pyr)
    f64 = flow.double().permute(0, 3, 1, 2).requires_grad_(True)
    r = F.interpolate(f64, size=(h, w), mode="bilinear", align_corners=False)
    r = torch.stack((r[:, 0] * (w / wu), r[:, 1] * (h / hu)), 1)
    (r * torch.cat([gf, gb]).reshape(P, 2, h, w).double()).sum().backward()
    assert _rel(got, f64.grad.permute(0, 2, 3, 1)) < 1e-5


# ------------------------------------------------------------------------------------------------- the module
def _generator(cuda, hq=False, seed=0, flow_scale=1.0):
    import importlib
    net = importlib.import_module("model.e2fgvi_hq" if hq else "model.e2fgvi")
    g = net.InpaintGenerator(init_weights=False)
    sd = synth_spynet_state_dict(seed, prefix="", flow_scale=flow_scale)
    g.update_spynet.load_state_dict(sd)
    return g.to(cuda), sd


def _restate_grads(sd, frames, dfwd, dbwd, slopes=None, record=None):
    dev = frames.device
    params = restate_flow.params_from_state_dict(sd, "", device=dev, requires_grad=True)
    mean, std = sd["mean"].to(dev).double(), sd["std"].to(dev).double()
    f, b = restate_flow.forward_bidirect_flow(params, mean, std, frames.double(), slopes, record)
    ((f * dfwd.double()).sum() + (b * dbwd.double()).sum()).backward()
    return (f, b), params


# (b, l_t, H, W, model, whole): the training size; flows that are not a multiple of 32 (30x50 -> 32x64); the HQ model.
# ``whole``: also run the whole generator (the base model's fold size is fixed to 240x432 frames).
# ``kxn``: the default conv kernels, or E2F_KXN=0's (the convs 3 and 4 then keep row-gapped operands, not dense ones).
@pytest.mark.parametrize("kxn", [True, False])
@pytest.mark.parametrize("b,l_t,H,W,hq,whole", [(1, 3, 240, 432, False, True), (2, 2, 120, 200, False, False),
                                                (1, 3, 120, 216, True, True)])
def test_module_gradients_against_float64(cuda, monkeypatch, b, l_t, H, W, hq, whole, kxn):
    monkeypatch.setattr(ops, "KXN_CONVS", kxn)
    # Flows of about 3 pixels (they still clamp at the border).  The warp's coordinate gradient jumps where a sample
    # crosses an integer coordinate or the border; with flows of tens of pixels a few samples of the finest levels lie
    # within fp32 rounding of such a kink, take the other side than in float64, and that O(1) difference reaches every
    # coarser level's gradient (up to 5e-2 L2-relative at 250-pixel flows).  The per-op test above checks the warp's
    # adjoint at identical sample points.
    g, sd = _generator(cuda, hq, seed=b + l_t, flow_scale=0.25)
    mf = synth_frames(b, l_t + 2, H, W, seed=3).to(cuda)
    frames = (mf[:, :l_t] + 1) / 2
    fwd, bwd = g.forward_bidirect_flow(frames)
    assert fwd.grad_fn is not None
    with torch.no_grad():
        ref_flows = g(mf, l_t)[1] if whole else g.update_spynet.bidirect_flows(mf, l_t)
    assert torch.equal(fwd, ref_flows[0]) and torch.equal(bwd, ref_flows[1])
    gen = torch.Generator().manual_seed(11)
    dfwd = torch.randn(fwd.shape, generator=gen).to(cuda)
    dbwd = torch.randn(bwd.shape, generator=gen).to(cuda)
    torch.autograd.backward([fwd, bwd], [dfwd, dbwd])
    got = [t.grad for lv in g.update_spynet.basic_module for h_ in lv.basic_module for t in (h_.conv.weight, h_.conv.bias)]
    (f64, b64), params = _restate_grads(sd, frames, dfwd, dbwd)
    assert _rel(fwd, f64) < 1e-3 and _rel(bwd, b64) < 1e-3
    want = [t.grad for row in params for pair in row for t in pair]
    plain = [_l2rel(a, w_) for a, w_ in zip(got, want)]
    # The same with the ReLU decisions the GPU forward took (the hi parts of its saved activations): where a
    # pre-activation lies within rounding of 0, fp32 and fp64 legitimately take different sides of the kink
    keep = []
    with torch.no_grad():
        g.update_spynet._bidirect_flows(frames, l_t, True, keep)
    slopes = [[(o.dense() if isinstance(o, ops.RowsNHWC) else o.hi.float().permute(0, 3, 1, 2)) > 0 for o in kept[1][1:]]
              for kept in keep]
    _, params_m = _restate_grads(sd, frames, dfwd, dbwd, slopes=slopes)
    matched = [_l2rel(a, t.grad) for a, t in zip(got, [t for row in params_m for pair in row for t in pair])]
    names = [f"{lv}.{k}.{kind}" for lv in range(6) for k in range(5) for kind in ("w", "b")]
    print(f"max L2-relative error: matched {max(matched):.2e}, plain {max(plain):.2e}")
    if not kxn:
        assert any(isinstance(o, ops.RowsNHWC) for o in keep[-1][1][3:])      # the E2F_KXN=0 operands were exercised
    # The finest level's gradients reach no warp adjoint: with the ReLU decisions matched they are held to 1e-4.  The
    # coarser levels' gradients pass through the finest levels' warps.  Even at these flows a few of the ~65k sample
    # coordinates of the finest level lie within the fp32 / fp64 flow difference (~3e-5 px) of an integer, where the
    # coordinate gradient jumps; that reaches every coarser level as a common error of up to ~1e-3.
    fine = [e for n_, e in zip(names, matched) if n_.startswith("5.")]
    assert max(fine) < 1e-4, {n_: e for n_, e in zip(names, matched) if n_.startswith("5.") and e >= 1e-4}
    assert max(matched) < 2e-3, {n_: e for n_, e in zip(names, matched) if e >= 2e-3}
    assert max(plain) < 2e-2, {n_: e for n_, e in zip(names, plain) if e >= 2e-2}


@pytest.mark.parametrize("case", ["base", "odd", "hq"])
def test_module_against_reference_goldens(cuda, case):
    """forward_bidirect_flow + FlowCompletionLoss + backward against the unmodified reference run in float64
    (oracle/gen_golden_flow.py): flows, loss, and each parameter's gradient projected on 8 fixed vectors."""
    import os

    import numpy as np

    from e2fgvi_b200.loss import FlowCompletionLoss
    from oracle.gen_golden_dis import projections
    from oracle.gen_golden_flow import CASES, frames, weights
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", f"flow_{case}.npz"))
    b, l_t, h, w, hq, seed = CASES[case]
    upd, fix = weights(seed)
    g, _ = _generator(cuda, hq)
    g.update_spynet.load_state_dict(upd)
    loss_fn = FlowCompletionLoss(pretrained=fix).to(cuda)
    masked, gt = frames(b, l_t, h, w, seed)
    pred = g.forward_bidirect_flow(masked.float().to(cuda))
    for got, key in zip(pred, ("flows_forward", "flows_backward")):
        assert _rel(got.detach().cpu(), torch.from_numpy(gold[key])) < 1e-4
    loss = loss_fn(pred, gt.float().to(cuda))
    assert abs(loss.item() - float(gold["loss"])) <= 1e-5 * float(gold["loss"])
    loss.backward()
    errs = {}
    for name, p in g.update_spynet.named_parameters():
        proj = projections(name, p.numel(), seed) @ p.grad.double().cpu().reshape(-1)
        want = torch.from_numpy(gold["g_" + name])
        errs[name] = (proj - want).norm().item() / want.norm().item()
        assert p.grad.abs().max().item() == pytest.approx(float(gold["gmax_" + name]), rel=1e-2), name
    print(f"{case}: worst projected-gradient L2-relative error {max(errs.values()):.2e}")
    # fp32 against float64, ReLU and warp kinks included (see test_module_gradients_against_float64)
    assert max(errs.values()) < 3e-3, {k: v for k, v in errs.items() if v >= 3e-3}
    assert max(v for k, v in errs.items() if k.startswith("basic_module.5.")) < 1e-3


def test_backward_is_deterministic(cuda):
    g, _ = _generator(cuda, seed=5)
    frames = (synth_frames(2, 3, 240, 432, seed=2).to(cuda) + 1) / 2
    runs = []
    for _ in range(2):
        g.zero_grad(set_to_none=True)
        f, b = g.forward_bidirect_flow(frames)
        (f.square().sum() + b.abs().sum()).backward()
        runs.append([p.grad.clone() for p in g.update_spynet.parameters()])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_frozen_and_no_grad_keep_the_inference_launches(cuda):
    g, _ = _generator(cuda, seed=1)
    frames = (synth_frames(1, 3, 240, 432, seed=4).to(cuda) + 1) / 2
    with torch.no_grad():
        g.forward_bidirect_flow(frames)                  # packs the weights once (cached per parameter)
        g.forward_bidirect_flow(frames * 1)
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        f_ng, _ = g.forward_bidirect_flow(frames)
        torch.cuda.synchronize()
        n_nograd = ops.launch_count() - n0
    for p in g.update_spynet.parameters():
        p.requires_grad_(False)
    n0 = ops.launch_count()
    f_fr, _ = g.forward_bidirect_flow(frames)
    n_frozen = ops.launch_count() - n0
    assert f_ng.grad_fn is None and f_fr.grad_fn is None
    assert n_nograd == n_frozen
    for p in g.update_spynet.parameters():
        p.requires_grad_(True)
    g.forward_bidirect_flow(frames)                      # packs the kx-in-N weights once
    n0 = ops.launch_count()
    f_tr, _ = g.forward_bidirect_flow(frames)
    assert ops.launch_count() - n0 == 1 + 6 * 6 + 1     # the fused path: pyramid, per level input + 5 convs, final
    assert f_tr.grad_fn is not None


def test_partly_frozen_launches_no_weight_gradient_for_frozen_convs(cuda):
    g, _ = _generator(cuda, seed=2)
    frames = (synth_frames(1, 3, 120, 216, seed=4).to(cuda) + 1) / 2
    for lv in g.update_spynet.basic_module[:5]:
        for p in lv.parameters():
            p.requires_grad_(False)
    f, b = g.forward_bidirect_flow(frames)
    (f.sum() + b.sum()).backward()                       # packs the input gradients' weights once
    f, b = g.forward_bidirect_flow(frames)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    (f.sum() + b.sum()).backward()
    torch.cuda.synchronize()
    n_bw = ops.launch_count() - n0
    # only the finest level trains: final backward, then per conv wgrad (3 launches) and 4 input gradients + 1 pack
    assert n_bw == 1 + 1 + 5 * 3 + 4, n_bw
    assert all(p.grad is None for lv in g.update_spynet.basic_module[:5] for p in lv.parameters())
    assert all(p.grad is not None for p in g.update_spynet.basic_module[5].parameters())


def test_frames_that_require_grad_raise(cuda):
    g, _ = _generator(cuda)
    frames = ((synth_frames(1, 2, 64, 128, seed=1).to(cuda) + 1) / 2).requires_grad_(True)
    with pytest.raises(ValueError, match="frames"):
        g.forward_bidirect_flow(frames)


def test_generator_forward_stays_untracked(cuda):
    g, _ = _generator(cuda)
    mf = synth_frames(1, 4, 240, 432, seed=1).to(cuda)
    pred, flows = g(mf, 3)
    assert pred.grad_fn is None and flows[0].grad_fn is None and flows[1].grad_fn is None


def test_flow_completion_step_with_adam(cuda):
    from e2fgvi_b200.loss import FlowCompletionLoss
    g, _ = _generator(cuda, seed=3)
    gt_sd = synth_spynet_state_dict(7)                 # a SPyNet state dict, as the reference's checkpoint file
    loss_fn = FlowCompletionLoss(pretrained=gt_sd).to(cuda)
    assert not any(p.requires_grad for p in loss_fn.parameters())
    mf = synth_frames(2, 3, 240, 432, seed=6).to(cuda)
    gt = (synth_frames(2, 3, 240, 432, seed=6, holes=False).to(cuda) + 1) / 2
    optim = torch.optim.Adam(g.update_spynet.parameters(), lr=1e-4)
    pred = g.forward_bidirect_flow((mf + 1) / 2)
    loss = loss_fn(pred, gt)
    # the float64 restatement of the loss
    mean, std = gt_sd["mean"].to(cuda).double(), gt_sd["std"].to(cuda).double()
    want = restate_flow.flow_completion_loss(restate_flow.params_from_state_dict(gt_sd, "", device=cuda), mean, std,
                                             (pred[0].detach().double(), pred[1].detach().double()), gt.double())
    assert abs(loss.item() - want.item()) <= 1e-4 * abs(want.item())
    optim.zero_grad()
    loss.backward()
    before = g.update_spynet.basic_module[5].basic_module[4].conv.weight.detach().clone()
    optim.step()
    assert not torch.equal(before, g.update_spynet.basic_module[5].basic_module[4].conv.weight)
    # the next forward uses the new weights: the packed-weight caches follow optimizer.step()
    again = g.forward_bidirect_flow((mf + 1) / 2)
    with torch.no_grad():
        plain = g(mf, 3)[1]
    assert torch.equal(again[0].detach(), plain[0])
    assert not torch.equal(again[0].detach(), pred[0].detach())


def test_in_place_weight_change_and_second_backward_raise(cuda):
    g, _ = _generator(cuda, seed=1)
    frames = (synth_frames(1, 2, 64, 128, seed=1).to(cuda) + 1) / 2
    f, b = g.forward_bidirect_flow(frames)
    with torch.no_grad():
        g.update_spynet.basic_module[5].basic_module[2].conv.weight.add_(1e-3)      # as an optimizer.step() would
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        (f.sum() + b.sum()).backward()
    f, b = g.forward_bidirect_flow(frames)
    (f.sum() + b.sum()).backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second time"):
        (f.sum() + b.sum()).backward()
