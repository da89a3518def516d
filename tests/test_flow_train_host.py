"""CPU: the flow-completion training pieces that need no GPU — argument checks of the new entry points, the input
gradient's transposed weight pack, ``FlowCompletionLoss``'s state dict and weight loading, the float64 restatement."""
import warnings

import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.synth import synth_spynet_state_dict
from oracle import restate, restate_flow


def test_argument_errors_without_gpu(lib):
    # dgrad: null pointers, dy layout, channel counts, leads
    assert lib.e2f_conv2d_dgrad_bf16x3(None, 16, 32, 3, 16, 16, None, 0, 16, None, None, 0, 1, 8, 8, 32, None) == -1
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 32, 3, 16, 16, None, 0, None, None, None, 0, 1, 8, 8, 32, None) == -1
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 32, 2, 16, 16, None, 0, 16, None, None, 0, 1, 8, 8, 32, None) == -1
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 4, 3, 16, 16, None, 0, 16, None, None, 0, 1, 8, 8, 32, None) == -2
    assert b"8, 16 or 32" in lib.e2f_last_error()
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 12, 0, 16, 16, None, 0, 16, None, None, 0, 1, 8, 8, 32, None) == -2
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 32, 3, 16, 16, None, 0, 16, None, None, 0, 1, 8, 8, 128, None) == -2
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 32, 3, 16, 16, None, 0, 16, 16, 16, 3, 1, 8, 8, 64, None) == -2
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 32, 3, 16, 16, 16, 3, 16, None, None, 0, 1, 8, 8, 24, None) == -2   # act
    assert lib.e2f_conv2d_dgrad_bf16x3(16, 16, 32, 3, 16, 16, None, 0, 16, None, None, 3, 1, 8, 8, 32, None) == -1
    assert lib.e2f_conv2d_dgrad_bf16x3(8, 16, 32, 3, 16, 16, None, 0, 16, None, None, 0, 1, 8, 8, 32, None) == -3
    # wgrad
    assert lib.e2f_conv2d_wgrad_work_elems(1, 8, 8, 12, 32) == -1
    assert lib.e2f_conv2d_wgrad_work_elems(1, 8, 8, 32, 2) == -1
    assert lib.e2f_conv2d_wgrad_work_elems(4, 64, 128, 32, 64) > 0
    assert lib.e2f_conv2d_wgrad_bf16x3(16, 16, 16, 0, 16, None, None, 1, 8, 8, 32, 64, None) == -1      # no workspace
    assert lib.e2f_conv2d_wgrad_bf16x3(16, 16, 16, 3, 16, None, 16, 1, 8, 8, 64, 64, None) == -1       # rows: cin <= 32
    assert lib.e2f_conv2d_wgrad_bf16x3(16, 16, 16, 3, 16, None, 16, 1, 8, 8, 24, 64, None) == -1       # rows: 8/16/32
    assert lib.e2f_conv2d_wgrad_bf16x3(8, 16, 16, 0, 16, None, 16, 1, 8, 8, 32, 64, None) == -3
    # glue
    assert lib.e2f_spynet_pyramid_unit(None, 16, 1, 3, 3, 240, 432, 60, 108, 64, 128, 16, 16, None) == -1
    assert lib.e2f_spynet_pyramid_unit(16, 16, 1, 3, 3, 240, 432, 60, 108, 60, 128, 16, 16, None) == -1
    assert lib.e2f_spynet_level_input_backward(16, 16, 16, 16, None, 1, 3, 64, 128, None) == -1
    assert lib.e2f_spynet_level_input_backward(16, 16, 16, 16, 16, 1, 3, 63, 128, None) == -1
    assert lib.e2f_spynet_level_input_backward(16, 16, 16, 16, 16, 1, 1, 64, 128, None) == -1
    assert lib.e2f_spynet_level_input_backward(16, 12, 16, 16, 16, 1, 3, 64, 128, None) == -3
    assert lib.e2f_spynet_final_backward(16, None, 16, 1, 3, 60, 108, 64, 128, None) == -1
    assert lib.e2f_spynet_final_backward(16, 16, 16, 1, 3, 60, 108, 32, 128, None) == -1
    assert lib.e2f_spynet_final_backward(16, 16, 12, 1, 3, 60, 108, 64, 128, None) == -3


@pytest.mark.parametrize("cout,cin", [(2, 16), (16, 32), (32, 64), (64, 32), (32, 8)])
def test_dgrad_weight_is_the_transposed_flipped_kernel(cout, cin):
    """Wt[ci][co][ky][kx] = W[co][ci][6 - ky][6 - kx]: conv(dY, Wt, pad 3) is the input gradient of conv(X, W, pad 3)."""
    w = torch.randn(cout, cin, 7, 7, dtype=torch.float64)
    wt = ops.conv_dgrad_weight(w.float()).double()
    assert wt.shape == (cin, cout, 7, 7)
    assert wt[cin - 1, 0, 1, 5].item() == pytest.approx(w[0, cin - 1, 5, 1].item(), rel=1e-6)
    x = torch.randn(2, cin, 9, 11, dtype=torch.float64, requires_grad=True)
    dy = torch.randn(2, cout, 9, 11, dtype=torch.float64)
    F.conv2d(x, w, None, 1, 3).backward(dy)
    assert torch.allclose(F.conv2d(dy, wt, None, 1, 3), x.grad, rtol=1e-6, atol=1e-6 * x.grad.abs().max().item())


def test_flow_completion_loss_state_dict_and_loading(tmp_path):
    from e2fgvi_b200.loss import FlowCompletionLoss
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        plain = FlowCompletionLoss()
    assert any("untrained" in str(w_.message) for w_ in rec)
    keys = set(plain.state_dict())
    # the reference's layout: fix_spynet.basic_module.{0..5}.basic_module.{0..4}.conv.{weight,bias} + mean / std
    want = {f"fix_spynet.basic_module.{lv}.basic_module.{k}.conv.{n}" for lv in range(6) for k in range(5)
            for n in ("weight", "bias")} | {"fix_spynet.mean", "fix_spynet.std"}
    assert keys == want
    assert not any(p.requires_grad for p in plain.parameters())
    sd = synth_spynet_state_dict(3)
    # a checkpoint file as mmcv saves it: {"state_dict": {"module.<key>": ...}}
    path = tmp_path / "spynet.pth"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, path)
    loaded = FlowCompletionLoss(pretrained=str(path))
    for k, v in sd.items():
        assert torch.equal(loaded.fix_spynet.state_dict()[k], v)
    assert torch.equal(FlowCompletionLoss(pretrained=sd).fix_spynet.basic_module[2].basic_module[1].conv.weight,
                       sd["basic_module.2.basic_module.1.conv.weight"])
    with pytest.raises(RuntimeError):
        FlowCompletionLoss(pretrained={k: v for k, v in sd.items() if "basic_module.5" not in k})   # strict
    with pytest.raises(ValueError, match="URL"):
        FlowCompletionLoss(pretrained="https://example.invalid/spynet.pth")


def test_restatement_matches_the_oracle_forward():
    """restate_flow's SPyNet (grid_sample warp) equals the oracle's (explicit gather) in float64."""
    sd = {"update_spynet." + k: v.double() for k, v in synth_spynet_state_dict(1).items()}
    frames = torch.rand(1, 3, 3, 128, 256, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    want = restate.bidirect_flow(sd, frames)
    params = restate_flow.params_from_state_dict(sd, "update_spynet")
    got = restate_flow.forward_bidirect_flow(params, sd["update_spynet.mean"], sd["update_spynet.std"], frames)
    for a, b in zip(got, want):
        assert (a - b).abs().max().item() <= 1e-9 * b.abs().max().item()


def test_restatement_slopes_replace_relu_derivative():
    x = torch.tensor([-1.0, 0.5, 2.0], dtype=torch.float64, requires_grad=True)
    y = restate_flow._ReluWithSlopes.apply(x, torch.tensor([1.0, 0.0, 1.0], dtype=torch.float64))
    y.sum().backward()
    assert torch.equal(y.detach(), F.relu(x.detach()))
    assert x.grad.tolist() == [1.0, 0.0, 1.0]


# ------------------------------------------------------------------------------------- against the reference's goldens
import json  # noqa: E402
import os  # noqa: E402

import numpy as np  # noqa: E402

from oracle.gen_golden_dis import projections  # noqa: E402
from oracle.gen_golden_flow import CASES, frames, weights  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_loss_layout_matches_reference():
    from e2fgvi_b200.loss import FlowCompletionLoss
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sd = FlowCompletionLoss().state_dict()
    with open(os.path.join(GOLDEN, "flow_layout.json")) as f:
        want = json.load(f)
    assert [[k, list(v.shape)] for k, v in sd.items()] == want


@pytest.mark.parametrize("case", sorted(CASES))
def test_restatement_matches_reference_goldens(case):
    """oracle/restate_flow.py (float64) reproduces the unmodified reference's flows, loss and gradients."""
    gold = np.load(os.path.join(GOLDEN, f"flow_{case}.npz"))
    b, l_t, h, w, hq, seed = CASES[case]
    upd, fix = weights(seed)
    masked, gt = frames(b, l_t, h, w, seed)
    params = restate_flow.params_from_state_dict(upd, "", requires_grad=True)
    mean, std = upd["mean"].double(), upd["std"].double()
    f, bw = restate_flow.forward_bidirect_flow(params, mean, std, masked)
    for got, key in ((f, "flows_forward"), (bw, "flows_backward")):
        want = torch.from_numpy(gold[key]).double()
        assert (got.detach() - want).abs().max().item() <= 1e-6 * want.abs().max().item()
    loss = restate_flow.flow_completion_loss(restate_flow.params_from_state_dict(fix, ""), mean, std, (f, bw), gt)
    assert abs(loss.item() - float(gold["loss"])) <= 1e-12 * abs(float(gold["loss"]))
    loss.backward()
    for lv in range(6):
        for k in range(5):
            for i, kind in enumerate(("weight", "bias")):
                name = f"basic_module.{lv}.basic_module.{k}.conv.{kind}"
                grad = params[lv][k][i].grad
                proj = projections(name, grad.numel(), seed) @ grad.reshape(-1)
                want = torch.from_numpy(gold["g_" + name])
                assert (proj - want).norm().item() <= 1e-9 * want.norm().item() + 1e-300, name
                assert grad.abs().max().item() == pytest.approx(float(gold["gmax_" + name]), rel=1e-9)
