"""CPU: host-side logic of tools/train_bench.py (no GPU): every stage parses, refuses to run without a GPU, keeps the
default shape and step counts its README table states, counts the README's algorithmic work at that shape, and leaves
the TF32 flags as it found them."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "tools", "train_bench.py")
sys.path.insert(0, os.path.join(ROOT, "tools"))

import train_bench as tb  # noqa: E402

DEFAULTS = {
    "dis": dict(batch=8, frames=8, height=240, width=432, iters=20, warmup=5),
    "flow": dict(batch=8, local=5, height=240, width=432, iters=20, warmup=5),
    "encdec": dict(clips=8, frames=8, height=240, width=432, iters=20, warmup=5),
    "ffn": dict(clips=8, frames=8, height=60, width=108, iters=20, warmup=5),
    "attn": dict(clips=8, frames=8, height=20, width=36, iters=10, warmup=3),
    "block": dict(clips=8, frames=8, iters=10, warmup=3),
    "align": dict(n=8, iters=10, warmup=3),
    "prop": dict(b=8, t=5, iters=10, warmup=3),
}


def test_every_stage_is_listed():
    assert list(tb.STAGES) == list(DEFAULTS)


@pytest.mark.parametrize("stage", list(DEFAULTS))
def test_help_exits_zero(stage):
    r = subprocess.run([sys.executable, SCRIPT, stage, "--help"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and f"train_bench.py {stage}" in r.stdout, r.stderr


@pytest.mark.parametrize("stage", list(DEFAULTS))
def test_defaults(stage):
    a = vars(tb.parse_args([stage]))
    assert a.pop("stage") == stage and a.pop("profile") is False and a.pop("out") is None
    assert a == DEFAULTS[stage]


@pytest.mark.parametrize("stage", list(DEFAULTS))
def test_no_gpu_times_nothing(stage):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, SCRIPT, stage], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 2, r.stderr
    assert "nothing was timed" in r.stderr and r.stdout == ""


def test_work_at_default_shapes():
    a = tb.parse_args(["dis"])
    dis, gen = tb.dis_flops(a.batch, a.frames, a.height, a.width)
    assert round(dis / 1e9, 2) == 2137.47 and round(gen / 1e9, 2) == 728.21
    assert round(tb.flow_flop(64, 64, 128) / 1e9, 2) == 1341.30          # 64 pairs at 64x128
    a = tb.parse_args(["encdec"])
    fwd, bwd = tb.encdec_flops(a.height, a.width)
    assert round(fwd / 1e9, 3) == 75.456 and round(bwd / 1e9, 3) == 150.822
    a = tb.parse_args(["ffn"])
    tokens = a.clips * a.frames * ((a.height - 1) // 3 + 1) * ((a.width - 1) // 3 + 1)
    fwd, bwd = tb.ffn_flops(tokens)
    assert tokens == 46080 and round(fwd / 1e12, 5) == 0.77687 and round(bwd / 1e12, 5) == 1.25779
    a = tb.parse_args(["attn"])
    fwd, bwd = tb.attn_flops(a.clips, a.frames, a.height, a.width)
    assert round(fwd / 1e12, 5) == 0.25679 and round(bwd / 1e12, 5) == 0.59286
    a = tb.parse_args(["block"])
    assert tb.block_bytes(a.clips, a.frames) == {"layernorm_backward_kernel": 471_859_200,
                                                 "layernorm_pool_backward_kernel": 379_584_512}


@pytest.mark.parametrize("before", [(False, True), (True, False), (False, False), (True, True)])
def test_tf32_flags_come_back(before):
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = before
        for on in (False, True):
            with tb.tf32(on):
                assert (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32) == (on, on)
            assert (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32) == before
        with pytest.raises(RuntimeError), tb.tf32(not before[0]):
            raise RuntimeError("a step failed")
        assert (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32) == before
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
