"""CPU: the C-ABI library builds, loads and exports every symbol include/e2fgvi_b200.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "e2fgvi_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(e2f_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree(lib):
    from e2fgvi_b200 import _lib
    assert _declared() == sorted(_lib.SIGNATURES)
    for name in _declared():
        assert hasattr(lib, name)


def test_version_and_error_string(lib):
    assert b"sm_90a" in lib.e2f_version()
    assert isinstance(lib.e2f_last_error(), bytes)


def test_argument_errors_without_gpu(lib):
    """Validation happens before any CUDA call, so it is testable on a CPU-only box."""
    assert lib.e2f_flow_warp(None, None, None, 1, 4, 4, 8, 0, 0, None) == -1
    assert b"null" in lib.e2f_last_error()
    assert lib.e2f_flow_warp(16, 16, 16, 1, 4, 4, 6, 0, 0, None) == -2          # C not a vector multiple
    assert lib.e2f_flow_warp(16, 16, 16, 1, 4, 4, 8, 7, 0, None) == -1          # bad dtype
    assert lib.e2f_flow_warp(8, 16, 16, 1, 4, 4, 8, 0, 0, None) == -3           # misaligned
    assert lib.e2f_focal_window_attention(16, 16, 16, 1, 2, 10, 18, 4, 64, 5, 9, 2, 4, 5, 9, 1, 0.1, 0, None) == -2
    assert lib.e2f_focal_window_attention(16, 16, 16, 1, 2, 11, 18, 4, 128, 5, 9, 2, 4, 5, 9, 1, 0.1, 0, None) == -1
    assert lib.e2f_modulated_deform_conv2d(32, 16, 16, 128, None, 16, 1, 4, 4, 64, 128, 16, 0, 0, None) == -2
    assert b"specialised" in lib.e2f_last_error()


def test_argument_errors_new_entry_points(lib):
    """Video-driver and propagation-prologue entry points validate before any CUDA call."""
    assert lib.e2f_video_prepare_clip(None, 16, 16, 16, 2, 8, 8, 60, 108, None) == -1
    assert lib.e2f_video_prepare_clip(16, 16, 16, 16, 2, 100, 200, 240, 216, None) == -1      # hp > 2h: not a mirror pad
    assert b"mirror" in lib.e2f_last_error()
    assert lib.e2f_video_compose(16, 16, 16, 16, None, 1, 8, 8, 60, 108, None) == -1
    assert lib.e2f_video_blend(16, 16, 16, 16, 1, 0, None) == -1
    assert lib.e2f_video_finalize(16, None, 10, None) == -1
    args = [16, 16, 16, 0, 16, 0] + [16] * 9
    assert lib.e2f_prop_prologue(*args, 1, 4, 4, 24, None) == -1                             # C % 16
    assert lib.e2f_prop_prologue(16, None, 16, 0, 16, 0, *[16] * 9, 1, 4, 4, 32, None) == -1   # feat_n2 without flow_prev
    assert b"both" in lib.e2f_last_error()
    assert lib.e2f_prop_prologue(8, 16, 16, 0, 16, 0, *[16] * 9, 1, 4, 4, 32, None) == -3      # misaligned prop


def test_conv_launcher_rejections_without_gpu(lib):
    """The conv launchers' own shape checks come before the driver is asked to encode a tensor map."""
    src = (ctypes.c_void_p * 1)(16)
    channels = (ctypes.c_int * 1)(64)
    # kx-in-N conv: only 3x3 and 7x7 kernels
    assert lib.e2f_conv_kxn_bf16x3(1, src, src, channels, 16, 16, None, None, 16, None, None,
                                   1, 8, 32, 32, 1, 32, 5, 1.0, 0, None) == -2
    assert b"conv_kxn: unsupported shape" in lib.e2f_last_error()
    # generic conv: the bias is staged in shared memory for at most 512 output channels
    assert lib.e2f_conv2d_rows_bf16x3(1, src, src, channels, 0, 16, 16, None, None, None, 16, 16, 0,
                                      1, 8, 16, 520, 1, 1.0, 3, 1, 1, None) == -2
    assert b"at most 512 output channels" in lib.e2f_last_error()


def test_no_cpu_fallback():
    import torch
    from e2fgvi_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.flow_warp(torch.zeros(1, 8, 4, 4), torch.zeros(1, 4, 4, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.modulated_deform_conv2d(torch.zeros(1, 256, 4, 4), torch.zeros(1, 288, 4, 4), torch.zeros(1, 144, 4, 4),
                                    torch.zeros(128, 256, 3, 3), None, 1, 1, 1, 1, 16)
