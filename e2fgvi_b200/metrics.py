"""evaluate.py's per-frame PSNR and SSIM (reference core/metrics.py:20-54) on the GPU.

``frame_metrics(a, b)`` runs one fused CUDA pass (``csrc/metrics.cu``) over a whole video: per frame the exact sum of
squared errors and skimage 0.16.2's ``compare_ssim(a, b, data_range=255, multichannel=True, win_size=65)`` (uniform
window, sample covariance, the S map cropped by 32 on every side, channel mean).  PSNR is formed on the host from the
SSE with the reference's own expression, ``inf`` included.

Exactness.  evaluate.py's composite is a blend of uint8 frames by at most three windows, so every value is a multiple
of 1/4 in [0, 255].  Then every 65x65 box sum of x, y, x^2, y^2 and xy, and every per-frame sum of (x - y)^2, is a
multiple of 1/16 below 2^43 (1080p included): exact in fp64 in any summation order.  So:

* the SSE is exact, as are numpy's pairwise partial sums, and the PSNR is bit-identical to ``calculate_psnr``;
* the box means are correctly rounded.  scipy's running ``uniform_filter1d`` is not, and the final mean's summation
  order differs, so SSIM agrees with the skimage formulation to within a few units in the last place (<= 2.2e-16 on
  240x432x3 frames), not bit for bit.

Arbitrary fp32 operands get the same fp64 accumulation and land within about 1e-13 of it.

Drop-ins with the reference's signatures: ``calculate_psnr`` and ``calc_psnr_and_ssim`` (numpy in, Python floats out).
"""
import numpy as np
import torch

from . import _lib
from .ops import _need_cuda, _stream

SSIM_WIN = 65          # core/metrics.py:49
DATA_RANGE = 255.0


def _operand(x):
    if x.dtype == torch.uint8:
        return 1
    if x.dtype == torch.float32:
        return 0
    raise TypeError(f"frame_metrics: operands must be uint8 or float32, got {x.dtype}")


def psnr_from_sse(sse, count):
    """``calculate_psnr`` from the exact sum of squared errors of ``count`` values: np.mean's sum / count, then
    ``20 log10(255 / sqrt(mse))``, ``inf`` when the images are equal (float64 scalars, as the reference computes)."""
    mse = np.float64(sse) / count
    if mse == 0:
        return float("inf")
    return 20. * np.log10(255. / np.sqrt(mse))


def frame_metrics(a, b, win_size=SSIM_WIN, data_range=DATA_RANGE):
    """Per-frame PSNR and SSIM of two device tensors (N, H, W, C), each uint8 or float32, C <= 4.

    Returns host float64 arrays ``(psnr, ssim)`` of length N after one device-to-host copy.  SSIM is skimage 0.16.2's
    ``compare_ssim(a[f], b[f], data_range=data_range, multichannel=True, win_size=win_size)``; ``win_size`` must be odd
    and fit the frame (ValueError, as skimage raises).  PSNR uses the reference's constant 255 whatever ``data_range``."""
    n, h, w, c = _shape(a, b)
    if win_size > min(h, w):
        raise ValueError(f"win_size {win_size} exceeds image extent {h}x{w}")
    if win_size % 2 != 1:
        raise ValueError("Window size must be odd.")
    sse, ssim = _run(a, b, win_size, data_range)
    count = h * w * c
    return np.array([psnr_from_sse(s, count) for s in sse]), ssim


def frame_sse(a, b):
    """Per-frame exact sum of squared errors of two device tensors (N, H, W, C), uint8 or float32, C <= 4: a host
    float64 array of length N (no SSIM work; any H, W >= 1)."""
    _shape(a, b)
    return _run(a, b, 0, DATA_RANGE)[0]


def _shape(a, b):
    _need_cuda(a, b)
    if a.shape != b.shape or a.dim() != 4:
        raise ValueError(f"frame_metrics: a and b must both be (N, H, W, C), got {tuple(a.shape)} / {tuple(b.shape)}")
    _operand(a), _operand(b)
    return a.shape


def _run(a, b, win, data_range):
    """``e2f_frame_metrics``: host (sse, ssim) after one copy; win = 0 computes the SSE alone (ssim is then unset)."""
    n, h, w, c = a.shape
    lib = _lib.load()
    elems = lib.e2f_frame_metrics_work_elems(n, h, w, c, win)
    if elems < 0:
        _lib.check(int(elems), "e2f_frame_metrics_work_elems")
    a, b = a.contiguous(), b.contiguous()
    out = torch.empty((2, n), dtype=torch.float64, device=a.device)
    work = torch.empty(elems, dtype=torch.float64, device=a.device)
    st = lib.e2f_frame_metrics(a.data_ptr(), _operand(a), b.data_ptr(), _operand(b), out[0].data_ptr(),
                               out[1].data_ptr() if win else None, work.data_ptr(), n, h, w, c, win,
                               float(data_range), _stream())
    _lib.check(st, "e2f_frame_metrics")
    return out.cpu().numpy()


# ----------------------------------------------------------------------------------------------- drop-ins
def _pair(img1, img2):
    assert img1.shape == img2.shape, (f'Image shapes are differnet: {img1.shape}, {img2.shape}.')
    out = []
    for x in (img1, img2):
        if x.dtype not in (np.uint8, np.float32):
            raise TypeError(f"expected a uint8 or float32 array, got {x.dtype}")
        x = x if x.ndim == 3 else x[..., None]
        out.append(torch.from_numpy(np.ascontiguousarray(x)).cuda().unsqueeze(0))
    return out


def calculate_psnr(img1, img2):
    """``core.metrics.calculate_psnr`` on (H, W) or (H, W, C) images in [0, 255], uint8 or float32 (other dtypes raise
    TypeError).  The difference is taken in float64, as ``calc_psnr_and_ssim`` takes it; the reference's function
    applied directly to uint8 arrays would subtract modulo 256."""
    a, b = _pair(img1, img2)
    return float(psnr_from_sse(frame_sse(a, b)[0], a.numel()))


def calc_psnr_and_ssim(img1, img2):
    """``core.metrics.calc_psnr_and_ssim``: ``(psnr, ssim)`` of two (H, W, C) images in [0, 255], uint8 or float32
    (other dtypes raise TypeError), SSIM with a 65x65 window, so both sides must be at least 65."""
    a, b = _pair(img1, img2)
    psnr, ssim = frame_metrics(a, b)
    return float(psnr[0]), float(ssim[0])
