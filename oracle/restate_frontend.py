"""TEST INFRASTRUCTURE — numpy restatement of test.py's front end: ``resize_frames`` (PIL bicubic, test.py:98-103) as
Pillow's integer separable resample, and the body of ``read_mask`` (test.py:56-70: NEAREST resize, ``> 0``, 4x cross
dilation).  Both take the product's tables (``e2fgvi_b200.video.bicubic_coeffs`` / ``nearest_index``), so that the
tables are checked against ``PIL.Image.resize`` where Pillow is importable, and the CUDA kernels are checked against
this restatement on a GPU machine that has neither Pillow nor OpenCV.  The goldens of
``oracle/gen_golden_frontend.py`` pin it against the unmodified script.
"""
import numpy as np

from e2fgvi_b200.video import RESAMPLE_BITS, bicubic_coeffs, nearest_index
from oracle.restate_video import dilate_cross


def _pass(img, n_out, axis):
    """One fixed-point pass of Pillow's resample along ``axis`` of a uint8 array."""
    img = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((n_out,) + img.shape[1:], np.int64)
    for i, (first, k) in enumerate(bicubic_coeffs(img.shape[0], n_out)):
        acc = np.full(img.shape[1:], 1 << (RESAMPLE_BITS - 1), np.int64)
        for j, kj in enumerate(k):
            acc += img[first + j] * kj
        assert np.abs(acc).max(initial=0) < 2 ** 31              # Pillow and the kernel sum in int32
        out[i] = np.clip(acc >> RESAMPLE_BITS, 0, 255)
    return np.moveaxis(out.astype(np.uint8), 0, axis)


def resize_bicubic(frames, size):
    """(N,H,W,3) or (H,W,3) uint8 -> resized to ``size = (W', H')``: horizontal pass first into uint8, then vertical;
    a pass whose size is unchanged is skipped."""
    w2, h2 = size
    a = np.asarray(frames)
    h, w = a.shape[-3:-1]
    if w2 != w:
        a = _pass(a, w2, a.ndim - 2)
    if h2 != h:
        a = _pass(a, h2, a.ndim - 3)
    return np.ascontiguousarray(a)


def nearest(masks, size):
    """(N,Hm,Wm) or (Hm,Wm) -> NEAREST-resized to ``size = (W', H')``."""
    w2, h2 = size
    m = np.asarray(masks)
    hm, wm = m.shape[-2:]
    return m[..., list(nearest_index(hm, h2)), :][..., list(nearest_index(wm, w2))]


def read_mask(masks, size):
    """'L' planes (N,Hm,Wm) uint8 -> (N,H',W') uint8 in {0,1}: test.py:62-68 after ``Image.open``."""
    m = (nearest(masks, size) > 0).astype(np.uint8)
    return np.stack([dilate_cross(x) for x in m])
