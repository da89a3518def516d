"""TEST INFRASTRUCTURE — a restatement of scikit-image 0.16.2's ``skimage.measure.compare_ssim`` for the arguments
the reference's ``core.metrics.calc_psnr_and_ssim`` passes (``data_range=255, multichannel=True, win_size=65``):
uniform window (``scipy.ndimage.uniform_filter``, its default ``reflect`` mode), sample covariance, per-channel mean
of the S map cropped by ``(win_size - 1) // 2``, then the mean over channels; and the library's ``ValueError``s for
mismatched shapes, a window larger than the image and an even window.  Any other option (``gaussian_weights``,
``full``, ``gradient``, non-default constants, ``data_range=None``) raises NotImplementedError.

scikit-image 0.16.2 is not part of this project's environment, so this is what SSIM is checked against.
"""
import numpy as np
from scipy.ndimage import uniform_filter


def compare_ssim(X, Y, win_size=None, gradient=False, data_range=None, multichannel=False, gaussian_weights=False,
                 full=False, **kwargs):
    if not X.shape == Y.shape:
        raise ValueError("Input images must have the same dimensions.")
    if gradient or full or gaussian_weights:
        raise NotImplementedError("only the uniform-window mean SSIM is restated (no gradient, full or gaussian_weights)")
    if multichannel:
        mssim = np.empty(X.shape[-1])
        for ch in range(X.shape[-1]):
            mssim[ch] = compare_ssim(X[..., ch], Y[..., ch], win_size=win_size, data_range=data_range, **kwargs)
        return mssim.mean()
    if kwargs.get("K1", 0.01) != 0.01 or kwargs.get("K2", 0.03) != 0.03 or \
            not kwargs.get("use_sample_covariance", True) or set(kwargs) - {"K1", "K2", "use_sample_covariance"}:
        raise NotImplementedError(f"options {sorted(kwargs)} are not restated")
    if win_size is None:
        win_size = 7
    if np.any((np.asarray(X.shape) - win_size) < 0):
        raise ValueError("win_size exceeds image extent.  If the input is a multichannel (color) image, set "
                         "multichannel=True.")
    if not (win_size % 2 == 1):
        raise ValueError("Window size must be odd.")
    if data_range is None:
        raise NotImplementedError("data_range=None (the dtype's range) is not restated")

    X = X.astype(np.float64)
    Y = Y.astype(np.float64)
    NP = win_size ** X.ndim
    cov_norm = NP / (NP - 1)
    ux = uniform_filter(X, size=win_size)
    uy = uniform_filter(Y, size=win_size)
    uxx = uniform_filter(X * X, size=win_size)
    uyy = uniform_filter(Y * Y, size=win_size)
    uxy = uniform_filter(X * Y, size=win_size)
    vx = cov_norm * (uxx - ux * ux)
    vy = cov_norm * (uyy - uy * uy)
    vxy = cov_norm * (uxy - ux * uy)
    R = data_range
    C1 = (0.01 * R) ** 2
    C2 = (0.03 * R) ** 2
    A1, A2, B1, B2 = (2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2)
    S = (A1 * A2) / (B1 * B2)
    pad = (win_size - 1) // 2
    return S[tuple(slice(pad, n - pad) for n in S.shape)].mean()


def calc_psnr_and_ssim(img1, img2):
    """``core.metrics.calc_psnr_and_ssim`` with this restatement as its SSIM."""
    img1 = img1.astype(np.float64)
    img2 = img2.astype(np.float64)
    assert img1.shape == img2.shape
    mse = np.mean((img1 - img2) ** 2)
    psnr = float("inf") if mse == 0 else 20. * np.log10(255. / np.sqrt(mse))
    return psnr, compare_ssim(img1, img2, data_range=255, multichannel=True, win_size=65)
