"""Import-only stand-in for scikit-image: the reference's core/metrics.py imports ``skimage.measure`` (for SSIM, which
the I3D / VFID code never calls)."""
