def compare_ssim(*args, **kwargs):
    raise NotImplementedError("skimage is not installed; the oracle only imports core.metrics for I3D and VFID")
