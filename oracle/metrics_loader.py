"""Import the UNMODIFIED reference's ``core.metrics`` (InceptionI3d, calculate_vfid, ...) from the reference root.

Its imports of scikit-image, matplotlib and torchvision are served by ``metrics_shim`` (import-only stand-ins; the
I3D and VFID code never calls them).  Only usable where the reference is present."""
import importlib
import os
import sys

from .reference_loader import REFERENCE_ROOT, ReferenceUnavailable

SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "metrics_shim")
_SHADOWED = ("core", "skimage", "matplotlib", "torchvision")


def available():
    return os.path.isfile(os.path.join(REFERENCE_ROOT, "core", "metrics.py"))


def _ours(k):
    return any(k == p or k.startswith(p + ".") for p in _SHADOWED)


def import_metrics():
    """The reference's ``core.metrics`` module; the shim modules are removed from ``sys.modules`` afterwards."""
    if not available():
        raise ReferenceUnavailable(f"{REFERENCE_ROOT} is not present")
    saved_path = list(sys.path)
    saved = {k: v for k, v in sys.modules.items() if _ours(k)}
    for k in saved:
        del sys.modules[k]
    sys.path[:] = [SHIM, REFERENCE_ROOT] + saved_path
    try:
        mod = importlib.import_module("core.metrics")
        mod.__reference_modules__ = {k: v for k, v in sys.modules.items() if _ours(k)}
    finally:
        sys.path[:] = saved_path
        for k in list(sys.modules):
            if _ours(k):
                del sys.modules[k]
        sys.modules.update(saved)
    assert os.path.abspath(mod.__file__).startswith(os.path.abspath(REFERENCE_ROOT)), mod.__file__
    return mod
