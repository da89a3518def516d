import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def lib():
    """The built C-ABI library (built on demand; nvcc cross-compiles without a GPU)."""
    from e2fgvi_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from e2fgvi_b200 import build
    build.build()
    return torch.device("cuda:0")
