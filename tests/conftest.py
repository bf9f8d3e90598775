import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session")
def native_lib():
    """Build (if needed) and load libposecnn_b200.so."""
    from posecnn_b200.build import build_native
    build_native()
    from posecnn_b200 import _lib
    return _lib.lib()


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from posecnn_b200.build import build_native
    build_native()
    return torch.device("cuda:0")
