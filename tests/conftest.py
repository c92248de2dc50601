import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def lib():
    from gdrnpp_bop2022_b200 import _lib, build

    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.lib()


@pytest.fixture(scope="session")
def dev():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")

