import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def cuda_lib():
    import torch

    from magicdrive_b200 import _lib
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    L = _lib.lib()
    assert L.mdb_device_ok() == 1, "C-ABI library loaded but no sm_90 device usable"
    return L
