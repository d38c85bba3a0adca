import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle
    oracle.lib()
    return oracle


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from paddle3d_b200 import _lib
    _lib.lib()  # must exist on a GPU box: fail loudly, never fall back
    return torch.device("cuda:0")


def golden(name):
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", name))
