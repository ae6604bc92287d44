import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure). Built on demand with gcc."""
    from oracle import pyoracle

    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def cuda():
    """Initialised product library on cuda:0; fails loudly when the extension is missing."""
    import torch

    if not torch.cuda.is_available():
        pytest.fail("a gpu-marked test was selected but no CUDA device is present")
    from granite_b200 import capi

    torch.cuda.set_device(0)
    capi.lib()
    capi.init()
    return capi
