import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    pyoracle.lib()
    return pyoracle


@pytest.fixture(scope="session")
def svs():
    """The product library through its C ABI.  Fails loudly when it is not built."""
    from scavislam_b200 import capi
    capi.lib()
    return capi
