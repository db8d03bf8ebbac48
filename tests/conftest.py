import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    pyoracle.lib()
    return pyoracle


@pytest.fixture(scope="session")
def vb():
    """The product library, initialised on cuda:0.  GPU tests only."""
    import libvips_b200 as vb
    vb.init(0)
    return vb
