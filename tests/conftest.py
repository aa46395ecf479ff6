import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
TESTS_DIR = os.path.dirname(os.path.abspath(__file__))
if TESTS_DIR not in sys.path:
    sys.path.insert(0, TESTS_DIR)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle's function table (test infrastructure)."""
    from oracle import binding
    return binding.load()


@pytest.fixture(scope="session")
def orc_ctx(orc):
    from lvio_fusion_b200 import backend
    return backend.Context(orc)


@pytest.fixture(scope="session")
def lvb():
    """The CUDA library's function table; fails loudly when it is not built."""
    from lvio_fusion_b200 import _capi
    return _capi.load()


@pytest.fixture(scope="session")
def lvb_ctx(lvb):
    from lvio_fusion_b200 import backend
    return backend.Context(lvb)
