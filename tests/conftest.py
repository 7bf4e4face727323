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
    """CPU oracle (test infrastructure); built on demand with g++."""
    from oracle import ovo_py
    ovo_py.build()
    return ovo_py


@pytest.fixture(scope="session")
def engine_lib():
    from open_vins_b200 import capi
    return capi.load_library()
