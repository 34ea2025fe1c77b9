import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def built():
    """Builds (or reuses) the in-tree shared objects and the C oracle; returns the package."""
    import __graft_entry__
    __graft_entry__.build()
    import libjpeg_b200
    return libjpeg_b200


@pytest.fixture(scope="session")
def oracle(built):
    from tests import oracle_binding
    return oracle_binding.load()
