import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session")
def oracle_mod():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def lib():
    import __graft_entry__ as g
    g.build()
    from limbo_b200 import _lib
    return _lib.load()
