import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def lib_built():
    """Build (or reuse) libidxtts.so — nvcc cross-compiles without a GPU."""
    import __graft_entry__ as ge
    ge.build()
    return ge.LIB


@pytest.fixture(scope="session")
def engine(lib_built):
    from indextts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()
