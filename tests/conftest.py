import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real GPU, an H100 (run with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure libcno.so and the oracle exist (normally built by __graft_entry__.build())."""
    from cppnumericalsolvers_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from cppnumericalsolvers_b200 import build
        build.build()
    from oracle import oracle_binding as ob
    if not os.path.exists(ob.ORACLE_LIB):
        ob.build()
    yield
