import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def b2m_ctx():
    """One libb2m context on cuda:0 for the whole session (GPU tests only)."""
    import ctypes

    from marlin_b200 import _lib

    L = _lib.lib()
    h = ctypes.c_void_p()
    _lib.check(L.b2m_ctx_create(0, ctypes.byref(h)))
    yield h
    L.b2m_ctx_destroy(h)
