import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine with one)")


@pytest.fixture(scope="session")
def nv():
    """The ctypes binding; building the library is the driver's build() step, never done silently here."""
    from lotus_b200 import _native
    _native.lib()
    return _native


@pytest.fixture(scope="session")
def gpu(nv):
    """GPU tests FAIL (not skip) when no H100 is visible: a silent skip would hide a fallback."""
    assert nv.device_count() >= 1, "no sm_90 device visible: -m gpu tests must run on an H100"
    return nv
