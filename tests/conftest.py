import os
import subprocess
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def oracle():
    """ctypes handle of the CPU oracle (built on demand; it is test infrastructure)."""
    from tests import orc
    return orc.load()
