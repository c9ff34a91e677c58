import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real CUDA device (run with -m gpu on a machine with an H100)")


@pytest.fixture(scope="session")
def oracle():
    import oracle_py
    return oracle_py.load()


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def abb():
    """the CUDA library through its ctypes binding; builds it if needed (nvcc, no GPU required)"""
    from abyss_b200 import build
    build.build()
    from abyss_b200 import capi
    capi.load()
    return capi
