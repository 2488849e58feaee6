import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(autouse=True, scope="session")
def _gpu_tests_on_the_host_build():
    """SERFSIM_GPU_TESTS_ON_EMU=1: run the `-m gpu` test FILES against the host-compiled kernels (tests/emu) — a dry run of the
    test code itself on a machine without a GPU (python -m pytest tests -m gpu with that variable set).  It proves nothing about
    the device; it makes sure that what fails on the GPU box is never a typo in a test."""
    if os.environ.get("SERFSIM_GPU_TESTS_ON_EMU"):
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import emu_lib
        from serf_b200 import sim
        sim._LIB = emu_lib.lib()
    yield
