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
    from tests import support
    return support.Oracle()


@pytest.fixture(scope="session")
def hostcore():
    from tests import support
    return support.HostCore()


@pytest.fixture(params=["thread", "wide"])
def kernel_choice(request, monkeypatch):
    """Run a GPU test once per kernel family: LBFT_FORCE_KERNEL (read by lbft_create) overrides the host's automatic choice
    between the thread-per-instance and the warp-per-instance kernel."""
    monkeypatch.setenv("LBFT_FORCE_KERNEL", request.param)
    return request.param
