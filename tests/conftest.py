import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90)")


@pytest.fixture(scope="session")
def sb():
    """The product package (CUDA path through the C ABI)."""
    import stheno_jl_b200
    return stheno_jl_b200


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (checker only)."""
    from oracle import stheno_oracle
    return stheno_oracle
