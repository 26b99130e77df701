import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a)")


@pytest.fixture(scope="session")
def oracle():
    from oracle.oracle import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def ref():
    """The reference's own compiled CPU code (oracle/_ref). Skips if it has not been built."""
    from oracle.oracle import Ref
    try:
        return Ref()
    except (FileNotFoundError, OSError) as e:
        pytest.skip(f"oracle/_ref unavailable: {e}")
