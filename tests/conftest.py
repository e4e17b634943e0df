import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def ctx():
    """One sdb context on cuda:0 for the whole GPU session (fails loudly without the CUDA library)."""
    from stable_diffusion_burn_b200 import _lib
    c = _lib.Context(0)
    yield c
    c.close()
