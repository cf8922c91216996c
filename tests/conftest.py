import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def ctx():
    """One C-ABI context on cuda:0 for the GPU tests.  Fails loudly if the CUDA library/device is missing."""
    from lz4_flex_b200 import block
    c = block.Context(0)
    yield c
    c.close()
