import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def lib():
    """Build (if needed) and load libvitb200.so."""
    from vit_tensorflow_b200 import build, _lib
    build.build()
    return _lib.load()
