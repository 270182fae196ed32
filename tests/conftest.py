import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _build_checkers():
    """The CPU checkers (oracle/) are test infrastructure; build them once per session if missing."""
    from oracle import oracle

    if not os.path.exists(os.path.join(ROOT, "oracle", "libtinympc_oracle.so")):
        oracle.build()
    yield
