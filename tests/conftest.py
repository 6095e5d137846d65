import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


def pytest_sessionstart(session):
    """A fresh checkout has no built artefacts (they are git-ignored): build the CUDA library
    (nvcc cross-compiles without a GPU) and the oracle before the first test.  The product path
    itself never builds or falls back: without the library it raises."""
    from pvnet_b200 import _build
    if not os.path.exists(_build.LIB):
        _build.build()
    from oracle import pvnet_oracle
    pvnet_oracle.build()
