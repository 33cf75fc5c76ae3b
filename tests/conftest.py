import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def native_lib():
    """Builds (if stale) and loads libb200_collective.so."""
    from ray_b200 import _native, build

    build.build()
    return _native.load()


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    path = os.path.join(ROOT, "tests", "golden", "collective_golden.npz")
    return np.load(path, allow_pickle=False)
