import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def live_golden(golden_dir):
    """What the reference's own classes computed on a test's scenario (tests/golden/live_<name>.npz, oracle/make_golden.py)."""
    def load(name):
        return np.load(os.path.join(golden_dir, "live_" + name + ".npz"))

    return load
