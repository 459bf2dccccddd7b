import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (H100, sm_90a)")


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


@pytest.fixture
def golden():
    return load_golden


def rel_err(a, b):
    """max|a-b| / max|b| -- the tolerance definition of SURVEY App. A.5."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))
