import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "deep-neuroevolution_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(GOLDEN, "ref_numpy.npz"))


@pytest.fixture(scope="session")
def small_noise():
    """400k-element prefix of the reference noise table (es.py:54-60, seed 123)."""
    from oracle import oracle
    return oracle.noise_table(400_000)
