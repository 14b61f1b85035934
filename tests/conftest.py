import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(GOLDEN, "golden_small.npz"))


@pytest.fixture(scope="session")
def g_weights():
    from oracle import cmgan_oracle as O
    return O.load_weights_npz(os.path.join(GOLDEN, "weights_g.npz"))


@pytest.fixture(scope="session")
def d_weights():
    from oracle import cmgan_oracle as O
    return O.load_weights_npz(os.path.join(GOLDEN, "weights_d.npz"))
