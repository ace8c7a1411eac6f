import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on a machine with an H100)")


@pytest.fixture(scope="session")
def golden_ref():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_numpy.npz"))


@pytest.fixture(scope="session")
def golden_ops():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "oracle_ops.npz"))
