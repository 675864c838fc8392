import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def golden(name):
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def golden_loader():
    return golden
