import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    cache = {}

    def load(name):
        if name not in cache:
            cache[name] = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
        return cache[name]

    return load
