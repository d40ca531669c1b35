import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLD = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")
    config.addinivalue_line("markers", "gpu_staged: GPU test of a path that has not had its first H100 run yet; skipped without a "
                                       "device and NOT selected by `-m gpu` (run with `-m gpu_staged`, then promote it to `gpu`)")


@pytest.fixture(scope="session")
def gold():
    import numpy as np

    return {n[:-4]: np.load(os.path.join(GOLD, n)) for n in os.listdir(GOLD) if n.endswith(".npz")}
