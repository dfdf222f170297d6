import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    data = dict(np.load(os.path.join(ROOT, "tests", "golden", "distance_golden.npz")))
    # the unexpanded L2 forms have the same exact values as the expanded ones: stored once (tests/golden/make_golden.py)
    for case in ("small", "cfg1"):
        data[f"{case}_L2Unexpanded"] = data[f"{case}_L2Expanded"]
        data[f"{case}_L2SqrtUnexpanded"] = data[f"{case}_L2SqrtExpanded"]
    return data
