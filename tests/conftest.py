import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden():
    import json

    import numpy as np

    d = os.path.join(ROOT, "tests", "golden")
    inputs = dict(np.load(os.path.join(d, "inputs.npz")))
    with open(os.path.join(d, "expected.json")) as f:
        expected = json.load(f)
    return inputs, expected


@pytest.fixture(scope="session")
def accumulator_golden():
    """Merged final rows of the reference's updating-aggregate goldens (tests/golden/make_golden.py)."""
    import json
    with open(os.path.join(ROOT, "tests", "golden", "accumulators.json")) as f:
        return json.load(f)
