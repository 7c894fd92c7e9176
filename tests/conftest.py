import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "ml-ease_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def fixture_data():
    """examples/sample-data.avro of the reference, decoded by tests/golden/make_golden.py."""
    from oracle import oracle as orc
    d = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    return orc.Csr(d["rowptr"], d["colidx"], d["val"], d["response"], d["weight"], d["offset"], len(d["feature_names"]))


@pytest.fixture(scope="session")
def sklearn_fp():
    return np.load(os.path.join(GOLDEN, "sklearn_fixed_point.npz"))


@pytest.fixture(scope="session")
def frozen():
    return np.load(os.path.join(GOLDEN, "oracle_frozen.npz"))
