import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build product + checker libraries once (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def sort_model():
    return open(os.path.join(GOLDEN, "sort6_model.bin"), "rb").read()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_bits_equal(a, b, what=""):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    ne = np.nonzero(a.view(np.uint8).reshape(-1) != b.view(np.uint8).reshape(-1))[0]
    assert ne.size == 0, f"{what}: {ne.size} differing bytes, first at byte {ne[:4]}"
