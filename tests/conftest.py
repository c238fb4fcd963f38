import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "make-a-scene_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def rel_err(a, b, floor=1e-5):
    """norm-wise relative error ||a-b|| / max(||b||, floor*sqrt(numel)): quantities that are mathematically zero
    (e.g. the key-bias gradient of a softmax attention) are compared on an absolute 1e-5-per-element scale."""
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).norm() / max(float(b.norm()), floor * b.numel() ** 0.5))
