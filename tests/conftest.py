import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built():
    """Make sure the in-tree libraries exist (no-op when they are up to date)."""
    from aprilsam_b200.build import build
    return build()


@pytest.fixture(scope="session")
def m3500(built):
    from aprilsam_b200.harness import PoseGraphData
    return PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))


def golden(name):
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", name))
