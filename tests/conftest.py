import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLD = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90a, H100) device")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def gold():
    import numpy as np

    def load(name):
        path = os.path.join(GOLD, name + ".npz")
        if not os.path.exists(path):
            pytest.skip(f"{name}.npz not generated")
        return np.load(path)

    return load
