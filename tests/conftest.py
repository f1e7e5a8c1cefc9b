import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLD = os.path.join(ROOT, "tests", "golden")
SNAP = os.path.join(ROOT, "headposeestimation-whenet_b200", "data", "whenet_weights.npz")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def sample_crops():
    return np.load(os.path.join(GOLD, "sample_crops.npy"))


@pytest.fixture(scope="session")
def jitter_crops():
    return np.load(os.path.join(GOLD, "jitter_crops.npy"))


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(GOLD, "golden.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def oracle64():
    from whenet_oracle import load_oracle
    return load_oracle(SNAP, np.float64)


@pytest.fixture(scope="session")
def oracle32():
    from whenet_oracle import load_oracle
    return load_oracle(SNAP, np.float32)
