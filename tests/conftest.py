import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    data = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    meta = json.load(open(os.path.join(GOLDEN, f"{name}.json")))
    return data, meta


@pytest.fixture(scope="session")
def golden_contract():
    return load_golden("contract")


@pytest.fixture(scope="session")
def golden_decomp():
    return load_golden("decomp")


@pytest.fixture(scope="session")
def golden_mps():
    return load_golden("mps_dmrg")


@pytest.fixture(scope="session")
def golden_decomp2():
    return load_golden("decomp2")


@pytest.fixture(scope="session")
def golden_boundary():
    return load_golden("boundary")


@pytest.fixture(scope="session")
def golden_tebd():
    return load_golden("tebd")


@pytest.fixture(scope="session")
def golden_mps_ops():
    return load_golden("mps_ops")


@pytest.fixture(scope="session")
def golden_decomp3():
    return load_golden("decomp3")
