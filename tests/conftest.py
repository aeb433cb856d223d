import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def _arr(d):
    return np.asarray(d["data"], dtype=np.float64).reshape(d["shape"])


@pytest.fixture(scope="session")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "reference_kats.json")) as fh:
        raw = json.load(fh)
    return raw


@pytest.fixture(scope="session")
def arr():
    return _arr
