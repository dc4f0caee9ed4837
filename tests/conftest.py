import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests skip (instead of erroring in the CUDA driver) on a machine without a device.  On a GPU box a missing
    libesr_b200.so is NOT a skip: the tests run and fail loudly in esr_b200._lib (no fallback path exists)."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_events():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "events_golden.npz"))
