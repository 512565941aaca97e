"""pytest configuration: the `gpu` marker selects tests that need an H100 (`-m gpu`)."""

import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); everything else must pass on a CPU-only host")
    config.addinivalue_line("markers", "unvalidated: new GPU test that has not passed on an H100 yet -- skipped unless MORL_RUN_UNVALIDATED=1, "
                                       "so that a bring-up failure cannot take the validated suite down with it; the marker is removed once it has passed")


def pytest_collection_modifyitems(config, items):
    if os.environ.get("MORL_RUN_UNVALIDATED", "0") == "1":
        return
    skip = pytest.mark.skip(reason="not yet validated on an H100 (set MORL_RUN_UNVALIDATED=1 to run)")
    for item in items:
        if "unvalidated" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    path = os.path.join(ROOT, "tests", "golden", "operators.npz")
    return np.load(path, allow_pickle=False)


@pytest.fixture(scope="session")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("this test is marked gpu and requires a CUDA device; there is no CPU fallback")
    return torch.device("cuda:0")
