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


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need a CUDA device: skip them (instead of failing) when none is visible, so plain `pytest tests`
    is green on a CPU box as well as `-m "not gpu"`."""
    try:
        import torch
        has_cuda = torch.cuda.is_available()
    except Exception:      # noqa: BLE001
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


@pytest.fixture(scope="session")
def rf():
    """The product package (loads the C-ABI library; no compute without a GPU)."""
    import ransac_flow_b200
    return ransac_flow_b200
