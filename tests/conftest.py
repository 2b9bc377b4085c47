import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-gan_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a; select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


def rel_err(a, b):
    """Norm-relative error ||a-b|| / ||b|| in fp64 (the north star's 1e-3 metric)."""
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    den = b.norm().item()
    return (a - b).norm().item() / (den if den > 0 else 1.0)
