import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _restore_grad_mode():
    """Tests that switch autograd off globally (torch.set_grad_enabled(False)) must not leak it into the next test."""
    import torch
    prev = torch.is_grad_enabled()
    yield
    torch.set_grad_enabled(prev)


def rel_err(a, b):
    """max|a-b| / max|b|  -- the tolerance metric of SURVEY.md 8(d)."""
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))
