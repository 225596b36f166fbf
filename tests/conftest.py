import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a machine without CUDA skips the GPU tests instead of failing them."""
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason='needs a CUDA device (H100)')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)
