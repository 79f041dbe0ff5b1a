import os
import sys

import pytest

# Ranks are threads sharing one GPU in the GPU tests: a rank loading a (torch) kernel for
# the first time must not block behind another rank's waiting collective kernel.
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs at least 2 CUDA devices")
    config.addinivalue_line("markers", "slow: long-running sweep")


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
