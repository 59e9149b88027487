import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    # the CPU oracle is what the GPU tests wait for: a sane thread count beats 128-way oversubscription
    try:
        import torch

        torch.set_num_threads(min(16, os.cpu_count() or 1))
    except Exception:
        pass
    config.addinivalue_line("markers", "gpu: test needs a CUDA (sm_90a) device")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
