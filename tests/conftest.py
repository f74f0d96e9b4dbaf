import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        have = torch.cuda.is_available()
        ngpu = torch.cuda.device_count() if have else 0
    except Exception:
        have, ngpu = False, 0
    for item in items:
        if "gpu" in item.keywords and not have:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))
