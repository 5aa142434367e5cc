import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "openal-soft_b200"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "ref: needs the compiled reference under oracle/_ref")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    from helpers import refal
    have_ref = refal.available()
    have_gpu = _has_gpu()
    for item in items:
        if "gpu" in item.keywords and not have_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device here (runs on an H100)"))
        if "ref" in item.keywords and not have_ref:
            item.add_marker(pytest.mark.skip(reason="oracle/_ref not built"))
