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


@pytest.fixture
def lib_option():
    """set_option(name, value) on the library for the duration of one test (restored afterwards)"""
    from fasterseg_b200 import _lib
    saved = []

    def setter(name, value):
        saved.append((name, _lib.get_option(name)))
        _lib.set_option(name, value)
    yield setter
    for name, old in reversed(saved):
        _lib.set_option(name, old)
