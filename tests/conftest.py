import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU")


def pytest_collection_modifyitems(config, items):
    """gpu-marked tests are skipped (not failed) on a machine without an sm_90 device"""
    try:
        import torch
        ok = torch.cuda.is_available() and torch.cuda.get_device_capability(0)[0] == 9
    except Exception:
        ok = False
    if ok:
        return
    skip = pytest.mark.skip(reason="needs an H100 (sm_90) GPU")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def lib():
    from lwm_b200 import _lib
    return _lib.load()
