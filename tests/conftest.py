import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def _has_gpu():
    try:
        from selkies_b200 import _native
        return _native.lib().b2v_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a GPU-less box must fail loudly rather than silently pass on a fallback:
    # GPU tests are only skipped when the user did not ask for them explicitly.
    if "gpu" in (config.getoption("-m") or ""):
        return
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
