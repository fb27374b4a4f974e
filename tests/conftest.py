import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _cuda_devices():
    """Number of CUDA devices the product library sees (0 when the library is missing or there is no driver)."""
    try:
        import sdk_b200._lib as L
        return int(L.LIB.b200pir_device_count())
    except Exception:
        return 0


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU (or a plain `pytest tests`) skips the GPU tests instead of failing in ctx_create;
    # on a GPU box they all run: no GPU test is gated by an environment variable.
    if not any("gpu" in item.keywords for item in items):
        return
    if _cuda_devices() > 0:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible to libb200pir.so")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
