import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
ORACLE = os.path.join(ROOT, 'oracle')
if ORACLE not in sys.path:
    sys.path.insert(0, ORACLE)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


def pytest_collection_modifyitems(config, items):
    # GPU tests never run implicitly on a machine without a device
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for it in items:
        if 'gpu' in it.keywords:
            it.add_marker(skip)


@pytest.fixture(autouse=True)
def _release_device_engines():
    """every live g4r handle owns a constant-memory slot of the library (24 per process): drop unreachable engines between tests"""
    yield
    import gc
    gc.collect()
