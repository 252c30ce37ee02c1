import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        ngpu = 0
    for item in items:
        if "gpu" in item.keywords and ngpu == 0:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 CUDA devices"))


@pytest.fixture(scope="session", autouse=True)
def _build_native():
    """Make sure the in-tree native libraries exist (nvcc cross-compiles without a GPU)."""
    from draco_b200 import build
    build.build_host()
    try:
        build.build_cuda()
    except Exception as e:  # no nvcc on this box: CPU tests still run
        print("cuda build skipped:", e)
    yield
