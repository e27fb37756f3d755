import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_cuda():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Every test may assume the in-tree library exists.  Without a GPU it is built incrementally (nvcc
    cross-compiles sm_90a); with a GPU an existing .so (the one build() made) is used as is -- file times of a copied
    tree are not meaningful -- and only a missing library triggers a build."""
    from purejaxql_b200 import build
    if _has_cuda() and os.path.exists(build.OUT):
        return build.OUT
    return build.build()
