import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def built():
    """Native artefacts are built in-tree (python feature-3dgs_b200/build.py); fail loudly if absent."""
    lib = os.path.join(ROOT, "feature-3dgs_b200", "libf3dgs_b200.so")
    if not os.path.exists(lib):
        sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
        import build as _b

        _b.build_all()
    assert os.path.exists(lib)
    return lib
