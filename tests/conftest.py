import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _cuda_usable() -> bool:
    try:
        import torch
        return torch.cuda.is_available() and torch.cuda.device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need an H100: on a machine without a usable CUDA device they are skipped (not failed), so a plain
    `pytest` is green on CPU and `-m gpu` is the explicit device run."""
    if _cuda_usable():
        return
    skip = pytest.mark.skip(reason="no usable CUDA device (gpu-marked tests run on an H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """The in-tree .so is prebuilt by __graft_entry__.build(); build it when a checkout lacks it."""
    lib = os.path.join(ROOT, "matrel_b200", "libmatrel_b200.so")
    if not os.path.exists(lib):
        import __graft_entry__ as g
        g.build()


@pytest.fixture(scope="session")
def session():
    import matrel_b200 as mb
    s = mb.MatfastSession(device=0)
    yield s
    s.stop()
