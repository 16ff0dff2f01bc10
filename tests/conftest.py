import importlib.util
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


def pytest_collection_modifyitems(config, items):
    """On a box without a CUDA device the gpu-marked tests are skipped instead of erroring (a plain `pytest` is green there);
    on the GPU box nothing is skipped - a missing libvfi_b200.so still fails loudly, by design."""
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs an H100 (torch.cuda.is_available() is False)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def load_pkg():
    """Import the product package (its directory name has a hyphen, like every ComfyUI custom node)."""
    import __graft_entry__ as ge
    return ge.load_package()


@pytest.fixture(scope="session")
def pkg():
    return load_pkg()
