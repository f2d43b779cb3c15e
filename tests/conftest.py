import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def amb_lib():
    """The sm_90a C-ABI library; built on demand (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as ge

    if not os.path.exists(ge.LIB_PATH):
        ge.build()
    from actionmesh_b200 import _lib

    return _lib.load_library()


def load_golden(name):
    import torch

    return torch.load(os.path.join(GOLDEN, name), map_location="cpu", weights_only=False)
