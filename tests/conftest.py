import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def golden():
    import torch
    return torch.load(os.path.join(ROOT, "tests", "golden", "gradtts_golden.pt"), weights_only=False)


@pytest.fixture(scope="session")
def sbk_lib():
    """libsbk.so, built in-tree if missing (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as ge
    ge.build()
    from speech_backbones_b200.binding import load_library
    return load_library()
