import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (an H100)")


@pytest.fixture(scope="session")
def tok_lib():
    """libtok8s.so, built in-tree on demand (nvcc cross-compiles sm_90a without a GPU)."""
    from torch_on_k8s_b200 import _ffi
    if not os.path.exists(_ffi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _ffi.lib()


@pytest.fixture(scope="session")
def n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0
