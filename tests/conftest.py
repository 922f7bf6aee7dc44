import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def _usable_gpu() -> bool:
    """One probe per session: is there a CUDA device of compute capability 9.0 (libertgpu is sm_90a only)?"""
    try:
        import torch
        return torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0)
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """CPU-only machines: every test marked `gpu` is skipped (not failed, not an error at collection) -- the
    product has no CPU fallback to run them on."""
    if any("gpu" in item.keywords for item in items) and not _usable_gpu():
        skip = pytest.mark.skip(reason="no sm_90 CUDA device: GPU parity tests need an H100 (run with -m gpu there)")
        for item in items:
            if "gpu" in item.keywords:
                item.add_marker(skip)


@pytest.fixture(scope="session")
def sample_iq():
    import numpy as np
    return np.fromfile(os.path.join(GOLDEN, "sample_cl78.bin"), dtype=np.uint8)


@pytest.fixture(scope="session")
def built():
    """Make sure the in-tree shared libraries exist (compiles on CPU, no GPU needed)."""
    import __graft_entry__ as g
    g.build()
    return True
