import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (H100, sm_90a)")


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference CPU library (oracle/_ref); skipped where it was never built."""
    from oracle import ref as r

    if not r.available():
        pytest.skip("oracle/_ref not built (needs /root/reference at build time)")
    return r


@pytest.fixture(scope="session")
def golden():
    path = os.path.join(ROOT, "tests", "golden", "golden.npz")
    return np.load(path)


@pytest.fixture(scope="session")
def res():
    import faiss_b200 as fb

    return fb.StandardGpuResources()
