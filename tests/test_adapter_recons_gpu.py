"""search_and_reconstruct and reconstruct_batch through the compiled faiss::Index adapter, on adapter clones of
IndexFlatL2, IndexIVFFlat and IndexIVFPQ with ids stored twice, against the CPU indexes
(tests/adapter/adapter_recons_test.cpp)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "adapter", "_build", "adapter_recons_test")


@pytest.mark.gpu
def test_search_and_reconstruct_through_the_adapter():
    if not os.path.exists(BIN):
        pytest.skip("adapter binary not built (needs /root/reference at build time)")
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ADAPTER_RECONS_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
