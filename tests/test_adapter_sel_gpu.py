"""Filtered search through the compiled faiss::Index adapter: the reference's own IDSelectors and a user subclass (the
callback path), on adapter clones of IndexFlatL2 and IndexIVFFlat, against the CPU
indexes searched with the same parameters (tests/adapter/adapter_sel_test.cpp)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "adapter", "_build", "adapter_sel_test")


@pytest.mark.gpu
def test_reference_selectors_through_the_adapter():
    if not os.path.exists(BIN):
        pytest.skip("adapter binary not built (needs /root/reference at build time)")
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ADAPTER_SEL_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
