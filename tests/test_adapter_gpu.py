"""The compiled faiss::Index adapter (faiss_b200/adapter): built against the reference's own headers and
CPU library, then driven by the reference's own code -- faiss::Clustering::train, faiss::IndexShards, the cloner
pair -- on the GPU (tests/adapter/adapter_test.cpp)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "adapter", "_build", "adapter_test")


def test_adapter_compiles_against_reference_headers():
    """no GPU needed: the adapter and its driver compile and link against /root/reference + oracle/_ref"""
    if not os.path.isdir("/root/reference/faiss"):
        if not os.path.exists(BIN):
            pytest.skip("the reference tree is not mounted here and no prebuilt adapter binary travelled")
        return
    from tests.adapter.build_adapter import build_adapter

    out = build_adapter(verbose=False)
    assert out and os.path.exists(out)
    syms = subprocess.run(["nm", "-C", out], capture_output=True, text=True).stdout
    for cls in ("B200IndexFlat", "B200IndexIVFPQ", "index_cpu_to_b200", "index_b200_to_cpu"):
        assert cls in syms


@pytest.mark.gpu
def test_reference_drivers_over_the_adapter():
    if not os.path.exists(BIN):
        pytest.skip("adapter binary not built (needs /root/reference at build time)")
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ADAPTER_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
