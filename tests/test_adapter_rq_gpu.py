"""The reference's ResidualQuantizer through the adapter (tests/adapter/adapter_rq_test.cpp): B200ResidualQuantizer's
compute_codes against the CPU's byte for byte on integer data, in both modes and for every search type; a plain
ResidualQuantizer with B200ProgressiveDimIndexFactory as its assign_index_factory (the reference's TestGpuResidualQuantizer
check); and a B200ResidualQuantizer trained through the factory, whose encode error matches the CPU encoder's."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "adapter", "_build", "adapter_rq_test")


@pytest.mark.gpu
def test_rq_through_the_adapter():
    if not os.path.exists(BIN):
        pytest.skip("adapter binary not built (needs /root/reference at build time)")
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "ADAPTER_RQ_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
