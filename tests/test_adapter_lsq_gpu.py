"""The reference's LocalSearchQuantizer with B200IcmEncoderFactory as its icm_encoder_factory, against the CPU encoder:
compute_codes byte for byte and the caller's generator state on integer data, and train's encode error on float data
(tests/adapter/adapter_lsq_test.cpp)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "adapter", "_build", "adapter_lsq_test")


@pytest.mark.gpu
def test_lsq_through_the_adapter():
    if not os.path.exists(BIN):
        pytest.skip("adapter binary not built (needs /root/reference at build time)")
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "ADAPTER_LSQ_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
