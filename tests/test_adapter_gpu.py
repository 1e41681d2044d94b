"""The compiled faiss::Index adapter (faiss_b200/adapter): built against the reference's own headers and
CPU library, then driven by the reference's own code on the GPU, one driver binary per feature
(tests/adapter/adapter[_<name>]_test.cpp, built by tests/adapter/build_adapter.py):
  adapter_test         faiss::Clustering::train, faiss::IndexShards and the cloner pair over the adapter
  adapter_sel_test     filtered search with the reference's own IDSelectors and a user subclass (the callback path),
                       on adapter clones of IndexFlatL2 and IndexIVFFlat, against the CPU indexes
  adapter_recons_test  search_and_reconstruct and reconstruct_batch on adapter clones of IndexFlatL2, IndexIVFFlat
                       and IndexIVFPQ with ids stored twice, against the CPU indexes
  adapter_lsq_test     LocalSearchQuantizer with B200IcmEncoderFactory as its icm_encoder_factory, against the CPU
                       encoder: compute_codes byte for byte and the caller's generator state on integer data, and
                       train's encode error on float data
  adapter_rq_test      B200ResidualQuantizer's compute_codes against the CPU's byte for byte on integer data, in both
                       modes and for every search type; a plain ResidualQuantizer with B200ProgressiveDimIndexFactory
                       as its assign_index_factory (the reference's TestGpuResidualQuantizer check); and a
                       B200ResidualQuantizer trained through the factory, whose encode error matches the CPU encoder's"""
import os
import subprocess

import pytest

from oracle import ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "adapter", "_build")
BIN = os.path.join(BUILD, "adapter_test")


def test_adapter_compiles_against_reference_headers():
    """no GPU needed: the adapter and its driver compile and link against the reference tree + oracle/_ref"""
    if not os.path.isdir(os.path.join(ref.REF, "faiss")):
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
@pytest.mark.parametrize(
    "binary, marker, timeout",
    [
        ("adapter_test", "ADAPTER_OK", 600),
        ("adapter_sel_test", "ADAPTER_SEL_OK", 600),
        ("adapter_recons_test", "ADAPTER_RECONS_OK", 600),
        ("adapter_lsq_test", "ADAPTER_LSQ_OK", 900),
        ("adapter_rq_test", "ADAPTER_RQ_OK", 900),
    ],
)
def test_reference_drivers_over_the_adapter(binary, marker, timeout):
    path = os.path.join(BUILD, binary)
    if not os.path.exists(path):
        pytest.skip("adapter binary not built (needs the reference tree at build time)")
    r = subprocess.run([path], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    assert r.returncode == 0 and marker in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
