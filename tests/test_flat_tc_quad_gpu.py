"""The four-warpgroup tensor-core Flat kernel (112 < d <= 128): two warpgroups write each candidate segment through a
16-bit shared-memory count.  Segments that overflow must still flag their queries for the exact kernel, in the round
mode and in the k = 1 streaming mode, and a k-means-sized assignment must not overflow at all."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("d", [120, 128])
def test_segment_overflow_falls_back_to_exact(res, d):
    """2500 copies of each of 16 rows, one coordinate moved by 1: near-ties overflow the segments of their queries"""
    import faiss_b200 as fb

    rs = np.random.RandomState(21)
    base = np.floor(rs.rand(16, d) * 16).astype(np.float32)
    dup = np.repeat(base, 2500, axis=0)
    dup[np.arange(len(dup)), rs.randint(0, d, len(dup))] += 1.0
    far = -np.abs(rs.randn(40000, d) * 8).astype(np.float32)
    xb = np.vstack([dup, far])
    xq = np.vstack([base[rs.randint(0, 16, 64)], -np.abs(rs.randn(200, d) * 8).astype(np.float32)])
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    D, I = idx.search(xq, 100)
    info = idx.lastSearchInfo()
    assert info["tensor_cores"] == 1 and info["fallback_queries"] > 0
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, 100)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)


def test_streaming_ties_overflow_falls_back_to_exact(res):
    """k = 1: every distinct row 1500 times, so each query ties with more rows than a segment holds"""
    import faiss_b200 as fb

    rs = np.random.RandomState(22)
    base = np.floor(rs.rand(64, 128) * 8).astype(np.float32)
    xb = np.tile(base, (1500, 1))
    xq = base[rs.randint(0, 64, size=300)] + 0.0
    idx = fb.GpuIndexFlatL2(res, 128)
    idx.add(xb)
    D, I = idx.search(xq, 1)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, 1)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)
    assert (D == 0).all() and (I < 64).all()


def test_streaming_assignment_has_no_fallbacks(res):
    """k-means assignment shape: 4096 centroids, d = 128; no query needs the exact kernel and the labels are exact"""
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda").manual_seed(23)
    cent = torch.randn(4096, 128, device="cuda", generator=g)
    x = cent[torch.randint(0, 4096, (65536,), device="cuda", generator=g)]
    x = x + 0.7 * torch.randn(x.shape, device="cuda", generator=g)
    idx = fb.GpuIndexFlatL2(res, 128)
    idx.add(cent)
    D, I = idx.search(x, 1)
    assert idx.lastSearchInfo() == {"tensor_cores": 1, "fallback_queries": 0}
    idx.setUseTensorCores(False)
    De, Ie = idx.search(x, 1)
    assert torch.equal(I, Ie) and torch.equal(D, De)
