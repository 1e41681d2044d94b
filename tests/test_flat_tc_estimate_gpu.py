"""Estimated thresholds in the tensor-core Flat search (DESIGN.md 3.1): the rounds may filter against a query's j-th
best score so far instead of its k-th, the last round checks every estimate against the final threshold, and a
query whose estimate overshot is searched again with provable thresholds.  Whatever the estimates did, the results
must equal the exact kernel's bit for bit, and a repair is never counted as an exact-kernel recompute."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _exact(idx, xq, k, **kw):
    idx.setUseTensorCores(False)
    out = idx.search(xq, k, **kw)
    idx.setUseTensorCores(True)
    return out


# (d, k, nq, bits): d = 128 scores on the int8 tensor cores, d = 96 in fp16; k = 1024 takes the sorted-list selection
# and 2048-query batches, so 5000 queries run as three batches
CASES = [(128, 2, 300, 8), (128, 10, 300, 8), (128, 100, 1000, 8), (128, 128, 300, 8),
         (96, 10, 300, 16), (96, 100, 1000, 16), (96, 1024, 5000, 16)]


@pytest.mark.parametrize("d,k,nq,bits", CASES)
def test_estimated_search_equals_exact(res, d, k, nq, bits):
    import faiss_b200 as fb

    rs = np.random.RandomState(d * 7 + k)
    n = 400_000
    xb = rs.rand(n, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    assert idx.lastSearchOperandBits() == bits
    assert idx.lastSearchRepairedQueries() >= 0
    De, Ie = _exact(idx, xq, k)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)


@pytest.mark.parametrize("d,bits", [(128, 8), (96, 16)])
def test_estimated_search_with_row_mask_equals_exact(res, d, bits):
    import faiss_b200 as fb

    rs = np.random.RandomState(d)
    n, k = 300_000, 100
    xb = rs.rand(n, d).astype(np.float32)
    xq = rs.rand(500, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    params = fb.SearchParameters(sel=fb.IDSelectorRange(20_000, 250_000))
    D, I = idx.search(xq, k, params=params)
    assert idx.lastSearchOperandBits() == bits
    assert ((I >= 20_000) & (I < 250_000)).all()
    De, Ie = _exact(idx, xq, k, params=params)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)


def _crowded_tile(rs, d, n, k, offset):
    """n rows and queries whose k nearest rows all sort into the tile the rounds scan first.

    The layouts store rows by (centred) norm and round 0 starts at tile T / 3 of that order, so exactly 256 * (T / 3)
    rows get a small norm, the k near-duplicates of the query a middling one, and the rest a large one.  Every row
    but the near-duplicates comes with its negation, which puts the int8 layout's centre at `offset`."""
    T = (n + 255) // 256
    small, large = 256 * (T // 3), n - 256 * (T // 3) - k
    assert small % 2 == 0 and large % 2 == 0

    def shell(m, lo, hi):
        v = rs.normal(size=(m // 2, d))
        v *= (rs.uniform(lo, hi, size=(m // 2, 1)) / np.linalg.norm(v, axis=1, keepdims=True))
        return np.concatenate([v, -v])

    p = rs.normal(size=d)
    p /= np.linalg.norm(p)
    dups = p + 0.01 * rs.normal(size=(k, d))
    xb = np.concatenate([shell(small, 0.1, 0.5), dups, shell(large, 2.0, 3.0)]) + offset
    xq = np.repeat((p + offset)[None], 16, axis=0)  # 16 queries: the fewest the index sends to the tensor cores
    return xb.astype(np.float32), xq.astype(np.float32)


@pytest.mark.parametrize("d,bits,offset", [(128, 8, 2.0), (96, 16, 0.0)])
def test_overshooting_estimate_is_repaired(res, d, bits, offset):
    import faiss_b200 as fb

    rs = np.random.RandomState(11)
    n, k = 200_000, 100
    xb, xq = _crowded_tile(rs, d, n, k, offset)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchOperandBits() == bits
    first = 256 * ((n + 255) // 256 // 3)
    assert all(set(row.tolist()) == set(range(first, first + k)) for row in I)
    assert idx.lastSearchRepairedQueries() == len(xq)
    assert idx.lastSearchInfo()["fallback_queries"] == 0
    De, Ie = _exact(idx, xq, k)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)
