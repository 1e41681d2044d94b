"""int8 search on a database whose row norms spread widely: uniform [0, 1) rows scaled by per-row factors in [0.5, 1].
The rows are stored sorted by norm, so neighbouring tiles, and the two halves of a tile, then have clearly different
biases, and a filter whose exact test read the biases of the wrong tile or half-tile would change the candidate sets
(on uniform data neighbouring tiles have nearly equal biases, which would hide it).  The spread still passes the int8
fitness test, which the operand-bits assertion guards.  Results must equal the exact kernel's bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _spread_rows(rs, n, d):
    return (rs.rand(n, d) * rs.uniform(0.5, 1.0, (n, 1))).astype(np.float32)


def _exact(idx, xq, k, **kw):
    idx.setUseTensorCores(False)
    out = idx.search(xq, k, **kw)
    idx.setUseTensorCores(True)
    return out


# 112 < d <= 128, with a tail tile (N mod 256 != 0), whose second half lies wholly past N when the tail is <= 128
@pytest.mark.parametrize("d,tail,k,fp16", [(128, 129, 100, False), (120, 1, 10, True), (113, 200, 128, False)])
def test_int8_spread_norms_equals_exact(res, d, tail, k, fp16):
    import faiss_b200 as fb

    rs = np.random.RandomState(d * 1000 + tail + k)
    n = 131072 + tail
    xb = _spread_rows(rs, n, d)
    xq = rs.rand(300, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d, use_float16=fp16)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchOperandBits() == 8
    info = idx.lastSearchInfo()
    assert info["tensor_cores"] == 1 and info["fallback_queries"] == 0, info
    De, Ie = _exact(idx, xq, k)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)


def test_int8_spread_norms_with_row_mask_equals_exact(res):
    import faiss_b200 as fb

    rs = np.random.RandomState(9)
    d, n, k = 128, 100000, 100
    xb = _spread_rows(rs, n, d)
    xq = rs.rand(200, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    params = fb.SearchParameters(sel=fb.IDSelectorRange(1000, 90000))
    D, I = idx.search(xq, k, params=params)
    assert idx.lastSearchOperandBits() == 8
    assert ((I >= 1000) & (I < 90000)).all()
    De, Ie = _exact(idx, xq, k, params=params)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)
