"""int8 scoring of the tensor-core Flat L2 search (112 < d <= 128, 2 <= k <= 128, unsharded): the results must equal
the exact kernel's bit for bit, whatever the dimension, the tail of the last tile, k, the storage type or a row mask,
and the search must say which operands it ran."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _exact(idx, xq, k, **kw):
    idx.setUseTensorCores(False)
    out = idx.search(xq, k, **kw)
    idx.setUseTensorCores(True)
    return out


# every d, tail (N mod 256), k and storage type appears at least once
CASES = [
    (113, 0, 2, False),
    (120, 1, 10, True),
    (127, 128, 100, False),
    (128, 129, 128, True),
    (128, 0, 100, False),
    (113, 129, 128, False),
    (120, 128, 2, False),
    (127, 1, 10, True),
]


@pytest.mark.parametrize("d,tail,k,fp16", CASES)
def test_int8_equals_exact(res, d, tail, k, fp16):
    import faiss_b200 as fb

    rs = np.random.RandomState(d * 1000 + tail + k)
    n = 65536 + tail
    xb = rs.rand(n, d).astype(np.float32)
    xq = rs.rand(300, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d, use_float16=fp16)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    assert idx.lastSearchOperandBits() == 8
    De, Ie = _exact(idx, xq, k)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)


def test_int8_with_row_mask_equals_exact(res):
    import faiss_b200 as fb

    rs = np.random.RandomState(5)
    d, n, k = 128, 100000, 100
    xb = rs.rand(n, d).astype(np.float32)
    xq = rs.rand(200, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    params = fb.SearchParameters(sel=fb.IDSelectorRange(1000, 90000))
    D, I = idx.search(xq, k, params=params)
    assert idx.lastSearchOperandBits() == 8
    assert ((I >= 1000) & (I < 90000)).all()
    De, Ie = _exact(idx, xq, k, params=params)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)


def test_operands_of_other_searches_stay_fp16(res):
    """int8 only for unsharded L2 at 112 < d <= 128 and 2 <= k <= 128 on a database that passes the fitness test"""
    import faiss_b200 as fb

    rs = np.random.RandomState(6)
    xb = rs.rand(40000, 128).astype(np.float32)
    xq = rs.rand(100, 128).astype(np.float32)
    l2 = fb.GpuIndexFlatL2(res, 128)
    l2.add(xb)
    l2.search(xq, 10)
    assert l2.lastSearchOperandBits() == 8
    for k in (1, 129):
        l2.search(xq, k)
        assert l2.lastSearchOperandBits() == 16, k
    ip = fb.GpuIndexFlatIP(res, 128)
    ip.add(xb)
    ip.search(xq, 10)
    assert ip.lastSearchOperandBits() == 16
    narrow = fb.GpuIndexFlatL2(res, 112)
    narrow.add(xb[:, :112].copy())
    narrow.search(xq[:, :112].copy(), 10)
    assert narrow.lastSearchOperandBits() == 16
    # one huge coordinate: s_y collapses and every ordinary row would quantise to zero
    out = xb.copy()
    out[7, 3] = 1e6
    o = fb.GpuIndexFlatL2(res, 128)
    o.add(out)
    D, I = o.search(xq, 10)
    assert o.lastSearchOperandBits() == 16
    De, Ie = _exact(o, xq, 10)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)
    l2.setUseTensorCores(False)
    l2.search(xq, 10)
    assert l2.lastSearchOperandBits() == 0


def test_int8_no_fallbacks_at_2m(res):
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda").manual_seed(7)
    xb = torch.rand(2_000_000, 128, device="cuda", generator=g)
    xq = torch.rand(2048, 128, device="cuda", generator=g)
    idx = fb.GpuIndexFlatL2(res, 128)
    idx.add(xb)
    D, I = idx.search(xq, 100)
    assert idx.lastSearchOperandBits() == 8
    assert idx.lastSearchInfo()["fallback_queries"] == 0
    De, Ie = _exact(idx, xq[:256].contiguous(), 100)
    assert torch.equal(I[:256], Ie) and torch.equal(D[:256], De)


def test_raw_int8_scores_are_integer_dot_products(res):
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda").manual_seed(8)
    n, nq = 700, 130  # n mod 256 != 0: the rows past n must score 0
    Q8 = torch.randint(-127, 128, (nq, 128), device="cuda", dtype=torch.int8, generator=g)
    Y8 = torch.randint(-127, 128, (n, 128), device="cuda", dtype=torch.int8, generator=g)
    S = fb.flat_tc_scores_debug(res, Q8, Y8)
    torch.cuda.synchronize()
    ref = Q8.double() @ Y8.double().T  # exact: |dot| <= 128 * 127^2
    assert torch.equal(S[:, :n].double(), ref)
    assert (S[:, n:] == 0).all()
