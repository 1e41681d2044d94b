"""CPU tests of the scalar-quantiser restatement (oracle/oracle_sq_np.py) against the IVF-SQ fixture
(tests/golden/ivfsq.npz) and, where oracle/_ref was built, against the live reference."""
import numpy as np
import pytest

from oracle import oracle_np as o
from oracle import oracle_sq_np as so
from tests.golden import make_golden_ivfsq as g


@pytest.fixture(scope="module")
def cases():
    return g.load()


@pytest.fixture(scope="module")
def ref_sq():
    from oracle import ref_sq as r

    if not r.available():
        pytest.skip("oracle/_ref/libfaiss_ref_sq.so not built (needs /root/reference at build time)")
    return r


def _assign(x, centroids, metric):
    return o.knn_flat(x, centroids, 1, metric)[1][:, 0]


def test_fixture_codes_bit_exact(cases):
    """re-encoding each case's database with the fixture's centroids and trained parameters reproduces the
    reference's list bytes"""
    for c in cases:
        a = _assign(c["xb"], c["centroids"], c["metric"])
        src = c["xb"] - c["centroids"][a] if c["by_residual"] else c["xb"]
        codes = so.sq_encode(src, c["qtype"], c["trained"])
        for l in range(g.NLIST):
            rows = c["ids"][l]
            assert np.array_equal(codes[rows].reshape(-1), c["codes"][l]), (c["i"], l)


def test_fixture_trained_bit_exact(cases):
    for c in cases:
        x = c["xt"]
        if c["by_residual"]:
            x = x - c["centroids"][_assign(x, c["centroids"], c["metric"])]
        t = so.train_minmax(x, c["qtype"])
        assert np.array_equal(t.view(np.uint32), c["trained"].view(np.uint32)), c["i"]


def test_fixture_search(cases):
    for c in cases:
        D, I = so.ivfsq_search(c["xq"], g.K, g.NPROBE, c["centroids"], c["qtype"], c["trained"], c["codes"], c["ids"],
                               c["metric"], c["by_residual"])
        o.compare_lists(c["D"], c["I"], D, I, eps=1e-5, pct_max_diff1=0.02, pct_max_diffN=0.01)


def test_code_size():
    assert [so.code_size(q, 36) for q in range(7)] == [36, 18, 36, 18, 72, 36, 27]
    assert so.code_size(so.QT_6bit, 38) == 29 and so.code_size(so.QT_4bit, 39) == 20


@pytest.mark.parametrize("qtype", range(7))
@pytest.mark.parametrize("d", [36, 38, 64])
def test_live_reference_encode_train(ref_sq, qtype, d):
    """fresh seeds: trained parameters and codes (4-/6-bit double-product truncation, 6-bit packing, odd d)
    bit-exact with the reference"""
    rs = np.random.RandomState(7 * d + qtype)
    scale = 256 if qtype == so.QT_8bit_direct else 5
    xt = (rs.rand(1500, d) * scale).astype(np.float32)
    if qtype == so.QT_8bit_direct:
        xt = np.floor(xt)
    idx = ref_sq.IndexIVFScalarQuantizer(d, 4, qtype, 1, qtype != so.QT_8bit_direct)
    idx.set_cp(niter=3)
    idx.train(xt)
    x = xt
    if idx.by_residual:
        x = xt - idx.centroids()[idx.quantizer_search(xt, 1)[1][:, 0]]
    t = idx.trained()
    assert np.array_equal(t.view(np.uint32), so.train_minmax(x, qtype).view(np.uint32))
    xb = (rs.rand(2000, d) * scale * 1.2 - 0.1 * scale).astype(np.float32)  # some values outside the trained range
    a = idx.quantizer_search(xb, 1)[1][:, 0]
    src = xb - idx.centroids()[a] if idx.by_residual else xb
    assert np.array_equal(idx.encode(xb, a), so.sq_encode(src, qtype, t))
