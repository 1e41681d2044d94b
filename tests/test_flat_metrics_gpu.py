"""GPU tests of the extra metrics of GpuIndexFlat / bfKnn (L1, Linf, Lp, Canberra, BrayCurtis, JensenShannon,
Jaccard, Gower) against the reference CPU IndexFlat of the same metric (oracle/_ref) where it travelled to this
box, else against the numpy restatement of knn_extra_metrics (oracle/oracle_metrics_np.py).

  * every metric x {fp32, fp16 storage} x shapes covering odd d, the database split (nq <= 5), every top-k
    path (k = 1, list sizes up to 1024) and one large case: distances within 1e-4 relative;
  * integer-valued data: ids and distances bit-exact for L1, Linf, BrayCurtis and Jaccard; Linf on floats too;
  * NaN rows never appear, missing results are (-1, FLT_MAX / -FLT_MAX);
  * direction (Jaccard is a similarity) through the shard merge, topk_merge and the empty index.
"""
import numpy as np
import pytest

from oracle import oracle_metrics_np as m
from oracle import oracle_np as o
from tests.golden import make_golden_metrics as g

pytestmark = pytest.mark.gpu

METRICS = [
    ("L1", m.METRIC_L1, 0.0),
    ("Linf", m.METRIC_Linf, 0.0),
    ("Lp0.5", m.METRIC_Lp, 0.5),
    ("Lp3", m.METRIC_Lp, 3.0),
    ("Canberra", m.METRIC_Canberra, 0.0),
    ("BrayCurtis", m.METRIC_BrayCurtis, 0.0),
    ("JensenShannon", m.METRIC_JensenShannon, 0.0),
    ("Jaccard", m.METRIC_Jaccard, 0.0),
    ("Gower", m.METRIC_GOWER, 0.0),
]
EXACT_INT = [("L1", m.METRIC_L1), ("Linf", m.METRIC_Linf), ("BrayCurtis", m.METRIC_BrayCurtis), ("Jaccard", m.METRIC_Jaccard)]


def _truth(xq, xb, k, metric, arg=0.0):
    from oracle import ref_metrics

    if ref_metrics.available():
        idx = ref_metrics.IndexFlat(xb.shape[1], metric, arg)
        idx.add(xb)
        return idx.search(xq, k)
    return m.knn_extra(xq, xb, k, metric, arg)


def _index(res, d, metric, arg=0.0, fp16=False, tc=True):
    import faiss_b200 as fb

    idx = fb.GpuIndexFlat(res, d, metric, use_tensor_cores=tc, use_float16=fp16)
    idx.metric_arg = arg
    return idx


def _round16(x):
    return x.astype(np.float16).astype(np.float32)


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("name,metric,arg", METRICS, ids=[t[0] for t in METRICS])
@pytest.mark.parametrize("N,d,nq,k", [(3000, 17, 5, 10), (4000, 64, 1, 100), (2500, 100, 5, 1024), (3000, 128, 1, 1),
                                      (6000, 40, 37, 1500), (50000, 32, 256, 10)])
def test_every_metric(res, name, metric, arg, fp16, N, d, nq, k):
    rs = np.random.RandomState(N + d + nq + k + metric)
    xb = m.metric_data(metric, rs, N, d)
    xq = m.metric_data(metric, rs, nq, d)
    idx = _index(res, d, metric, arg, fp16)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 0
    if fp16:  # the truth is the CPU index over the fp16-rounded data
        xb, xq = _round16(xb), _round16(xq)
    rD, rI = _truth(xq, xb, k, metric, arg)
    o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)


@pytest.mark.parametrize("k", [1, 100])
@pytest.mark.parametrize("name,metric", EXACT_INT, ids=[t[0] for t in EXACT_INT])
def test_integer_data_bit_exact(res, name, metric, k):
    """floor(16 u) + 1: every partial sum is exact, so ids and distances are bit-exact, including Linf's tie groups of
    thousands of rows at rank k (the k best by (distance, id))"""
    rs = np.random.RandomState(11 + metric + k)
    xb = m.integers(rs, 50000, 40)
    xq = m.integers(rs, 5, 40)
    if metric == m.METRIC_Linf:
        if k == 1:  # each query repeated 2000 times at random positions: a tie group of 2000 at distance 0
            for q in range(5):
                xb[rs.permutation(50000)[:2000]] = xq[q]
        else:  # queries in {8, 9}: about 3800 rows tie at distance 7, the distance at rank 100
            xq = (np.floor(2 * rs.rand(5, 40)) + 8).astype(np.float32)
    idx = _index(res, 40, metric)
    idx.add(xb)
    D, I = idx.search(xq, k)
    nD, nI = m.knn_extra(xq, xb, k, metric)
    assert np.array_equal(I, nI)
    assert np.array_equal(D.view(np.uint32), nD.view(np.uint32))
    if metric == m.METRIC_Linf:
        assert (m.pairwise_extra(xq, xb, metric) == D[:, -1:]).sum(axis=1).min() > 1000  # the rank-k tie group
    from oracle import ref_metrics

    if ref_metrics.available():
        m.assert_same_knn(*_truth(xq, xb, k, metric), D, I)


@pytest.mark.parametrize("k", [1, 10])
def test_linf_float_bit_exact(res, k):
    """max does not depend on the order: Linf on floats is bit-exact"""
    rs = np.random.RandomState(5)
    xb = m.metric_data(m.METRIC_Linf, rs, 5000, 100)
    xq = m.metric_data(m.METRIC_Linf, rs, 5, 100)
    idx = _index(res, 100, m.METRIC_Linf)
    idx.add(xb)
    D, I = idx.search(xq, k)
    nD, nI = m.knn_extra(xq, xb, k, m.METRIC_Linf)
    assert np.array_equal(I, nI) and np.array_equal(D, nD)


def test_lp_dispatch(res):
    """p = 1 is the L1 kernel, p = 2 the L2 path with tensor cores; metric_arg set after add takes effect"""
    import faiss_b200 as fb

    rs = np.random.RandomState(3)
    d = 64
    xb = rs.rand(40000, d).astype(np.float32)  # large enough for the tensor-core path at k = 10
    xq = rs.rand(64, d).astype(np.float32)
    lp = _index(res, d, fb.METRIC_Lp, 1.0)
    lp.add(xb)
    l1 = _index(res, d, fb.METRIC_L1)
    l1.add(xb)
    D, I = lp.search(xq, 10)
    D1, I1 = l1.search(xq, 10)
    assert np.array_equal(I, I1) and np.array_equal(D, D1)

    lp.metric_arg = 2.0
    assert lp.metric_arg == 2.0
    D, I = lp.search(xq, 10)
    assert lp.lastSearchInfo()["tensor_cores"] == 1
    l2 = fb.GpuIndexFlatL2(res, d)
    l2.add(xb)
    D2, I2 = l2.search(xq, 10)
    assert l2.lastSearchInfo()["tensor_cores"] == 1
    assert np.array_equal(I, I2) and np.array_equal(D, D2)

    lp.metric_arg = 3.0
    D, I = lp.search(xq, 10)
    assert lp.lastSearchInfo()["tensor_cores"] == 0
    rD, rI = _truth(xq, xb, 10, fb.METRIC_Lp, 3.0)
    o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)


def test_golden_fixture(res):
    """every fixture case, including NaN rows (zero components for Canberra / JensenShannon, out-of-range or mixed
    values for Gower) and queries with fewer valid rows than k, whose (-1, FLT_MAX) padding must equal the reference's"""
    for c in g.load():
        idx = _index(res, c["d"], c["metric"], c["arg"])
        idx.add(c["xb"])
        D, I = idx.search(c["xq"], c["k"])
        if c["kind"] == "int" and c["metric"] in (m.METRIC_L1, m.METRIC_Linf, m.METRIC_BrayCurtis, m.METRIC_Jaccard):
            m.assert_same_knn(c["D"], c["I"], D, I)
        else:
            o.compare_lists(c["D"], c["I"], D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)
        miss = c["I"] < 0
        assert np.array_equal(I < 0, miss) and (D[miss] == m.FLT_MAX).all()
        if c["kind"] in ("nan", "pad"):
            bad = np.isnan(m.pairwise_extra(c["xq"], c["xb"], c["metric"], c["arg"]))
            for q in range(I.shape[0]):
                assert not bad[q, I[q][I[q] >= 0]].any()


@pytest.mark.parametrize("k", [1, 5])
def test_nan_rows_k1_and_split(res, k):
    """NaN rows are excluded on the k = 1 packed path and across the database split as well"""
    rs = np.random.RandomState(9)
    d = 20
    for metric in (m.METRIC_Canberra, m.METRIC_JensenShannon, m.METRIC_GOWER):
        xb = m.metric_data(metric, rs, 4000, d)
        xq = m.metric_data(metric, rs, 3, d)
        g._spoil(metric, rs, xb, xq, rs.permutation(4000)[:3990])
        idx = _index(res, d, metric)
        idx.add(xb)
        D, I = idx.search(xq, k)
        rD, rI = m.knn_extra(xq, xb, k, metric)
        assert np.array_equal(I < 0, rI < 0)
        o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.0, pct_max_diffN=0.0)


@pytest.mark.parametrize("metric", [m.METRIC_L1, m.METRIC_Jaccard])
def test_shards_host_merge_direction(res, metric):
    import faiss_b200 as fb

    rs = np.random.RandomState(4)
    d = 24
    xb = m.metric_data(metric, rs, 6000, d)
    xq = m.metric_data(metric, rs, 20, d)
    full = _index(res, d, metric)
    full.add(xb)
    sh = fb.IndexShards(d)
    parts = [_index(res, d, metric), _index(res, d, metric)]
    parts[0].add(xb[:3000])
    parts[1].add(xb[3000:])
    for p in parts:
        sh.add_shard(p)
    D, I = sh.search(xq, 50)
    assert sh.lastSearchPath() == "host"
    Df, If = full.search(xq, 50)
    assert np.array_equal(I, If) and np.array_equal(D, Df)


@pytest.mark.parametrize("metric", [m.METRIC_L1, m.METRIC_Jaccard])
def test_topk_merge_direction(res, metric):
    import torch

    import faiss_b200 as fb

    # two lists per query, each sorted best first in the metric's direction
    a = np.array([0.1, 0.2, 0.3, 0.4], dtype=np.float32)
    b = np.array([0.15, 0.25, 0.35, 0.45], dtype=np.float32)
    if metric == m.METRIC_Jaccard:
        a, b = a[::-1].copy(), b[::-1].copy()
    D_in = torch.tensor(np.stack([a, b])[None], device="cuda")
    I_in = torch.tensor(np.array([[[0, 1, 2, 3], [10, 11, 12, 13]]], dtype=np.int64), device="cuda")
    D, I = fb.topk_merge(res, D_in, I_in, 3, metric=metric)
    torch.cuda.synchronize()
    if metric == m.METRIC_Jaccard:
        assert I.cpu().tolist() == [[10, 0, 11]]
    else:
        assert I.cpu().tolist() == [[0, 10, 1]]


def test_empty_index_sentinels(res):
    for metric in (m.METRIC_L1, m.METRIC_Jaccard, m.METRIC_GOWER):
        idx = _index(res, 8, metric)
        D, I = idx.search(np.ones((2, 8), dtype=np.float32), 4)
        assert (I == -1).all()
        assert (D == (-m.FLT_MAX if metric == m.METRIC_Jaccard else m.FLT_MAX)).all()


def test_bfknn_and_metric_type(res):
    import torch

    import faiss_b200 as fb

    rs = np.random.RandomState(8)
    d = 33
    xb = m.positive(rs, 3000, d)
    xq = m.positive(rs, 40, d)
    for metric, arg in ((fb.METRIC_Lp, 3.0), (fb.METRIC_Jaccard, 0.0), (fb.METRIC_Canberra, 0.0)):
        idx = _index(res, d, metric, arg)
        assert idx.metric_type == metric
        idx.add(xb)
        D, I = idx.search(xq, 20)
        bD, bI = fb.bfKnn(res, xq, xb, 20, metric=metric, metric_arg=arg)
        assert np.array_equal(I, bI) and np.array_equal(D, bD)
        tq, tb = torch.from_numpy(xq).cuda(), torch.from_numpy(xb).cuda()
        kD, kI = fb.knn_gpu(res, tq, tb, 20, metric=metric, metric_arg=arg)
        torch.cuda.synchronize()
        assert kD.is_cuda and np.array_equal(kI.cpu().numpy(), I) and np.array_equal(kD.cpu().numpy(), D)
    assert fb.GpuIndexFlat(res, d, fb.METRIC_GOWER).metric_type == fb.METRIC_GOWER
    assert fb.GpuIndexFlatIP(res, d).metric_type == fb.METRIC_INNER_PRODUCT


def test_rejections(res):
    import faiss_b200 as fb

    with pytest.raises(fb.FaissError, match="unsupported metric type 2"):
        fb.GpuIndexIVFFlat(res, 16, 4, metric=fb.METRIC_L1)
    with pytest.raises(fb.FaissError, match="unsupported metric type 23"):
        fb.GpuIndexIVFPQ(res, 16, 4, 4, metric=fb.METRIC_Jaccard)
    with pytest.raises(fb.FaissError, match="unsupported metric type 3"):
        fb.GpuIndexIVFScalarQuantizer(res, 16, 4, metric=fb.METRIC_Linf)
    x = np.random.RandomState(0).rand(500, 16).astype(np.float32)
    with pytest.raises(fb.FaissError, match="unsupported metric type 2"):
        fb.kmeans_ex(res, x, 4, niter=2, metric=fb.METRIC_L1)
    with pytest.raises(fb.FaissError, match="unimplemented metric type 24"):
        fb.GpuIndexFlat(res, 16, fb.METRIC_NaNEuclidean)
    with pytest.raises(fb.FaissError, match="unimplemented metric type 24"):
        fb.bfKnn(res, x[:4], x, 3, metric=fb.METRIC_NaNEuclidean)
