"""GPU tests of all-pairs distances (pairwise_distance_gpu, bfKnn with k = -1), knn_gpu's input formats and int32
ids, the paged host-resident matrix and bfKnn_tiling.

  (a) integer-valued data: bit-exact against the golden fixture and the CPU restatements for L2, IP, L1, Linf,
      BrayCurtis and Jaccard; the other metrics within test_flat_metrics_gpu.py's tolerance;
  (b) float data, L2 / IP: every entry within the float64 truth's certified bound;
  (c) pairwise[i, I[i, j]] == D[i, j] bit for bit against knn_gpu, on the tensor-core and the exact path, and each
      row's (distance, id) top-k is I;
  (d) fp32 / fp16 / bf16 x query / vector layout x host / device x int64 / int32: bit-identical to the fp32 row-major
      call on the widened values;
  (e) a device-resident matrix of more than 2^31 entries;
  (f) a host-resident matrix through >= 3 row blocks, and through column blocks: equal to the device result;
  (g) bfKnn_tiling over >= 3 x 3 shards equals bfKnn bit for bit.
"""
import os

import numpy as np
import pytest

from oracle import oracle_bound_np as ob
from oracle import oracle_metrics_np as m
from oracle import oracle_np as o

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ALL = [
    ("L2", m.METRIC_L2, 0.0),
    ("IP", m.METRIC_INNER_PRODUCT, 0.0),
    ("L1", m.METRIC_L1, 0.0),
    ("Linf", m.METRIC_Linf, 0.0),
    ("Lp1", m.METRIC_Lp, 1.0),
    ("Lp2", m.METRIC_Lp, 2.0),
    ("Lp0.5", m.METRIC_Lp, 0.5),
    ("Lp3", m.METRIC_Lp, 3.0),
    ("Canberra", m.METRIC_Canberra, 0.0),
    ("BrayCurtis", m.METRIC_BrayCurtis, 0.0),
    ("JensenShannon", m.METRIC_JensenShannon, 0.0),
    ("Jaccard", m.METRIC_Jaccard, 0.0),
    ("Gower", m.METRIC_GOWER, 0.0),
]
EXACT_INT = (m.METRIC_L2, m.METRIC_INNER_PRODUCT, m.METRIC_L1, m.METRIC_Linf, m.METRIC_BrayCurtis, m.METRIC_Jaccard)


def _cpu_pairwise(xq, xb, metric, arg=0.0):
    """the CPU's all-pairs matrix: the reference library where it was built, else its numpy restatement"""
    from oracle import ref_pairwise

    if ref_pairwise.available():
        return ref_pairwise.pairwise(xq, xb, metric, arg)
    if metric in (m.METRIC_L2, m.METRIC_INNER_PRODUCT):
        return o.pairwise(xq, xb, metric)
    if metric == m.METRIC_Lp and arg in (1.0, 2.0):
        return _cpu_pairwise(xq, xb, m.METRIC_L1 if arg == 1.0 else m.METRIC_L2)
    return m.pairwise_extra(xq, xb, metric, arg)


def _same(a, b):
    """bit-identical, NaN included"""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else x


# ------------------------------------------------------------------ (a)
@pytest.fixture(scope="module")
def fixture():
    return np.load(os.path.join(ROOT, "tests", "golden", "pairwise.npz"))


@pytest.mark.parametrize("name,metric,arg", ALL, ids=[t[0] for t in ALL])
def test_golden_fixture(res, fixture, name, metric, arg):
    import faiss_b200 as fb

    for kind in ("int", "float"):
        key = "%s_%s" % (name, kind)
        xq, xb, want = fixture[key + "_xq"], fixture[key + "_xb"], fixture[key + "_D"]
        D = fb.pairwise_distance_gpu(res, xq, xb, metric=metric, metric_arg=arg)
        if kind == "int" and (metric in EXACT_INT or (metric == m.METRIC_Lp and arg in (1.0, 2.0))):
            assert _same(D, want), key
        else:
            nan = np.isnan(want)
            assert np.array_equal(nan, np.isnan(D)), key
            np.testing.assert_allclose(D[~nan], want[~nan], rtol=1e-4, atol=1e-5, err_msg=key)


@pytest.mark.parametrize("name,metric,arg", ALL, ids=[t[0] for t in ALL])
def test_integer_data_vs_cpu(res, name, metric, arg):
    import faiss_b200 as fb

    rs = np.random.RandomState(5 + metric)
    xb = m.metric_data(metric, rs, 3001, 37, integer=True)
    xq = m.metric_data(metric, rs, 45, 37, integer=True)
    D = fb.pairwise_distance_gpu(res, xq, xb, metric=metric, metric_arg=arg)
    want = _cpu_pairwise(xq, xb, metric, arg)
    if metric in EXACT_INT or (metric == m.METRIC_Lp and arg in (1.0, 2.0)):
        assert _same(D, want)
    else:
        nan = np.isnan(want)
        assert np.array_equal(nan, np.isnan(D))
        np.testing.assert_allclose(D[~nan], want[~nan], rtol=1e-4, atol=1e-5)


def test_nan_written_as_computed(res):
    """zero components: Canberra's 0/0 and JensenShannon's 0 * log(0/0) are NaN on the CPU, and in the matrix"""
    import faiss_b200 as fb

    rs = np.random.RandomState(3)
    xb = m.positive(rs, 300, 8)
    xq = m.positive(rs, 6, 8)
    xq[0, 3] = 0.0
    xb[7, 3] = 0.0
    for metric in (m.METRIC_Canberra, m.METRIC_JensenShannon):
        D = fb.pairwise_distance_gpu(res, xq, xb, metric=metric)
        want = m.pairwise_extra(xq, xb, metric)
        assert np.isnan(want).any() and np.array_equal(np.isnan(D), np.isnan(want))


# ------------------------------------------------------------------ (b)
@pytest.mark.parametrize("metric", [m.METRIC_L2, m.METRIC_INNER_PRODUCT])
@pytest.mark.parametrize("d", [16, 67, 128, 300])
def test_float_within_float64_bound(res, metric, d):
    import faiss_b200 as fb

    rs = np.random.RandomState(d)
    xb = (rs.rand(2003, d) * 2 - 1).astype(np.float32)
    xq = (rs.rand(77, d) * 2 - 1).astype(np.float32)
    D = fb.pairwise_distance_gpu(res, xq, xb, metric=metric).astype(np.float64)
    t, B = (ob.l2_truth_many if metric == m.METRIC_L2 else ob.ip_truth_many)(xq, xb)
    assert (np.abs(D - t) <= B).all()


# ------------------------------------------------------------------ (c)
@pytest.mark.parametrize("name,metric,arg", ALL, ids=[t[0] for t in ALL])
@pytest.mark.parametrize("N,d,nq,k,tc", [(40000, 128, 64, 20, True), (3000, 40, 8, 50, False), (5001, 17, 33, 1, True)])
def test_pairwise_agrees_with_knn(res, name, metric, arg, N, d, nq, k, tc):
    import torch

    import faiss_b200 as fb

    rs = np.random.RandomState(N + d + metric)
    xb = torch.from_numpy(m.metric_data(metric, rs, N, d)).cuda()
    xq = torch.from_numpy(m.metric_data(metric, rs, nq, d)).cuda()
    D, I = fb.knn_gpu(res, xq, xb, k, metric=metric, metric_arg=arg)
    # knn_gpu searches a default GpuIndexFlat: this one shows which path the shape takes (tensor cores for the
    # metrics with a product form at the shapes with nq >= 16, the exact kernel otherwise), with the same results
    idx = fb.GpuIndexFlat(res, d, metric)
    idx.metric_arg = arg
    idx.add(xb)
    Di, Ii = idx.search(xq, k)
    product = metric in (m.METRIC_L2, m.METRIC_INNER_PRODUCT) or (metric == m.METRIC_Lp and arg == 2.0)
    assert idx.lastSearchInfo()["tensor_cores"] == int(tc and product)
    assert torch.equal(Di, D) and torch.equal(Ii, I)
    P = fb.pairwise_distance_gpu(res, xq, xb, metric=metric, metric_arg=arg)
    torch.cuda.synchronize()
    D, I, P = D.cpu().numpy(), I.cpu().numpy(), P.cpu().numpy()
    valid = I >= 0
    got = np.take_along_axis(P, np.where(valid, I, 0), axis=1)
    assert _same(np.where(valid, got, D), D)
    sim = metric in (m.METRIC_INNER_PRODUCT, m.METRIC_Jaccard)
    ids = np.arange(N)
    for i in range(nq):
        row = P[i]
        ok = ~np.isnan(row)
        order = np.lexsort((ids[ok], -row[ok] if sim else row[ok]))[: int(valid[i].sum())]
        assert np.array_equal(ids[ok][order], I[i][valid[i]]), (name, i)


# ------------------------------------------------------------------ (d)
def _formats():
    for dt in ("float32", "float16", "bfloat16"):
        for qcol in (False, True):
            for bcol in (False, True):
                for dev in (False, True):
                    yield dt, qcol, bcol, dev


def _as(x, dt, col, dev):
    import torch

    if dt == "bfloat16" or dev:
        t = torch.from_numpy(x).to(getattr(torch, dt))
        if dev:
            t = t.cuda()
        return t.t().contiguous().t() if col else t
    a = x.astype(np.float16) if dt == "float16" else x
    return np.asfortranarray(a) if col else np.ascontiguousarray(a)


@pytest.mark.parametrize("metric", [m.METRIC_L2, m.METRIC_INNER_PRODUCT, m.METRIC_L1])
def test_format_invariance(res, metric):
    import torch

    import faiss_b200 as fb

    rs = np.random.RandomState(metric)
    N, d, nq, k = 20000, 40, 50, 16
    xb0 = (rs.rand(N, d) * 2 - 1).astype(np.float32)
    xq0 = (rs.rand(nq, d) * 2 - 1).astype(np.float32)
    widened = {
        "float32": (xq0, xb0),
        "float16": (xq0.astype(np.float16).astype(np.float32), xb0.astype(np.float16).astype(np.float32)),
        "bfloat16": tuple(torch.from_numpy(x).bfloat16().float().numpy() for x in (xq0, xb0)),
    }
    base = {dt: (fb.knn_gpu(res, q, b, k, metric=metric), fb.pairwise_distance_gpu(res, q, b, metric=metric))
            for dt, (q, b) in widened.items()}
    for dt, qcol, bcol, dev in _formats():
        q, b = _as(xq0, dt, qcol, dev), _as(xb0, dt, bcol, dev)
        (rD, rI), rP = base[dt]
        for itype in ("int64", "int32"):
            if dev:
                I = torch.empty((nq, k), dtype=getattr(torch, itype), device="cuda")
            else:
                I = np.empty((nq, k), dtype=itype)
            D, I = fb.knn_gpu(res, q, b, k, I=I, metric=metric)
            P = fb.pairwise_distance_gpu(res, q, b, metric=metric)
            torch.cuda.synchronize()
            what = (dt, qcol, bcol, dev, itype)
            assert str(I.dtype).endswith(itype), what
            assert _same(_np(D), rD) and np.array_equal(_np(I).astype(np.int64), rI), what
            assert _same(_np(P), rP), what


def test_mixed_types_refused(res):
    import faiss_b200 as fb

    x = np.zeros((10, 8), dtype=np.float32)
    with pytest.raises(fb.FaissError, match="same"):
        fb.knn_gpu(res, x, x.astype(np.float16), 3)


# ------------------------------------------------------------------ (e)
def test_matrix_past_2_pow_31_entries(res):
    import torch

    import faiss_b200 as fb

    nq, N, d = 2100, 1 << 20, 8
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    xq = torch.rand(nq, d, device="cuda", generator=g)
    xb = torch.rand(N, d, device="cuda", generator=g)
    assert nq * N > 2**31
    D = torch.empty((nq, N), dtype=torch.float32, device="cuda")
    fb.pairwise_distance_gpu(res, xq, xb, D=D)
    rows = torch.tensor([0, 1, 1024, 2047, 2048, 2099], device="cuda")  # rows 2048.. start past 2^31 entries
    # the exact k-NN kernel: its distances at its ids, and the whole row from a one-row call
    exact = fb.GpuIndexFlat(res, d, fb.METRIC_L2, use_tensor_cores=False)
    exact.add(xb)
    Dk, Ik = exact.search(xq[rows], 100)
    assert exact.lastSearchInfo()["tensor_cores"] == 0
    assert torch.equal(torch.gather(D[rows], 1, Ik), Dk)
    for i in rows.tolist():
        want = fb.pairwise_distance_gpu(res, xq[i : i + 1], xb)
        assert torch.equal(D[i : i + 1], want), i
    torch.cuda.synchronize()
    del D


# ------------------------------------------------------------------ (f)
@pytest.mark.parametrize("metric", [m.METRIC_L2, m.METRIC_INNER_PRODUCT, m.METRIC_Canberra])
@pytest.mark.parametrize("N,nq,page", [(1000, 200, 40 * 4000), (5000, 100, 128 * 1024), (5001, 70, 16384), (5001, 3, 8000)])
def test_host_output_blocks(res, metric, N, nq, page):
    import torch

    import faiss_b200 as fb

    rs = np.random.RandomState(N + nq)
    xb = m.metric_data(metric, rs, N, 24)
    xq = m.metric_data(metric, rs, nq, 24)
    Dd = fb.pairwise_distance_gpu(res, torch.from_numpy(xq).cuda(), torch.from_numpy(xb).cuda(), metric=metric)
    torch.cuda.synchronize()
    Dh = np.full((nq, N), 7.0, dtype=np.float32)
    fb._distance_call(res, xq, xb, -1, Dh, None, metric, 0, 0.0, page_bytes=page)
    assert _same(Dh, Dd.cpu().numpy())
    # the default budget: one block
    assert _same(fb.pairwise_distance_gpu(res, xq, xb, metric=metric), Dh)


# ------------------------------------------------------------------ (g)
@pytest.mark.parametrize("metric", [m.METRIC_L2, m.METRIC_INNER_PRODUCT])
@pytest.mark.parametrize("itype", ["int64", "int32"])
def test_tiling_equals_bfknn(res, metric, itype):
    import faiss_b200 as fb

    rs = np.random.RandomState(metric + 17)
    N, d, nq, k = 30000, 32, 300, 25
    xb = np.floor(rs.rand(N, d) * 8).astype(np.float32)  # many ties: the merge must keep (distance, id) order
    xq = np.floor(rs.rand(nq, d) * 8).astype(np.float32)
    D, I = fb.knn_gpu(res, xq, xb, k, metric=metric)
    ls = 8 if itype == "int64" else 4
    vlim = 10000 * d * 4 + 100  # 3 vector shards
    qlim = 100 * (k * (4 + ls) + d * 4)  # 3 query shards
    many = 2000 * d * 4  # 15 vector shards: 14 running merges
    for v, q in ((vlim, 0), (0, qlim), (vlim, qlim), (many, 0), (many, qlim)):
        It = np.empty((nq, k), dtype=itype)
        Dt, It = fb.knn_gpu(res, xq, xb, k, I=It, metric=metric, vectorsMemoryLimit=v, queriesMemoryLimit=q)
        assert _same(Dt, D) and np.array_equal(It.astype(np.int64), I), (v, q)


def test_tiling_device_input_refused(res):
    import torch

    import faiss_b200 as fb

    x = torch.rand(100, 8, device="cuda")
    with pytest.raises(fb.FaissError, match="CPU memory"):
        fb.knn_gpu(res, x.cpu(), x, 5, vectorsMemoryLimit=1024)
    with pytest.raises(fb.FaissError, match="CPU memory"):
        fb.knn_gpu(res, x, x.cpu(), 5, queriesMemoryLimit=4096)


# ------------------------------------------------------------------ host inputs converted page by page
@pytest.mark.parametrize("col", [False, True])
def test_host_inputs_converted_in_pages(res, col):
    """fp16 host queries / vectors above the 256 MiB conversion page (fp32 rows) go through >= 2 pages: same results as
    the fp32 row-major call on the widened values"""
    import faiss_b200 as fb

    rs = np.random.RandomState(int(col))
    d, big = 8, 9_000_000  # 9M x 8 fp32 rows = 288 MB > 256 MiB
    lay = np.asfortranarray if col else np.ascontiguousarray
    small = (rs.rand(1000, d) * 2 - 1).astype(np.float16)
    many = (rs.rand(big, d) * 2 - 1).astype(np.float16)
    # many queries against a small database
    D, I = fb.knn_gpu(res, lay(many), lay(small), 2)
    rD, rI = fb.knn_gpu(res, many.astype(np.float32), small.astype(np.float32), 2)
    assert _same(D, rD) and np.array_equal(I, rI)
    # few queries against a large database
    D, I = fb.knn_gpu(res, lay(small[:50]), lay(many), 10)
    rD, rI = fb.knn_gpu(res, small[:50].astype(np.float32), many.astype(np.float32), 10)
    assert _same(D, rD) and np.array_equal(I, rI)
