"""CPU tests: the numpy model of the result rule (oracle/oracle_rule_np.py) against the unmodified reference, on data
with non-finite, overflowing and FLT_MAX-valued distances.  They pin the model to the reference's behaviour, so the
GPU tests that compare the kernels with the model compare them with the reference's rule."""
import numpy as np
import pytest

from oracle import oracle_rule_np as rm

L2, IP = rm.METRIC_L2, rm.METRIC_INNER_PRODUCT
D_DIM, NLIST = 16, 8


def _bits(a):
    # + 0 turns -0 into +0: the sign of an exact zero depends on the summation order
    return np.ascontiguousarray(np.asarray(a, np.float32) + np.float32(0)).view(np.uint32)


def _assert_same(D, I, Dm, Im, metric=L2):
    """bit-equal distances; equal ids under L2.  Under inner product the reference's heap (CMin) orders a tie group by
    decreasing id and keeps a scan-order-dependent part of the group cut at rank k, while the model keeps the
    smallest ids (as the GPU kernels do): there the ids must agree per tie group, and the cut group's ids must be
    stored ids of that exact distance."""
    np.testing.assert_array_equal(_bits(D), _bits(Dm))
    if metric == L2:
        np.testing.assert_array_equal(I, Im)
        return
    np.testing.assert_array_equal(I == -1, Im == -1)
    for q in range(D.shape[0]):
        vals = [v for v in dict.fromkeys(_bits(D[q]).tolist())]
        for j, v in enumerate(vals):
            got = set(I[q][_bits(D[q]) == v].tolist())
            want = set(Im[q][_bits(Dm[q]) == v].tolist())
            if j < len(vals) - 1 or I[q, -1] == -1:
                assert got == want, (q, v, got, want)
            else:
                assert len(got) == len(want), (q, v, got, want)


@pytest.fixture(scope="module")
def ref_sq():
    from oracle import ref_sq as r

    if not r.available():
        pytest.skip("oracle/_ref/libfaiss_ref_sq.so not built (needs /root/reference at build time)")
    return r


def test_special_rows_classes():
    """the constructed distances are what the data claims, and order-independent: the sum in reverse order is equal"""
    rs = np.random.RandomState(0)
    for metric in (L2, IP):
        xq = rm.queries(rs, 5, D_DIM, metric)
        spec, kinds = rm.special_rows(D_DIM, metric)
        dis = rm.distances(xq, spec, metric)
        rev = rm.distances(xq[:, ::-1], spec[:, ::-1], metric)
        np.testing.assert_array_equal(_bits(dis), _bits(rev))
        for j, kind in enumerate(kinds):
            col = dis[:, j]
            if kind == "flt_max":
                assert np.all(col == rm.FLT_MAX), (metric, kind, col)
            elif kind in ("nan", "inf*0"):
                assert np.all(np.isnan(col)), (metric, kind, col)
            elif kind == "-flt_max":
                assert np.all(col == -rm.FLT_MAX)
            else:
                assert np.all(np.isinf(col)), (metric, kind, col)
        # under L2 no special row is a result; under IP only +inf and +FLT_MAX are
        ok = rm.is_result(dis, metric)
        if metric == L2:
            assert not ok.any()
        else:
            assert ok[:, kinds.index("flt_max")].all() and not ok[:, kinds.index("-flt_max")].any()


@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
@pytest.mark.parametrize("nq", [5, 40], ids=["nq5", "nq40"])  # below and above 20: the sequential and the BLAS path
@pytest.mark.parametrize("n_ordinary", [7, 300], ids=["pad", "rank"])
def test_flat(ref, metric, nq, n_ordinary):
    rs = np.random.RandomState(1 + nq + n_ordinary)
    n = 320
    xb, _ = rm.database(rs, n, D_DIM, metric, n_ordinary, positions=[0, n - 1, 5, 63, 64])
    xq = rm.queries(rs, nq, D_DIM, metric)
    idx = ref.IndexFlat(D_DIM, metric)
    idx.add(xb)
    for k in (1, 10, 50):
        D, I = idx.search(xq, k)
        _assert_same(D, I, *rm.knn(xq, xb, k, metric), metric)


def _ivf_cases(ref, ref_sq_mod, kind):
    if kind == "flat":
        return ref.IndexIVFFlat(D_DIM, NLIST, L2)
    if kind == "pq":
        idx = ref.IndexIVFPQ(D_DIM, NLIST, 4, 8, L2)
        idx.set_pq_cp(niter=4)
        return idx
    return ref_sq_mod.IndexIVFScalarQuantizer(D_DIM, NLIST, ref_sq_mod.QT_8bit, L2, True)


@pytest.mark.parametrize("kind", ["flat", "pq", "sq"])
def test_ivf_add_drops_unassignable_rows(ref, request, kind):
    """add / add_with_ids: a row with no coarse result (inf, NaN or an overflowing coordinate under L2) is not stored;
    every other row goes to its best centroid, ties to the smaller list number"""
    sq = request.getfixturevalue("ref_sq") if kind == "sq" else None
    rs = np.random.RandomState(2)
    xt = rs.randint(-3, 4, (2000, D_DIM)).astype(np.float32)
    idx = _ivf_cases(ref, sq, kind)
    idx.set_cp(niter=4)
    idx.train(xt)
    # integer centroids: every coarse distance is exact, so the model's assignment is the reference's
    idx.set_centroids(xt[:NLIST] + 1)
    cent = idx.centroids()
    n = 300
    xb, where = rm.database(rs, n, D_DIM, L2, n - 40, positions=[0, n - 1, 5])
    ids = rs.permutation(n).astype(np.int64) * 3 + 7
    for with_ids in (False, True):
        idx.reset()
        if with_ids:
            idx.add_with_ids(xb, ids)
            want = rm.ivf_lists(xb, ids, cent, L2)
        else:
            idx.add(xb)
            want = rm.ivf_lists(xb, np.arange(n), cent, L2)
        assert idx.ntotal == n  # the reference counts every row
        got = [idx.get_list(l)[1] for l in range(NLIST)]
        for l in range(NLIST):
            np.testing.assert_array_equal(got[l], want[l], err_msg="%s list %d" % (kind, l))
        assert sum(g.size for g in got) == n - where.size


@pytest.mark.parametrize("kind", ["flat", "pq", "sq"])
@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_ivf_special_queries_have_no_result(ref, request, kind, metric):
    """a query with a NaN coordinate (and under L2 an inf or overflowing one) probes nothing and gets nothing"""
    sq = request.getfixturevalue("ref_sq") if kind == "sq" else None
    rs = np.random.RandomState(3)
    xt = rs.randint(-3, 4, (2000, D_DIM)).astype(np.float32)
    if kind == "flat":
        idx = ref.IndexIVFFlat(D_DIM, NLIST, metric)
    elif kind == "pq":
        idx = ref.IndexIVFPQ(D_DIM, NLIST, 4, 8, metric)
        idx.set_pq_cp(niter=4)
    else:
        idx = sq.IndexIVFScalarQuantizer(D_DIM, NLIST, sq.QT_8bit, metric, True)
    idx.set_cp(niter=4)
    idx.train(xt)
    idx.add(xt[:500])
    idx.set_nprobe(NLIST)
    xq = rm.special_queries(D_DIM, metric)
    for k in (1, 10):
        D, I = idx.search(xq, k)
        assert np.all(I == -1), (kind, metric, I)
        assert np.all(D == (rm.FLT_MAX if metric == L2 else -rm.FLT_MAX))


@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_ivfflat_search(ref, metric):
    """IVF-Flat under the rule, bit for bit: special stored rows (only +inf / +FLT_MAX count under IP), queries with
    one infinite coordinate, and stored ids equal to -1, INT64_MAX and INT64_MIN"""
    rs = np.random.RandomState(4)
    xt = rs.randint(-3, 4, (2000, D_DIM)).astype(np.float32)
    idx = ref.IndexIVFFlat(D_DIM, NLIST, metric)
    idx.set_cp(niter=4)
    idx.train(xt)
    idx.set_centroids(xt[:NLIST] + 1)
    cent = idx.centroids()
    n = 300
    xb, _ = rm.database(rs, n, D_DIM, metric, n - 40, positions=[0, n - 1, 5])
    ids = np.arange(n, dtype=np.int64) + 100
    ids[[1, 50, 150]] = [-1, np.iinfo(np.int64).max, np.iinfo(np.int64).min]
    idx.add_with_ids(xb, ids)
    lists_ids = [idx.get_list(l)[1] for l in range(NLIST)]
    lists_x = [idx.get_list(l)[0].view(np.float32).reshape(-1, D_DIM) for l in range(NLIST)]
    want = rm.ivf_lists(xb, ids, cent, metric)
    for l in range(NLIST):
        np.testing.assert_array_equal(lists_ids[l], want[l])
    xq = rm.queries(rs, 6, D_DIM, metric)
    if metric == IP:
        xq[4, 5] = np.inf
        xq[5, 6] = -np.inf
    for nprobe in (1, 3, NLIST):
        idx.set_nprobe(nprobe)
        for k in (5, 400):
            D, I = idx.search(xq, k)
            _assert_same(D, I, *rm.ivfflat_search(xq, k, nprobe, cent, lists_x, lists_ids, metric), metric)
