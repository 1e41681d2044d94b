"""Every selecting path against the reference's result rule (oracle/oracle_rule_np.py, itself checked against the
reference in test_result_rule_oracle.py): a candidate is a result only if its distance is strictly better than the
missing-result sentinel (dis < FLT_MAX for L2, dis > -FLT_MAX for inner product), NaN never; empty slots are
(+-FLT_MAX, -1); the IVF coarse quantiser stores no vector it cannot assign; and a stored id is returned whatever
its value.  The data makes every distance exact in fp32 whatever the summation order, so Flat and IVF-Flat must equal
the model bit for bit, and every path must give the same answer for the same query."""
import numpy as np
import pytest

import faiss_b200 as fb
from oracle import oracle_rule_np as rm

pytestmark = pytest.mark.gpu

L2, IP = rm.METRIC_L2, rm.METRIC_INNER_PRODUCT
I64_MAX, I64_MIN = np.iinfo(np.int64).max, np.iinfo(np.int64).min

N_FLAT = 40000  # the tensor-core paths need >= 32768 rows (k > 1) and 16 queries
KS = (1, 10, 1024, 2048)
# first and last rows, inside the first tile, and both sides of the exact kernel's database splits at nq <= 5
# (576 rows per split for k <= 1024, 1152 for k = 2048)
POSITIONS = [0, 1, 5, 63, 64, 575, 576, 577, 1151, 1152, 1153, 2303, 2304, N_FLAT - 2, N_FLAT - 1]


def _bits(a):
    # + 0 turns -0 into +0: the sign of an exact zero depends on the summation order
    return np.ascontiguousarray(np.asarray(a, np.float32) + np.float32(0)).view(np.uint32)


def _same(D, I, Dm, Im, what):
    np.testing.assert_array_equal(np.asarray(I), Im, err_msg=what)
    np.testing.assert_array_equal(_bits(D), _bits(Dm), err_msg=what)


def _same_cut(D, I, Dm, Im, groups, what):
    """_same, except for a tie group cut at rank k: the IVF scans keep such a group's members by list position and the
    model by id, so there the ids must be distinct members of the group (groups[q]: {distance bits: candidate ids},
    -1 included).  A cut group holding a stored -1 leaves the number of results open, so only the ranks before it
    are compared."""
    Db, Dmb = _bits(D), _bits(Dm)
    I = np.asarray(I)
    for q in range(Dm.shape[0]):
        if Im[q, -1] == -1:
            np.testing.assert_array_equal(I[q], Im[q], err_msg="%s q=%d" % (what, q))
            np.testing.assert_array_equal(Db[q], Dmb[q], err_msg="%s q=%d" % (what, q))
            continue
        v = Dmb[q, -1]
        before = Dmb[q] != v
        np.testing.assert_array_equal(Db[q][before], Dmb[q][before], err_msg="%s q=%d" % (what, q))
        np.testing.assert_array_equal(I[q][before], Im[q][before], err_msg="%s q=%d" % (what, q))
        members = groups[q][int(v)]
        if -1 in members:
            continue
        np.testing.assert_array_equal(Db[q], Dmb[q], err_msg="%s q=%d" % (what, q))
        cut = I[q][~before]
        assert len(set(cut.tolist())) == cut.size and set(cut.tolist()) <= members, (what, q, cut, members)


def _groups(D, I):
    """per query: {distance bits: set of ids} over all candidates"""
    out = []
    for q in range(D.shape[0]):
        g = {}
        for v, i in zip(_bits(D[q]).tolist(), np.asarray(I[q]).tolist()):
            g.setdefault(v, set()).add(i)
        out.append(g)
    return out


def _model_all_k(xq, stored, metric, ids=None):
    dis = rm.distances(xq, stored, metric)
    ids = np.arange(stored.shape[0], dtype=np.int64) if ids is None else ids
    out = {}
    for k in KS:
        r = [rm.select(dis[q], ids, k, metric) for q in range(xq.shape[0])]
        out[k] = (np.stack([a for a, _ in r]), np.stack([b for _, b in r]))
    return out


def _flat_data(metric, d, fill, seed):
    rs = np.random.RandomState(seed)
    # pad: fewer ordinary rows than k (every list is padded); rank: most rows ordinary
    n_ord = 7 if fill == "pad" else N_FLAT - 600
    xb, where = rm.database(rs, N_FLAT, d, metric, n_ord, positions=POSITIONS)
    xq = rm.queries(rs, 16, d, metric)
    return xb, xq, where


# ----------------------------------------------------------------------------------------------------------------
# Flat: exact kernel (list and k = 1 packed argmin, database split), tensor-core paths (fp16 and int8 scoring,
# streaming argmin), compacted selector search, IndexShards, DistributedIndexShards
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fill", ["pad", "rank"])
@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_flat_paths(res, metric, d, fp16, fill):
    xb, xq, where = _flat_data(metric, d, fill, seed=d + 2 * fp16 + (fill == "pad"))
    stored = xb.astype(np.float16).astype(np.float32) if fp16 else xb
    qs = xq.astype(np.float16).astype(np.float32) if fp16 else xq  # useFloat16 rounds the queries too
    want = _model_all_k(qs, stored, metric)
    idx = fb.GpuIndexFlat(res, d, metric, use_tensor_cores=True, use_float16=fp16)
    idx.add(xb)
    tc_seen = set()
    for k in KS:
        Dm, Im = want[k]
        # tensor-core paths (16 queries; k = 1 is the streaming argmin)
        idx.setUseTensorCores(True)
        D, I = idx.search(xq, k)
        if idx.lastSearchInfo()["tensor_cores"]:
            tc_seen.add(idx.lastSearchOperandBits())
        _same(D, I, Dm, Im, "tensor cores k=%d" % k)
        # exact kernel: 16 queries, and 5 queries (database split); k = 1 is the packed argmin
        idx.setUseTensorCores(False)
        D, I = idx.search(xq, k)
        _same(D, I, Dm, Im, "exact k=%d" % k)
        D, I = idx.search(xq[:5], k)
        _same(D, I, Dm[:5], Im[:5], "exact split k=%d" % k)
    # non-finite and huge rows make the int8 residual norms non-finite, so such a database always scores in fp16
    assert tc_seen == {16}, tc_seen


@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_flat_selector_compacted(res, metric):
    """a selector keeping at most 1 row in 40 searches the gathered rows with the exact kernel"""
    d = 64
    xb, xq, _ = _flat_data(metric, d, "rank", seed=21)
    lo, hi = 500, 1400  # holds special rows at 575-577 and 1151-1153
    idx = fb.GpuIndexFlat(res, d, metric)
    idx.add(xb)
    params = fb.SearchParameters(sel=fb.IDSelectorRange(lo, hi))
    ids = np.arange(lo, hi, dtype=np.int64)
    dis = rm.distances(xq, xb[lo:hi], metric)
    for k in (1, 10, 1024):
        D, I = idx.search(xq, k, params=params)
        r = [rm.select(dis[q], ids, k, metric) for q in range(xq.shape[0])]
        _same(D, I, np.stack([a for a, _ in r]), np.stack([b for _, b in r]), "compacted k=%d" % k)


@pytest.mark.parametrize("fill", ["pad", "rank"])
@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_flat_shards(res, metric, fill):
    """IndexShards over two Flat shards on one device (merge_knn_results: a negative id is a missing result), and a
    one-rank DistributedIndexShards (pooled thresholds on the tensor-core path)"""
    import torch  # noqa: F401  (maps PyTorch's NCCL, which the library then uses)

    d = 64
    xb, xq, _ = _flat_data(metric, d, fill, seed=31 + (fill == "pad"))
    want = _model_all_k(xq, xb, metric)
    # shards of >= 32768 rows keep the tensor-core path inside each shard
    xb2 = np.concatenate([xb, xb[:2 * 32768 - N_FLAT]])
    want2 = _model_all_k(xq, xb2, metric)
    shards = fb.IndexShards(d, threaded=False, successive_ids=True)
    parts = []
    for s in range(2):
        p = fb.GpuIndexFlat(res, d, metric)
        p.add(xb2[s * 32768:(s + 1) * 32768])
        parts.append(p)
        shards.add_shard(p)
    for k in KS:
        D, I = shards.search(xq, k)
        _same(D, I, *want2[k], "IndexShards k=%d" % k)
    full = fb.GpuIndexFlat(res, d, metric)
    full.add(xb)
    try:
        res.ncclInitAll([0])
    except fb.FaissError as e:
        if "NCCL unavailable" in str(e):
            pytest.skip("NCCL cannot be loaded: %s" % e)
        raise
    dist = fb.DistributedIndexShards(res, full)
    for k in KS:
        D, I = dist.search(xq, k)
        _same(D, I, *want[k], "DistributedIndexShards k=%d" % k)


@pytest.mark.parametrize("layout", ["row", "col"])
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_bfknn(res, metric, dtype, layout):
    import torch

    d = 64
    rs = np.random.RandomState(41)
    n = 5000
    xb, where = rm.database(rs, n, d, metric, 2000, positions=[0, 1, 63, 64, n - 1])
    xq = rm.queries(rs, 5, d, metric)
    if dtype == "bf16":
        tq, tb = torch.from_numpy(xq).bfloat16(), torch.from_numpy(xb).bfloat16()
        qs, stored = tq.float().numpy(), tb.float().numpy()
        if layout == "col":
            tq, tb = tq.t().contiguous().t(), tb.t().contiguous().t()
        aq, ab = tq.cuda(), tb.cuda()
    else:
        qs, stored = xq, xb
        aq, ab = (np.asfortranarray(xq), np.asfortranarray(xb)) if layout == "col" else (xq, xb)
    dis = rm.distances(qs, stored, metric)
    ids = np.arange(n, dtype=np.int64)
    for k in (1, 10, 2048):
        D, I = fb.knn_gpu(res, aq, ab, k, metric=metric)
        if dtype == "bf16":
            D, I = D.cpu().numpy(), I.cpu().numpy()
        r = [rm.select(dis[q], ids, k, metric) for q in range(qs.shape[0])]
        _same(D, I, np.stack([a for a, _ in r]), np.stack([b for _, b in r]), "knn_gpu k=%d" % k)


# ----------------------------------------------------------------------------------------------------------------
# IVF
# ----------------------------------------------------------------------------------------------------------------
NLIST = 8
IVF_KINDS = [
    ("flat_d128", "flat", {"d": 128}),  # the d % 128 == 0 scan
    ("flat_d36", "flat", {"d": 36}),  # the generic scan
    ("pq8_m8", "pq", {"M": 8, "nbits": 8}),  # flat layout
    ("pq8_m16", "pq", {"M": 16, "nbits": 8}),  # interleaved scan
    ("pq4_m8", "pq", {"M": 8, "nbits": 4}),
    ("pq5_m8", "pq", {"M": 8, "nbits": 5}),
    ("pq6_m8", "pq", {"M": 8, "nbits": 6}),
    ("sq8", "sq", {"qtype": 0}),
    ("sq4", "sq", {"qtype": 1}),
    ("sq8u", "sq", {"qtype": 2}),
    ("sqfp16", "sq", {"qtype": 4}),
    ("sq8direct", "sq", {"qtype": 5}),
]


def _ivf(res, kind, p, metric):
    d = p.get("d", 64)
    if kind == "flat":
        idx = fb.GpuIndexIVFFlat(res, d, NLIST, metric)
    elif kind == "pq":
        idx = fb.GpuIndexIVFPQ(res, d, NLIST, p["M"], p["nbits"], metric, interleaved_layout=p["nbits"] != 8)
        idx.setPQClustering(niter=4)
    else:
        idx = fb.GpuIndexIVFScalarQuantizer(res, d, NLIST, p["qtype"], metric, True)
    idx.setClustering(niter=4)
    rs = np.random.RandomState(5)
    lo = 0 if kind == "sq" and p["qtype"] == 5 else -3
    idx.train(rs.randint(lo, 4, (3000, d)).astype(np.float32))
    # integer centroids: every coarse distance is exact, so the model's assignment and probes are the index's
    idx.setCoarseCentroids(rs.randint(lo, 4, (NLIST, d)).astype(np.float32))
    return idx, d


def _ivf_db(d, metric, n=400, seed=6):
    rs = np.random.RandomState(seed)
    xb, where = rm.database(rs, n, d, metric, n - 48, positions=[0, 1, 31, 32, n - 1])
    return xb, where, rs


def _empty(D, I, metric, what):
    assert np.all(np.asarray(I) == -1), what
    assert np.all(np.asarray(D) == (rm.FLT_MAX if metric == L2 else -rm.FLT_MAX)), what


def _all_searches(idx, xq, k, assign, cdis):
    """(name, D, I) of search, search_preassigned, search_and_reconstruct and search_and_return_codes"""
    out = [("search",) + tuple(idx.search(xq, k))]
    out.append(("search_preassigned",) + tuple(idx.search_preassigned(xq, k, assign, cdis)))
    D, I, _ = idx.search_and_reconstruct(xq, k)
    out.append(("search_and_reconstruct", D, I))
    D, I, _ = idx.search_and_return_codes(xq, k)
    out.append(("search_and_return_codes", D, I))
    return out


@pytest.mark.parametrize("name,kind,p", IVF_KINDS, ids=[c[0] for c in IVF_KINDS])
def test_ivf_add_and_special_queries(res, name, kind, p):
    """L2: add / add_with_ids store no row the coarse quantiser cannot assign (ntotal still counts it); the index then
    answers every query as an index built from the ordinary rows alone; queries with a NaN, inf or overflowing
    coordinate get no result from any search entry point"""
    idx, d = _ivf(res, kind, p, L2)
    cent = idx.getCoarseCentroids()
    coarse = fb.GpuIndexFlat(res, d, L2)  # the coarse quantiser's search, for search_preassigned
    coarse.add(cent)
    xb, where, rs = _ivf_db(d, L2)
    n = xb.shape[0]
    keep = np.setdiff1d(np.arange(n), where)
    ids = rs.permutation(n).astype(np.int64) * 5 + 3
    xq = rm.queries(rs, 6, d, L2)
    idx.nprobe = 3
    for with_ids in (False, True):
        idx.reset()
        lab = ids if with_ids else np.arange(n, dtype=np.int64)
        if with_ids:
            idx.add_with_ids(xb, ids)
        else:
            idx.add(xb)
        assert idx.ntotal == n
        want = rm.ivf_lists(xb, lab, cent, L2)
        for l in range(NLIST):
            np.testing.assert_array_equal(idx.getListIndices(l), want[l], err_msg="%s list %d" % (name, l))
        Dc, Ic = coarse.search(xq, 3)
        got = {k: _all_searches(idx, xq, k, Ic, Dc) for k in (10, 400)}
        # the same index holding only the ordinary rows
        idx.reset()
        idx.add_with_ids(xb[keep], lab[keep])
        for k in (10, 400):
            D0, I0 = idx.search(xq, k)
            for what, D, I in got[k]:
                _same(D, I, D0, I0, "%s %s k=%d with_ids=%d" % (name, what, k, with_ids))
    xs = rm.special_queries(d, L2)
    Dc, Ic = coarse.search(xs, 3)
    _empty(Dc, Ic, L2, "coarse search of the special queries")
    for k in (1, 10):
        for what, D, I in _all_searches(idx, xs, k, Ic, Dc):
            _empty(D, I, L2, "%s %s k=%d" % (name, what, k))


@pytest.mark.parametrize("name,kind,p", IVF_KINDS, ids=[c[0] for c in IVF_KINDS])
def test_ivf_ip_nan_queries(res, name, kind, p):
    idx, d = _ivf(res, kind, p, IP)
    rs = np.random.RandomState(7)
    idx.add(rs.randint(-3, 4, (400, d)).astype(np.float32))
    idx.nprobe = NLIST
    xs = rm.special_queries(d, IP)
    Dc = np.full((xs.shape[0], NLIST), -rm.FLT_MAX, np.float32)
    Ic = np.full((xs.shape[0], NLIST), -1, np.int64)
    for k in (1, 10):
        for what, D, I in _all_searches(idx, xs, k, Ic, Dc):
            _empty(D, I, IP, "%s %s k=%d" % (name, what, k))


@pytest.mark.parametrize("name,kind,p", IVF_KINDS, ids=[c[0] for c in IVF_KINDS])
@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_ivf_sentinel_ids(res, name, kind, p, metric):
    """stored ids INT64_MAX and INT64_MIN are returned at their rank like any other id; a stored -1 takes its rank and
    is then dropped, the results behind it moving up and the list padded at its end (CPU heap_reorder); at k below
    and above the number of results"""
    idx, d = _ivf(res, kind, p, metric)
    rs = np.random.RandomState(8)
    n = 400
    lo = 0 if kind == "sq" and p["qtype"] == 5 else -3
    xb = rs.randint(lo, 4, (n, d)).astype(np.float32)
    xq = xb[rs.choice(n, 6)].copy()  # queries on stored rows, so the special ids rank first for some of them
    special = np.array([-1, I64_MAX, I64_MIN], np.int64)
    at = rs.choice(n, 30, replace=False)
    plain = np.arange(n, dtype=np.int64) + 10
    ids = plain.copy()
    ids[at] = special[np.arange(at.size) % 3]
    xq[:3] = xb[at[:3]]
    idx.nprobe = 2
    idx.add_with_ids(xb, plain)
    Dall, Iall = idx.search(xq, 400)  # every result of each query (fewer than 400)
    assert (Iall == -1).any(axis=1).all()
    idx.reset()
    idx.add_with_ids(xb, ids)
    back = dict(zip(plain.tolist(), ids.tolist()))
    groups = []
    for q in range(xq.shape[0]):
        ok = Iall[q] != -1
        groups += _groups(Dall[q : q + 1][:, ok], np.array([[back[int(v)] for v in Iall[q][ok]]], np.int64))
    for k in (5, 400):
        # the expected answer: every result under its new id, ordered by (key, id), cut at k, then the -1 dropped
        D0 = np.full((xq.shape[0], k), rm.FLT_MAX if metric == L2 else -rm.FLT_MAX, np.float32)
        I0m = np.full((xq.shape[0], k), -1, np.int64)
        for q in range(xq.shape[0]):
            ok = Iall[q] != -1
            dq = Dall[q][ok]
            iq = np.array([back[int(v)] for v in Iall[q][ok]], np.int64)
            order = np.lexsort((iq, rm.keys_of(dq, metric)))[:k]
            order = order[iq[order] != -1]
            D0[q, : order.size] = dq[order]
            I0m[q, : order.size] = iq[order]
        D, I = idx.search(xq, k)
        _same_cut(D, I, D0, I0m, groups, "%s k=%d" % (name, k))
        D, I, _ = idx.search_and_reconstruct(xq, k)
        _same_cut(D, I, D0, I0m, groups, "%s search_and_reconstruct k=%d" % (name, k))
        D, I, _ = idx.search_and_return_codes(xq, k)
        _same_cut(D, I, D0, I0m, groups, "%s search_and_return_codes k=%d" % (name, k))
    for s in special[1:]:
        assert (I == s).any(), (name, s)
    assert not (I == -1).all(axis=1).any()


@pytest.mark.parametrize("d", [128, 36])
@pytest.mark.parametrize("metric", [L2, IP], ids=["l2", "ip"])
def test_ivfflat_model(res, metric, d):
    """IVF-Flat bit for bit against the model: stored special rows (under IP +inf and +FLT_MAX are results), IP
    queries with one infinite coordinate, sentinel-valued ids"""
    idx, _ = _ivf(res, "flat", {"d": d}, metric)
    cent = idx.getCoarseCentroids()
    xb, where, rs = _ivf_db(d, metric, seed=9)
    n = xb.shape[0]
    ids = np.arange(n, dtype=np.int64) + 100
    ids[[2, 50, 150]] = [-1, I64_MAX, I64_MIN]
    idx.add_with_ids(xb, ids)
    assert idx.ntotal == n
    want = rm.ivf_lists(xb, ids, cent, metric)
    lists_ids = [idx.getListIndices(l) for l in range(NLIST)]
    for l in range(NLIST):
        np.testing.assert_array_equal(lists_ids[l], want[l])
    lists_x = [idx.getListVectorData(l).view(np.float32).reshape(-1, d) for l in range(NLIST)]
    xq = rm.queries(rs, 8, d, metric)
    if metric == IP:
        xq[5, 7] = np.inf
        xq[6, 8] = -np.inf
        xq[7, d - 1] = np.inf
    for nprobe in (1, 3, NLIST):
        idx.nprobe = nprobe
        Dc, Ic = rm.knn(xq, cent, nprobe, metric)
        # every candidate with the stored -1 kept (as -2, an id nothing else holds), for the tie groups
        tagged = [np.where(li == -1, -2, li) for li in lists_ids]
        Df, If = rm.ivfflat_search(xq, n, nprobe, cent, lists_x, tagged, metric)
        groups = _groups(Df, np.where(If == -2, -1, If))
        for k in (5, 500):
            Dm, Im = rm.ivfflat_search(xq, k, nprobe, cent, lists_x, lists_ids, metric)
            for what, D, I in _all_searches(idx, xq, k, Ic, Dc):
                _same_cut(D, I, Dm, Im, groups, "%s nprobe=%d k=%d" % (what, nprobe, k))
