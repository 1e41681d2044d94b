"""Filtered search: SearchParameters::sel on GpuIndexFlat and the IVF indexes.

Flat results must equal the numpy restatement of IndexFlat search over the selected rows (bit-exact on integer
data), on the masked tensor-core path, the compacted path and the exact kernel alike.  IVF results must only hold
selected ids and equal an unfiltered search of a clone that holds only the selected entries of each list."""
import numpy as np
import pytest

from oracle import oracle_np as o
from oracle import oracle_sel_np as osel

pytestmark = pytest.mark.gpu

L2, IP, L1 = 1, 0, 2


def to_fb(spec):
    import faiss_b200 as fb

    kind = spec[0]
    if kind == "range":
        return fb.IDSelectorRange(spec[1], spec[2])
    if kind == "array":
        return fb.IDSelectorArray(spec[1])
    if kind == "batch":
        return fb.IDSelectorBatch(spec[1])
    if kind == "bitmap":
        return fb.IDSelectorBitmap(spec[1])
    if kind == "not":
        return fb.IDSelectorNot(to_fb(spec[1]))
    cls = {"and": fb.IDSelectorAnd, "or": fb.IDSelectorOr, "xor": fb.IDSelectorXOr}[kind]
    return cls(to_fb(spec[1]), to_fb(spec[2]))


def int_data(n, d, seed):
    return np.floor(np.random.RandomState(seed).rand(n, d) * 16).astype(np.float32)


def flat(res, d, metric, fp16=False, tc=True):
    import faiss_b200 as fb

    return fb.GpuIndexFlat(res, d, metric, use_tensor_cores=tc, use_float16=fp16)


def fsearch(idx, xq, k, spec):
    import faiss_b200 as fb

    sel = to_fb(spec) if spec is not None else None
    return idx.search(xq, k, params=fb.SearchParameters(sel=sel))


N, D = 40000, 64
SELS = osel.reference_selectors(N)


@pytest.fixture(scope="module")
def flat_data():
    return int_data(N, D, 1), int_data(64, D, 2)


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("name", list(SELS))
def test_flat_selectors_tensor_core_and_exact(res, flat_data, name, metric, fp16):
    xb, xq = flat_data
    idx = flat(res, D, metric, fp16)
    idx.add(xb)
    spec = SELS[name]
    rD, rI = osel.knn_flat_sel(xq, xb, 20, spec, metric)
    D_, I_ = fsearch(idx, xq, 20, spec)  # 64 queries: the tensor-core path (every selector keeps > 1/32 of the rows)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    assert np.array_equal(I_, rI) and np.array_equal(D_, rD)
    D_, I_ = fsearch(idx, xq[:8], 20, spec)  # 8 queries: the exact kernel
    assert idx.lastSearchInfo()["tensor_cores"] == 0
    assert np.array_equal(I_, rI[:8]) and np.array_equal(D_, rD[:8])


@pytest.mark.parametrize("k", [1, 10, 100])
@pytest.mark.parametrize("metric", [L2, IP])
def test_flat_paths_agree(res, flat_data, metric, k):
    """masked tensor-core path (50 %), compacted path (1 %), and an index holding only the selected rows"""
    xb, xq = flat_data
    idx = flat(res, D, metric)
    idx.add(xb)
    for frac, want_tc in ((0.5, 1), (0.01, 0)):
        rows = np.sort(np.random.RandomState(3).choice(N, int(N * frac), replace=False))
        spec = ("batch", rows)
        D_, I_ = fsearch(idx, xq, k, spec)
        assert idx.lastSearchInfo()["tensor_cores"] == want_tc
        sub = flat(res, D, metric)
        sub.add(xb[rows])
        sD, sI = sub.search(xq, k)
        sI = np.where(sI >= 0, rows[np.maximum(sI, 0)], -1)
        assert np.array_equal(I_, sI) and np.array_equal(D_, sD)
        rD, rI = osel.knn_flat_sel(xq, xb, k, spec, metric)
        assert np.array_equal(I_, rI) and np.array_equal(D_, rD)


@pytest.mark.parametrize("metric", [L2, IP])
def test_flat_padding_and_empty_selection(res, flat_data, metric):
    xb, xq = flat_data
    idx = flat(res, D, metric)
    idx.add(xb)
    big = np.finfo(np.float32).max if metric == L2 else -np.finfo(np.float32).max
    spec = ("range", 100, 105)  # k > s
    D_, I_ = fsearch(idx, xq, 20, spec)
    rD, rI = osel.knn_flat_sel(xq, xb, 20, spec, metric)
    assert np.array_equal(I_, rI) and np.array_equal(D_, rD)
    assert (I_[:, 5:] == -1).all() and (D_[:, 5:] == big).all()
    for spec in (("range", 7, 7), ("array", []), ("bitmap", np.zeros(4, np.uint8)), ("range", -5, 0)):
        D_, I_ = fsearch(idx, xq, 10, spec)
        assert (I_ == -1).all() and (D_ == big).all()


def test_flat_array_duplicates_and_out_of_range_ids(res, flat_data):
    xb, xq = flat_data
    idx = flat(res, D, L2)
    idx.add(xb)
    ids = np.array([5, 5, 7, 7, 7, N + 10, -3, 1000], dtype=np.int64)
    D_, I_ = fsearch(idx, xq, 6, ("array", ids))
    rD, rI = osel.knn_flat_sel(xq, xb, 6, ("array", np.array([5, 7, 1000])), L2)
    assert np.array_equal(I_, rI) and np.array_equal(D_, rD)


@pytest.mark.parametrize("fp16", [False, True])
def test_flat_l1(res, flat_data, fp16):
    xb, xq = flat_data
    idx = flat(res, D, L1, fp16)
    idx.add(xb)
    for name in ("Range", "Bitmap", "XOr"):
        rows = np.nonzero(osel.is_member(SELS[name], np.arange(N)))[0]
        D_, I_ = fsearch(idx, xq, 10, SELS[name])
        sub = flat(res, D, L1, fp16)
        sub.add(xb[rows])
        sD, sI = sub.search(xq, 10)
        assert np.array_equal(I_, rows[sI]) and np.array_equal(D_, sD)


def test_flat_callback_selector(res, flat_data):
    import faiss_b200 as fb

    xb, xq = flat_data
    idx = flat(res, D, L2)
    idx.add(xb)
    seen = []

    def keep(i):
        seen.append(i)
        return i % 7 == 3

    D_, I_ = idx.search(xq, 10, params=fb.SearchParameters(sel=fb.IDSelectorCallback(keep)))
    assert len(seen) == N  # once per stored row and call
    rD, rI = osel.knn_flat_sel(xq, xb, 10, ("array", np.arange(3, N, 7)), L2)
    assert np.array_equal(I_, rI) and np.array_equal(D_, rD)


def test_flat_paged_host_queries(res, flat_data):
    import faiss_b200 as fb

    xb, _ = flat_data
    xq = int_data(3000, D, 9)
    idx = flat(res, D, L2)
    idx.add(xb)
    spec = SELS["Or"]
    D0, I0 = fsearch(idx, xq, 10, spec)
    idx2 = fb.GpuIndexFlatL2(res, D)
    idx2.add(xb)
    idx2.setMinPagingSize(0)
    D1, I1 = fsearch(idx2, xq, 10, spec)
    assert np.array_equal(I0, I1) and np.array_equal(D0, D1)
    rD, rI = osel.knn_flat_sel(xq[:50], xb, 10, spec, L2)
    assert np.array_equal(I1[:50], rI) and np.array_equal(D1[:50], rD)


def test_flat_certificate_fallbacks_stay_exact(res):
    """near-duplicate rows: the tensor-core certificate fails for many queries, whose exact recompute must
    honour the selector too"""
    rs = np.random.RandomState(5)
    base = np.floor(rs.rand(16, D) * 16).astype(np.float32)
    xb = np.repeat(base, N // 16, axis=0)
    xb[np.arange(N), rs.randint(0, D, N)] += 1.0
    xq = base[rs.randint(0, 16, 64)]
    idx = flat(res, D, L2)
    idx.add(xb)
    spec = SELS["XOr"]
    D_, I_ = fsearch(idx, xq, 100, spec)
    info = idx.lastSearchInfo()
    assert info["tensor_cores"] == 1 and info["fallback_queries"] > 0
    rD, rI = osel.knn_flat_sel(xq, xb, 100, spec, L2)
    assert np.array_equal(I_, rI) and np.array_equal(D_, rD)


# ---------------------------------------------------------------------------------------------------- IVF
NI, DI, NLIST = 20000, 64, 32


def ivf_ids(n):
    return osel.ivf_ids(n)


def ivf_selectors(ids):
    return osel.ivf_selectors(ids)


# name: (kind, metric, options)
IVF_CASES = {
    "flat_l2": ("flat", L2, {}),
    "flat_ip": ("flat", IP, {}),
    "pq_m16_l2": ("pq", L2, {"M": 16}),
    "pq_m16_ip": ("pq", IP, {"M": 16}),
    "pq_m32_precomputed": ("pq", L2, {"M": 32, "precomputed": True}),
    "pq_m32_no_precomputed": ("pq", L2, {"M": 32, "precomputed": False}),
    "pq_m8_vector_major": ("pq", L2, {"M": 8}),
    "pq_m32_4bit_nibble": ("pq", L2, {"M": 32, "nbits": 4}),
    "pq_m16_6bit_packed": ("pq", IP, {"M": 16, "nbits": 6}),
    "sq_8bit": ("sq", L2, {"qtype": 0}),
    "sq_4bit_ip": ("sq", IP, {"qtype": 1}),
    "sq_6bit": ("sq", L2, {"qtype": 6}),
    "sq_fp16": ("sq", L2, {"qtype": 4}),
}


def make_ivf(res, kind, metric, opt):
    import faiss_b200 as fb

    if kind == "flat":
        return fb.GpuIndexIVFFlat(res, DI, NLIST, metric)
    if kind == "pq":
        nbits = opt.get("nbits", 8)
        idx = fb.GpuIndexIVFPQ(res, DI, NLIST, opt["M"], nbits, metric, interleaved_layout=nbits != 8)
        idx.setPrecomputedCodes(opt.get("precomputed", False))  # the same policy for the clone
        return idx
    return fb.GpuIndexIVFScalarQuantizer(res, DI, NLIST, opt["qtype"], metric)


def clone_selected(res, idx, kind, metric, opt, spec):
    """a copy of idx holding only the selected entries of each list"""
    sub = make_ivf(res, kind, metric, opt)
    sub.setCoarseCentroids(idx.getCoarseCentroids())
    if kind == "pq":
        sub.setPQCentroids(idx.getPQCentroids())
    if kind == "sq" and idx.getTrained().size:
        sub.setTrained(idx.getTrained())
    sub.setIsTrained(True)
    cs = idx._code_size()
    for l in range(NLIST):
        ids = idx.getListIndices(l)
        codes = idx.getListVectorData(l).reshape(-1, cs)
        keep = osel.is_member(spec, ids)
        sub.setList(l, codes[keep], ids[keep])
    return sub


def live_reference(idx, kind, metric, opt):
    """(oracle.ref_sel, the reference CPU index holding idx's centroids, quantiser and lists), or (None, None) where
    oracle/_ref was not built"""
    from oracle import ref_sel

    if not ref_sel.available():
        return None, None
    from oracle import ref, ref_pq, ref_sq

    if kind == "flat":
        r = ref.IndexIVFFlat(DI, NLIST, metric)
    elif kind == "pq":
        r = ref_pq.IndexIVFPQ(DI, NLIST, opt["M"], opt.get("nbits", 8), metric)
        r.set_pq_centroids(idx.getPQCentroids())
    else:
        r = ref_sq.IndexIVFScalarQuantizer(DI, NLIST, opt["qtype"], metric, True)
        if idx.getTrained().size:
            r.set_trained(idx.getTrained())
    r.set_centroids(idx.getCoarseCentroids())
    for l in range(NLIST):
        ids = idx.getListIndices(l)
        if ids.size:
            r.add_entries(l, ids, idx.getListVectorData(l))
    r.set_is_trained(True)
    return ref_sel, r


@pytest.fixture(scope="module")
def ivf_data():
    rs = np.random.RandomState(7)
    xb = np.floor(rs.rand(NI, DI) * 16).astype(np.float32)
    xq = np.floor(rs.rand(40, DI) * 16).astype(np.float32)
    return xb, xq, ivf_ids(NI)


@pytest.mark.parametrize("case", list(IVF_CASES))
def test_ivf_selectors(res, ivf_data, case):
    import faiss_b200 as fb

    kind, metric, opt = IVF_CASES[case]
    xb, xq, ids = ivf_data
    idx = make_ivf(res, kind, metric, opt)
    idx.setClustering(niter=4)
    if kind == "pq":
        idx.setPQClustering(niter=4)
    idx.train(xb)
    idx.add_with_ids(xb, ids)
    idx.nprobe = 2  # the per-call nprobe below must win
    ref_sel, ref = live_reference(idx, kind, metric, opt)
    k, nprobe = 30, 8
    for name, spec in ivf_selectors(ids).items():
        D_, I_ = idx.search(xq, k, params=fb.SearchParametersIVF(nprobe=nprobe, sel=to_fb(spec)))
        got = I_[I_ >= 0]
        assert osel.is_member(spec, got).all(), name
        sub = clone_selected(res, idx, kind, metric, opt, spec)
        sub.nprobe = nprobe
        sD, sI = sub.search(xq, k)
        o.compare_lists(sD, sI, D_, I_, eps=1e-5, pct_max_diff1=0.02, pct_max_diffN=0.01)
        if kind == "pq":
            # the interleaved layout rotates each entry's codes by its position in the list, so the order of the
            # table sums (and the last bit of a distance) follows the entry's position, which the clone changes
            np.testing.assert_allclose(np.sort(D_, axis=1), np.sort(sD, axis=1), rtol=1e-5, err_msg=name)
        else:
            assert np.array_equal(np.sort(D_, axis=1), np.sort(sD, axis=1)), name
        if ref is not None:  # the reference CPU index cloned from this one, with the same selector and nprobe
            rD, rI = ref_sel.search(ref, xq, k, spec, nprobe=nprobe)
            assert osel.is_member(spec, rI[rI != -1]).all(), name
            if kind == "flat":  # integer data: bit-exact distances; tie order is the scan's list order vs the CPU heap's
                assert osel.equal_up_to_ties(D_, I_, rD, rI), name
            else:
                o.compare_lists(rD, rI, D_, I_, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)
    # without a selector nothing changes
    D0, I0 = idx.search(xq, k, params=fb.SearchParametersIVF(nprobe=nprobe))
    D1, I1 = idx.search(xq, k, params=fb.SearchParametersIVF(nprobe=nprobe, sel=fb.IDSelectorNot(fb.IDSelectorRange(0, 0))))
    assert np.array_equal(D0, D1) and np.array_equal(I0, I1)


def test_ivf_callback_selector(res, ivf_data):
    import faiss_b200 as fb

    xb, xq, ids = ivf_data
    idx = fb.GpuIndexIVFFlat(res, DI, NLIST, L2)
    idx.setClustering(niter=4)
    idx.train(xb)
    idx.add_with_ids(xb, ids)
    seen = []

    def keep(i):
        seen.append(i)
        return i < 0

    D_, I_ = idx.search(xq, 10, params=fb.SearchParametersIVF(nprobe=8, sel=fb.IDSelectorCallback(keep)))
    assert sorted(seen) == sorted(ids.tolist())  # called for the stored entries only
    D2, I2 = idx.search(xq, 10, params=fb.SearchParametersIVF(nprobe=8, sel=to_fb(("range", -(1 << 62), 0))))
    assert np.array_equal(D_, D2) and np.array_equal(I_, I2)
    assert (I_[I_ != -1] < 0).all()


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_ivfflat_matches_reference_fixture(res, metric):
    """IVF-Flat with the reference CPU's centroids and lists (tests/golden/idselector.npz): the filtered results of
    the reference IndexIVFFlat, whatever is built on this machine"""
    import os

    import faiss_b200 as fb
    from tests.golden import make_golden_idselector as g

    f = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "idselector.npz"))
    ids, assign = f["ivf_ids"], f["ivf_%s_assign" % metric]
    idx = fb.GpuIndexIVFFlat(res, g.D, g.NLIST, g.METRICS[metric])
    idx.setCoarseCentroids(f["ivf_%s_centroids" % metric])
    idx.setIsTrained(True)
    for l in range(g.NLIST):
        m = assign == l
        idx.setList(l, f["xi"][m].view(np.uint8), ids[m])
    for name, spec in osel.ivf_selectors(ids).items():
        D_, I_ = idx.search(f["xq"], g.K, params=fb.SearchParametersIVF(nprobe=g.NPROBE, sel=to_fb(spec)))
        rD, rI = f["ivf_%s_%s_D" % (metric, name)], f["ivf_%s_%s_I" % (metric, name)]
        # integer data: bit-exact distances; the scan breaks ties by list position, the CPU by its heap order
        assert osel.equal_up_to_ties(D_, I_, rD, rI), name


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_flat_matches_reference_fixture(res, metric):
    """GpuIndexFlat (tensor cores off: 20 queries) on the fixture's rows: the reference IndexFlat's filtered results"""
    import os

    from tests.golden import make_golden_idselector as g

    f = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "idselector.npz"))
    idx = flat(res, g.D, g.METRICS[metric])
    idx.add(f["xf"])
    for name, spec in osel.reference_selectors(g.NF).items():
        D_, I_ = fsearch(idx, f["xq"], g.K, spec)
        rD, rI = f["flat_%s_%s_D" % (metric, name)], f["flat_%s_%s_I" % (metric, name)]
        if metric == "l2":
            assert np.array_equal(I_, rI) and np.array_equal(D_, rD), name
        else:  # the CPU's inner-product heap puts a tie group in decreasing id order
            assert osel.equal_up_to_ties(D_, I_, rD, rI), name


def test_flat_tensor_core_fewer_selected_than_k(res, flat_data):
    """N/32 < s < k stays on the tensor-core path: the rounds keep a -inf threshold and the results pad"""
    xb, xq = flat_data
    idx = flat(res, D, L2)
    idx.add(xb)
    rows = np.sort(np.random.RandomState(8).choice(N, N // 32 + 50, replace=False))
    k = 2048
    D_, I_ = fsearch(idx, xq, k, ("batch", rows))
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    rD, rI = osel.knn_flat_sel(xq, xb, k, ("batch", rows), L2)
    assert np.array_equal(I_, rI) and np.array_equal(D_, rD)
    assert (I_[:, rows.size :] == -1).all()


def test_callback_exception_is_raised(res, flat_data):
    import faiss_b200 as fb

    xb, xq = flat_data
    idx = flat(res, D, L2)
    idx.add(xb[:1000])

    def bad(i):
        raise KeyError(i)

    with pytest.raises(KeyError):
        idx.search(xq, 5, params=fb.SearchParameters(sel=fb.IDSelectorAnd(fb.IDSelectorRange(0, 9), fb.IDSelectorCallback(bad))))
    D_, I_ = fsearch(idx, xq, 5, ("range", 0, 9))  # the index stays usable
    assert (I_ >= 0).all() and (I_ < 9).all()
