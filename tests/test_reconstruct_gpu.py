"""IVF retrieval on the GPU (reconstruct_n / reconstruct_batch / reconstruct, search_and_reconstruct,
search_and_return_codes) and GpuIndexFlat.search_and_reconstruct, against the numpy restatement of the CPU
IndexIVF (oracle/oracle_recons_np.py) and, where oracle/_ref was built, the reference's own reconstruct_n."""
import numpy as np
import pytest

import faiss_b200 as fb
from oracle import oracle_recons_np as rn
from oracle import oracle_sq_np as so

pytestmark = pytest.mark.gpu

NLIST, K = 16, 10

# (name, kind, parameters): every stored layout of the decoder
LAYOUTS = [
    ("flat", rn.FLAT, {}),
    ("pq8_m8", rn.PQ, {"M": 8, "nbits": 8}),  # vector-major
    ("pq8_m16", rn.PQ, {"M": 16, "nbits": 8}),  # interleaved by 32
    ("pq8_m32", rn.PQ, {"M": 32, "nbits": 8}),
    ("pq4_m8", rn.PQ, {"M": 8, "nbits": 4}),  # packed bitstring
    ("pq4_m32", rn.PQ, {"M": 32, "nbits": 4}),  # nibble pairs, interleaved
    ("pq4_m64", rn.PQ, {"M": 64, "nbits": 4}),
    ("pq5_m8", rn.PQ, {"M": 8, "nbits": 5}),
    ("pq6_m8", rn.PQ, {"M": 8, "nbits": 6}),
] + [("sq%d_%s_d%d" % (q, "res" if r else "nores", dd), rn.SQ, {"qtype": q, "by_residual": r, "d": dd})
     for q in range(7) for r in (True, False) for dd in (40, 36)]


def _data(rs, n, d, params):
    if params.get("qtype") == so.QT_8bit_direct:
        return np.floor(rs.rand(n, d) * 256).astype(np.float32)
    return (rs.rand(n, d) * 4).astype(np.float32)


def _build(res, kind, params, metric=fb.METRIC_L2, seed=0, n=3000):
    d = params.get("d", 64)
    rs = np.random.RandomState(seed)
    if kind == rn.FLAT:
        idx = fb.GpuIndexIVFFlat(res, d, NLIST, metric)
    elif kind == rn.PQ:
        idx = fb.GpuIndexIVFPQ(res, d, NLIST, params["M"], params["nbits"], metric, interleaved_layout=params["nbits"] != 8)
        idx.setPQClustering(niter=4)
    else:
        idx = fb.GpuIndexIVFScalarQuantizer(res, d, NLIST, params["qtype"], metric, params["by_residual"])
    idx.setClustering(niter=4)
    xb = _data(rs, n, d, params)
    idx.train(xb)
    # ids in random order, with some stored twice (different vectors under one id)
    ids = rs.permutation(n).astype(np.int64) + 1000
    ids[n - 50:] = ids[:50]
    idx.add_with_ids(xb, ids)
    return idx, xb, ids, d


def _lists(idx):
    return [idx.getListVectorData(l) for l in range(idx.nlist)], [idx.getListIndices(l) for l in range(idx.nlist)]


def _kw(idx, kind, params):
    if kind == rn.PQ:
        return {"M": params["M"], "nbits": params["nbits"], "pq": idx.getPQCentroids()}
    if kind == rn.SQ:
        return {"qtype": params["qtype"], "by_residual": params["by_residual"], "trained": idx.getTrained()}
    return {}


def _expected_all(idx, kind, params, d):
    """{id: vector of the entry last in (list, offset) order}, and {(list, offset): vector}"""
    codes, ids = _lists(idx)
    cent = idx.getCoarseCentroids()
    last, entry = {}, {}
    for l in range(idx.nlist):
        if ids[l].size == 0:
            continue
        x = rn.reconstruct_list(kind, codes[l], l, d, cent, **_kw(idx, kind, params))
        for off, i in enumerate(ids[l]):
            last[int(i)] = x[off]
            entry[(l, off)] = x[off]
    return last, entry, codes, ids


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("name,kind,params", LAYOUTS, ids=[l[0] for l in LAYOUTS])
def test_reconstruct_layouts(res, name, kind, params):
    idx, xb, ids, d = _build(res, kind, params)
    last, entry, codes, lids = _expected_all(idx, kind, params, d)
    lo = int(ids.min())
    ni = int(ids.max()) + 1 - lo

    # reconstruct_n over the id range: last-wins; rows of ids not stored are left as they are (pre-filled with 7)
    # (the CPU precondition i0 + ni <= ntotal: ids start at 1000, so query [0, ntotal) and check the stored part)
    n_tot = idx.ntotal
    out = np.full((n_tot, d), 7.0, np.float32)
    fb.check(fb.lib.faiss_Index_reconstruct_n(idx._h, fb.ctypes.c_int64(0), fb.ctypes.c_int64(n_tot), fb._ptr(out, fb._c_f)))
    for i in range(n_tot):
        if i in last:
            assert np.array_equal(_bits(out[i]), _bits(last[i])), (name, i)
        else:
            assert np.all(out[i] == 7.0)

    # reconstruct_batch on random keys (with repeats), and reconstruct
    rs = np.random.RandomState(1)
    keys = rs.choice(ids, 200).astype(np.int64)
    R = idx.reconstruct_batch(keys)
    E = np.stack([last[int(k)] for k in keys])
    assert np.array_equal(_bits(R), _bits(E)), name
    assert np.array_equal(_bits(idx.reconstruct(int(keys[0]))), _bits(E[0]))

    # search_and_reconstruct: D, I as search; R the returned entry
    xq = xb[rs.choice(xb.shape[0], 40)] + np.float32(0.01)
    idx.nprobe = 4
    D0, I0 = idx.search(xq, K)
    D, I, R = idx.search_and_reconstruct(xq, K)
    assert np.array_equal(D, D0) and np.array_equal(I, I0), name
    vecs = {}
    for (l, off), v in entry.items():
        vecs.setdefault(int(lids[l][off]), []).append(v)
    for q in range(xq.shape[0]):
        for j in range(K):
            assert any(np.array_equal(_bits(R[q, j]), _bits(v)) for v in vecs[int(I[q, j])]), (name, q, j)

    # search_and_return_codes: the CPU bytes, with and without the list number
    D2, I2, C = idx.search_and_return_codes(xq, K)
    D3, I3, CL = idx.search_and_return_codes(xq, K, include_listnos=True)
    assert np.array_equal(D2, D0) and np.array_equal(I3, I0)
    by_id = {}
    for l in range(idx.nlist):
        for off, i in enumerate(lids[l]):
            by_id.setdefault(int(i), []).append((l, codes[l].reshape(-1, C.shape[2])[off]))
    for q in range(xq.shape[0]):
        for j in range(K):
            opts = by_id[int(I[q, j])]
            assert any(np.array_equal(C[q, j], c) for _, c in opts)
            assert any(np.array_equal(CL[q, j], np.concatenate([rn.encode_listno(l, idx.nlist), c])) for l, c in opts)


def test_duplicates_return_the_searched_entry(res):
    # IVF-Flat, two entries under one id far apart: R is the vector whose distance the search returned
    d = 32
    idx = fb.GpuIndexIVFFlat(res, d, 4)
    rs = np.random.RandomState(3)
    xt = rs.rand(400, d).astype(np.float32)
    idx.setClustering(niter=3)
    idx.train(xt)
    a = np.zeros((1, d), np.float32)
    b = np.full((1, d), 3.0, np.float32)
    idx.add_with_ids(np.concatenate([xt, a, b]), np.concatenate([np.arange(400), [7000, 7000]]).astype(np.int64))
    idx.nprobe = 4
    for q, want in ((a, a), (b, b)):
        D, I, R = idx.search_and_reconstruct(q, 1)
        assert I[0, 0] == 7000 and D[0, 0] == 0.0
        assert np.array_equal(R[0, 0], want[0])
    # reconstruct follows the CPU's rule: the entry last in (list, offset) order wins
    last = [idx.getListVectorData(l).view(np.float32).reshape(-1, d)[off]
            for l in range(idx.nlist) for off, i in enumerate(idx.getListIndices(l)) if i == 7000][-1]
    assert np.array_equal(idx.reconstruct(7000), last)


def test_heavy_ties_equal_search(res):
    # integer data with every vector stored several times: many equal distances, ids not in arena order
    d = 16
    rs = np.random.RandomState(4)
    base = np.floor(rs.rand(200, d) * 3).astype(np.float32)
    xb = np.concatenate([base] * 5)
    ids = rs.permutation(xb.shape[0]).astype(np.int64)
    for make in (lambda: fb.GpuIndexIVFFlat(res, d, 8),
                 lambda: fb.GpuIndexIVFScalarQuantizer(res, d, 8, so.QT_8bit_direct, fb.METRIC_L2, False),
                 lambda: fb.GpuIndexIVFPQ(res, d, 8, 16, 8)):
        idx = make()
        idx.setClustering(niter=3)
        idx.train(xb)
        idx.add_with_ids(xb, ids)
        for nprobe in (1, 3, 8):
            idx.nprobe = nprobe
            xq = np.floor(rs.rand(64, d) * 3).astype(np.float32)
            D0, I0 = idx.search(xq, 20)
            D, I, R = idx.search_and_reconstruct(xq, 20)
            assert np.array_equal(D, D0) and np.array_equal(I, I0)


def test_missing_results_and_keys(res):
    idx, xb, ids, d = _build(res, rn.SQ, {"qtype": so.QT_8bit, "by_residual": True, "d": 40}, n=300)
    idx.nprobe = 2
    # k > what the probed lists hold: -1 results are all 0xFF, codes too
    D, I, R = idx.search_and_reconstruct(xb[:5], 200)
    miss = I < 0
    assert miss.any()
    assert np.all(_bits(R[miss]) == 0xFFFFFFFF)
    _, I2, C = idx.search_and_return_codes(xb[:5], 200, include_listnos=True)
    assert np.all(C[I2 < 0] == 0xFF)
    # under a selector: only the selected ids come back, the rest are -1 / 0xFF
    sel = fb.IDSelectorRange(int(ids.min()), int(ids.min()) + 20)
    p = fb.SearchParametersIVF(nprobe=NLIST, sel=sel)
    D0, I0 = idx.search(xb[:5], 30, params=p)
    D, I, R = idx.search_and_reconstruct(xb[:5], 30, params=p)
    assert np.array_equal(D, D0) and np.array_equal(I, I0)
    assert np.all(_bits(R[I < 0]) == 0xFFFFFFFF)
    assert np.all((I[I >= 0] >= ids.min()) & (I[I >= 0] < ids.min() + 20))
    # a missing key throws and writes nothing
    out = np.full((3, d), 5.0, np.float32)
    keys = np.array([ids[0], 10 ** 9, ids[1]], np.int64)
    with pytest.raises(fb.FaissError, match="key not found"):
        fb.check(fb.lib.faiss_Index_reconstruct_batch(idx._h, fb.ctypes.c_int64(3), fb._ptr(keys, fb._c_i64), fb._ptr(out, fb._c_f)))
    assert np.all(out == 5.0)


def test_torch_and_paged_host_queries(res):
    torch = pytest.importorskip("torch")
    idx, xb, ids, d = _build(res, rn.PQ, {"M": 16, "nbits": 8}, n=4000)
    idx.nprobe = 4
    xq = xb[:300] + np.float32(0.01)
    D0, I0, R0 = idx.search_and_reconstruct(xq, K)
    xt = torch.from_numpy(xq).cuda()
    D, I, R = idx.search_and_reconstruct(xt, K)
    assert R.is_cuda and np.array_equal(D.cpu().numpy(), D0) and np.array_equal(R.cpu().numpy(), R0)
    D, I, C = idx.search_and_return_codes(xt, K, include_listnos=True)
    assert C.is_cuda and C.dtype == torch.uint8
    # host-resident queries with setMinPagingSize(0): the slot-keeping search pages them itself, same results
    idx.setMinPagingSize(0)
    D, I, R = idx.search_and_reconstruct(xq, K)
    assert np.array_equal(D, D0) and np.array_equal(I, I0) and np.array_equal(R, R0)


@pytest.mark.parametrize("use_float16", [False, True])
@pytest.mark.parametrize("use_tc", [True, False])
def test_flat_search_and_reconstruct(res, use_float16, use_tc):
    d, n = 64, 5000
    rs = np.random.RandomState(5)
    xb = rs.rand(n, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d, use_tensor_cores=use_tc, use_float16=use_float16)
    idx.add(xb)
    xq = rs.rand(64, d).astype(np.float32)
    D0, I0 = idx.search(xq, K)
    D, I, R = idx.search_and_reconstruct(xq, K)
    assert np.array_equal(D, D0) and np.array_equal(I, I0)
    assert np.array_equal(R, idx.reconstruct_batch(I.reshape(-1)).reshape(R.shape))
    # k > ntotal: -1 rows are all 0xFF
    small = fb.GpuIndexFlatL2(res, d, use_tensor_cores=use_tc, use_float16=use_float16)
    small.add(xb[:5])
    D, I, R = small.search_and_reconstruct(xq[:3], 8)
    assert np.all(I[:, 5:] == -1) and np.all(_bits(R[:, 5:]) == 0xFFFFFFFF)


def test_reference_reconstruct_n(res):
    # the reference's own IndexIVF::reconstruct_n on the CPU index rebuilt from the GPU index's lists
    from oracle import ref, ref_sq

    if not (ref.available() and ref_sq.available()):
        pytest.skip("oracle/_ref not built (needs /root/reference at build time)")
    for name, kind, params in LAYOUTS:
        idx, xb, ids, d = _build(res, kind, params, n=1500)
        codes, lids = _lists(idx)
        if kind == rn.FLAT:
            cpu = ref.IndexIVFFlat(d, NLIST)
        elif kind == rn.PQ:
            cpu = ref.IndexIVFPQ(d, NLIST, params["M"], params["nbits"])
            cpu.set_pq_centroids(idx.getPQCentroids())
        else:
            cpu = ref_sq.IndexIVFScalarQuantizer(d, NLIST, params["qtype"], 1, params["by_residual"])
            cpu.set_trained(idx.getTrained())
        cpu.set_centroids(idx.getCoarseCentroids())
        for l in range(NLIST):
            if lids[l].size:
                cpu.add_entries(l, lids[l], codes[l])
        cpu.set_is_trained(True)
        # ids are [1000, 1000 + n) with duplicates: reconstruct that range on both sides
        lo, ni = 1000, int(ids.max()) + 1 - 1000
        if lo + ni > cpu.ntotal:  # the CPU precondition i0 + ni <= ntotal
            ni = cpu.ntotal - lo
        want = cpu.reconstruct_n(lo, ni, d)
        got = np.full((ni, d), np.nan, np.float32)
        fb.check(fb.lib.faiss_Index_reconstruct_n(idx._h, fb.ctypes.c_int64(lo), fb.ctypes.c_int64(ni), fb._ptr(got, fb._c_f)))
        stored = np.isin(np.arange(lo, lo + ni), ids)
        assert np.array_equal(_bits(got[stored]), _bits(want[stored])), name


def _ref_clone(ref, ref_sq, idx, kind, params, d, nlist):
    """the reference CPU index holding the GPU index's centroids, codebooks / ranges and list bytes"""
    codes, lids = _lists(idx)
    if kind == rn.FLAT:
        cpu = ref.IndexIVFFlat(d, nlist)
    elif kind == rn.PQ:
        cpu = ref.IndexIVFPQ(d, nlist, params["M"], params["nbits"])
        cpu.set_pq_centroids(idx.getPQCentroids())
    else:
        cpu = ref_sq.IndexIVFScalarQuantizer(d, nlist, params["qtype"], 1, params["by_residual"])
        cpu.set_trained(idx.getTrained())
    cpu.set_centroids(idx.getCoarseCentroids())
    for l in range(nlist):
        if lids[l].size:
            cpu.add_entries(l, lids[l], codes[l])
    cpu.set_is_trained(True)
    return cpu


@pytest.fixture(scope="module")
def refs():
    from oracle import ref, ref_recons, ref_sq

    if not (ref.available() and ref_sq.available() and ref_recons.available()):
        pytest.skip("oracle/_ref retrieval shim not built (needs /root/reference at build time)")
    return ref, ref_sq, ref_recons


@pytest.mark.parametrize("name,kind,params", LAYOUTS, ids=[l[0] for l in LAYOUTS])
def test_retrieval_matches_reference(res, refs, name, kind, params):
    # unique ids: the reference's make_direct_map + reconstruct is defined for them
    ref, ref_sq, ref_recons = refs
    d = params.get("d", 64)
    rs = np.random.RandomState(11)
    if kind == rn.FLAT:
        idx = fb.GpuIndexIVFFlat(res, d, NLIST)
    elif kind == rn.PQ:
        idx = fb.GpuIndexIVFPQ(res, d, NLIST, params["M"], params["nbits"], interleaved_layout=params["nbits"] != 8)
        idx.setPQClustering(niter=4)
    else:
        idx = fb.GpuIndexIVFScalarQuantizer(res, d, NLIST, params["qtype"], fb.METRIC_L2, params["by_residual"])
    idx.setClustering(niter=4)
    xb = _data(rs, 2000, d, params)
    idx.train(xb)
    ids = (rs.permutation(2000) * 7 + 3).astype(np.int64)
    idx.add_with_ids(xb, ids)
    cpu = _ref_clone(ref, ref_sq, idx, kind, params, d, NLIST)

    keys = rs.choice(ids, 300)
    assert np.array_equal(_bits(idx.reconstruct_batch(keys)), _bits(ref_recons.reconstruct(cpu, keys, d))), name

    xq = xb[rs.choice(2000, 30)] + np.float32(0.01)
    idx.nprobe = 4
    D, I, R = idx.search_and_reconstruct(xq, K)
    valid = I >= 0
    assert np.array_equal(_bits(R[valid]), _bits(ref_recons.reconstruct(cpu, I[valid], d))), name
    Dc, Ic, Rc = ref_recons.search_and_reconstruct(cpu, xq, K, 4)
    assert _agree_by_id(I, _bits(R), Ic, _bits(Rc)) > 0.9 * I.size, name
    _, I2, C = idx.search_and_return_codes(xq, K, include_listnos=True)
    _, Ic2, Cc = ref_recons.search_and_return_codes(cpu, xq, K, 4, include_listno=True)
    assert _agree_by_id(I2, C, Ic2, Cc) > 0.9 * I2.size, name


def _agree_by_id(I, rows, Ic, rows_c):
    """ids are unique: every id both sides returned must carry the same row (the two searches may order equal
    distances differently, so rows are matched by id, not by rank); returns how many results were compared"""
    want = {int(i): r for i, r in zip(Ic.reshape(-1), rows_c.reshape(Ic.size, -1)) if i >= 0}
    n = 0
    for i, r in zip(I.reshape(-1), rows.reshape(I.size, -1)):
        if int(i) in want:
            assert np.array_equal(r, want[int(i)]), int(i)
            n += 1
    return n


def test_return_codes_two_byte_listno_matches_reference(res, refs):
    # nlist = 300: 2-byte list numbers; integer data, so D is exact and I agrees with the CPU up to equal distances
    torch = pytest.importorskip("torch")
    ref, ref_sq, ref_recons = refs
    d, nlist, k = 8, 300, 8
    rs = np.random.RandomState(12)
    xb = np.floor(rs.rand(6000, d) * 16).astype(np.float32)
    idx = fb.GpuIndexIVFFlat(res, d, nlist)
    idx.setClustering(niter=3)
    idx.train(xb)
    idx.add_with_ids(xb, (rs.permutation(6000) * 5 + 1).astype(np.int64))
    cpu = _ref_clone(ref, ref_sq, idx, rn.FLAT, {}, d, nlist)
    assert idx.code_sizes() == (2, 4 * d) and ref_recons.coarse_code_size(cpu) == 2
    xq = np.floor(rs.rand(50, d) * 16).astype(np.float32) + np.float32(0.5)
    idx.nprobe = 20
    Dc, Ic, Cc = ref_recons.search_and_return_codes(cpu, xq, k, 20, include_listno=True)
    for x in (xq, torch.from_numpy(xq).cuda()):  # host and device outputs
        D, I, C = idx.search_and_return_codes(x, k, include_listnos=True)
        if not isinstance(D, np.ndarray):
            D, I, C = D.cpu().numpy(), I.cpu().numpy(), C.cpu().numpy()
        assert np.array_equal(D, Dc)
        # equal distances are frequent on integer data and may come in another order: compare by id
        assert _agree_by_id(I, C, Ic, Cc) > 0.5 * I.size
        assert int(C[I >= 0][:, 1].max()) == 1  # lists >= 256 were returned: the second list-number byte is used
