"""High-dimensional search paths against float64 truth, under the certified top-k check
(oracle/oracle_bound_np.py), plus the k-means update and top-k merge seams, bit for bit.

Data kinds: 'int' (small integers, every fp32 sum exact: bound 0, results bit-exact), 'clustered' (queries
next to database rows: a well separated top-k, so the completeness check has teeth), 'uniform' / 'gauss'
(concentrated distances; Gaussian IP cancels).  Every case keeps nq * |S| * d <= 2e9.
"""
import numpy as np
import pytest

from oracle import oracle_bound_np as ob
from oracle import oracle_ivf_check_np as oc
from oracle import oracle_sq_np as osq

pytestmark = pytest.mark.gpu

L2, IP = ob.METRIC_L2, ob.METRIC_INNER_PRODUCT
f32 = np.float32


def _data(kind, n, nq, d, seed):
    rs = np.random.RandomState(seed)
    if kind == "int":
        xb = rs.randint(-15, 16, (n, d)).astype(f32)
        xq = rs.randint(-15, 16, (nq, d)).astype(f32)
        xq[: nq // 2] = xb[rs.randint(0, n, nq // 2)]  # exact matches and, through them, ties
        return xb, xq
    if kind == "uniform":
        return rs.rand(n, d).astype(f32), rs.rand(nq, d).astype(f32)
    if kind == "gauss":
        return rs.randn(n, d).astype(f32), rs.randn(nq, d).astype(f32)
    cent = rs.randn(64, d) * 2.0
    xb = (cent[rs.randint(0, 64, n)] + 0.5 * rs.randn(n, d)).astype(f32)
    xq = (xb[rs.randint(0, n, nq)] + 0.01 * rs.randn(nq, d)).astype(f32)
    return xb, xq


def _truth(xq, xb, metric):
    return ob.l2_truth_many(xq, xb) if metric == L2 else ob.ip_truth_many(xq, xb)


# ------------------------------------------------------------------ Flat / bfKnn
# (d, k, N, nq, metric, fp16 storage, data, api): a pairwise-covering subset of d x k x nq x metric x storage x
# data x {index, bfKnn host, bfKnn device}; k covers the exact kernel's K1, TQ 32 / 16 / 8 and LIST 128 ... 2048
FLAT_CASES = [
    (256, 64, 40000, 33, L2, False, "clustered", "index"),  # tensor cores (d <= 256, N >= 32768, nq >= 16)
    (256, 100, 20011, 5, IP, False, "gauss", "index"),
    (257, 1, 20011, 200, L2, False, "uniform", "host"),
    (257, 2048, 20011, 200, L2, False, "int", "index"),
    (300, 257, 20011, 33, IP, True, "clustered", "index"),
    (384, 1025, 20011, 5, L2, False, "int", "device"),
    (512, 2048, 20011, 1, L2, True, "gauss", "index"),
    (513, 100, 19001, 200, IP, False, "int", "device"),
    (768, 64, 20011, 33, L2, False, "gauss", "device"),
    (1000, 2048, 8000, 5, IP, False, "uniform", "index"),
    (1024, 1, 20011, 5, IP, True, "int", "index"),
    (1024, 257, 20011, 33, L2, False, "clustered", "host"),
    (1536, 1025, 20011, 5, L2, True, "uniform", "index"),
    (1536, 1, 6007, 200, L2, False, "gauss", "index"),
    (2048, 64, 20011, 1, IP, False, "clustered", "index"),
    (2048, 100, 20011, 33, L2, False, "int", "host"),
    (2048, 2048, 20011, 5, IP, False, "gauss", "device"),
]


@pytest.mark.parametrize("d,k,N,nq,metric,fp16,kind,api", FLAT_CASES)
def test_flat_highdim_certified(res, d, k, N, nq, metric, fp16, kind, api):
    import torch

    import faiss_b200 as fb

    assert nq * N * d <= 2e9
    xb, xq = _data(kind, N, nq, d, seed=d + k + nq)
    if api == "index":
        idx = fb.GpuIndexFlat(res, d, metric, use_float16=fp16)
        idx.add(xb)
        D, I = idx.search(xq, k)
        assert idx.lastSearchInfo()["tensor_cores"] == int(d <= 256 and N >= 32768 and nq >= 16)
        xs = idx.reconstruct_n(0, N)  # the stored data
        if fp16:
            assert np.array_equal(xs, xb.astype(np.float16).astype(f32))
            xq = xq.astype(np.float16).astype(f32)  # fp16 storage rounds the queries too
    else:
        assert not fp16
        if api == "host":
            D, I = fb.bfKnn(res, xq, xb, k, metric)
        else:
            D, I = fb.bfKnn(res, torch.from_numpy(xq).cuda(), torch.from_numpy(xb).cuda(), k, metric)
            torch.cuda.synchronize()
            D, I = D.cpu().numpy(), I.cpu().numpy()
        xs = xb
    T, B = _truth(xq, xs, metric)
    ids = np.arange(N, dtype=np.int64)
    if kind == "int":
        B = np.zeros_like(T)  # every sum exact: bit-exact distances, ties by ascending id
        for qi in range(nq):
            eD, eI = ob.exact_topk(T[qi], ids, k, metric)
            assert np.array_equal(D[qi], eD) and np.array_equal(I[qi], eI), "query %d" % qi
    ob.check_knn(D, I, ids, T, B, k, metric, what="flat d=%d k=%d" % (d, k))


# ------------------------------------------------------------------ IVF-Flat
# d 384 / 512: the fast path with nch = 3 / 4 float4 chunks per lane; 640: a multiple of 128 past the fast path;
# 300 / 1000: the generic path.  (512, 2048, nprobe 1) probes the smallest list, fewer than k vectors: -1 padding.
IVFFLAT_CASES = [
    (384, 100, L2, 8),
    (384, 1, IP, 8),
    (512, 1024, IP, 8),
    (512, 2048, L2, 1),
    (640, 1, L2, 8),
    (640, 100, IP, 8),
    (300, 2048, IP, 4),
    (1000, 100, L2, 8),
    (1000, 1024, IP, 8),
]


@pytest.mark.parametrize("d,k,metric,nprobe", IVFFLAT_CASES)
def test_ivfflat_highdim_certified(res, d, k, metric, nprobe):
    import faiss_b200 as fb

    N, nq, nlist = 20000, 20, 64
    xb, xq = _data("clustered" if k != 1 else "gauss", N, nq, d, seed=d * 3 + k)
    idx = fb.GpuIndexIVFFlat(res, d, nlist, metric)
    idx.setClustering(niter=4, seed=7)
    idx.train(xb)
    idx.add(xb)
    probes, cdis = oc.probes(xq, idx.getCoarseCentroids(), nprobe, metric)
    if nprobe == 1:  # probe the smallest list: fewer than k candidates
        sizes = np.array([idx.getListLength(l) for l in range(nlist)])
        probes[:] = int(np.argmin(np.where(sizes > 0, sizes, N)))
    D, I = oc.search_preassigned(idx, xq, k, probes, cdis)
    for qi in range(nq):
        ls = oc.probed_lists(idx, probes[qi])
        ids = np.concatenate([i for _, i, _ in ls])
        Y = np.concatenate([v.view(f32).reshape(-1, d) for _, _, v in ls])
        for l, li, v in ls:
            assert np.array_equal(v.view(f32).reshape(-1, d), xb[li]), "stored vectors of list %d" % l
        t, beta = ob.l2_truth(xq[qi], Y) if metric == L2 else ob.ip_truth(xq[qi], Y)
        if nprobe == 1:
            assert ids.size < k  # the padding case
        ob.check_topk(D[qi], I[qi], ids, t, beta, k, metric, what="ivfflat d=%d query %d" % (d, qi))


# ------------------------------------------------------------------ IVF-PQ
def _pq_search_and_check(idx, xb, xq, k, metric, M, nbits, nprobe, precomp, exact=False):
    d = xb.shape[1]
    dsub = d // M
    cent = idx.getCoarseCentroids()
    pq = idx.getPQCentroids()
    probes, cdis = oc.probes(xq, cent, nprobe, metric)
    D, I = oc.search_preassigned(idx, xq, k, probes, cdis)
    checked = set()
    for qi in range(xq.shape[0]):
        ids_all, t_all, b_all = [], [], []
        for l, li, raw in oc.probed_lists(idx, probes[qi]):
            codes = oc.unpack(raw.reshape(li.size, -1), M, nbits)
            if l not in checked:
                oc.pq_check_codes(xb[li], cent[l], pq, codes, M, exact)
                checked.add(l)
            Yd = pq[np.arange(M)[None, :], codes].reshape(li.size, d)
            if metric == L2 and precomp:
                t, b = ob.pq_l2_precomp_truth(xq[qi], cent[l], Yd, dsub, M)
            elif metric == L2:
                t, b = ob.pq_l2_truth(xq[qi].astype(np.float64) - cent[l], Yd, dsub, M)
            else:
                t, b = ob.pq_ip_truth(xq[qi], cent[l], Yd, dsub, M)
            ids_all.append(li)
            t_all.append(t)
            b_all.append(b)
        t, b = np.concatenate(t_all), np.concatenate(b_all)
        if exact:
            b = np.zeros_like(b)
        ob.check_topk(D[qi], I[qi], np.concatenate(ids_all), t, b, k, metric,
                      what="ivfpq d=%d M=%d nbits=%d query %d" % (d, M, nbits, qi))


# (d, M, nbits, metric, precomputed tables): M 16 / 32 take the interleaved layout (nbits 4: the nibble-pair
# scan), the rest the vector-major scan (vec16 for M % 16 == 0, packed for nbits < 8); dsub covers the encode
# kernel's templated 8, 12, 16, 32 and its runtime branch (15, 24, 256).  (1024, 4): a 256 KiB codebook per
# sub-quantiser, more than a block's shared memory.
IVFPQ_CASES = [
    (768, 32, 8, L2, True),
    (768, 32, 8, IP, False),
    (512, 16, 8, L2, False),
    (1024, 32, 8, L2, True),
    (1024, 64, 8, L2, False),
    (384, 48, 8, IP, False),
    (300, 20, 8, L2, False),
    (1024, 4, 8, L2, False),
    (512, 32, 4, L2, False),
    (768, 64, 6, IP, False),
]


@pytest.mark.parametrize("d,M,nbits,metric,precomp", IVFPQ_CASES)
def test_ivfpq_highdim_certified(res, d, M, nbits, metric, precomp):
    import faiss_b200 as fb

    N, nq, nlist, nprobe, k = 10000, 10, 32, 4, 100
    xb, xq = _data("clustered", N, nq, d, seed=d + M + nbits)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, nbits, metric, interleaved_layout=nbits != 8)
    idx.setClustering(niter=4, seed=3)
    idx.setPQClustering(niter=4, seed=5)
    idx.setPrecomputedCodes(precomp)
    idx.train(xb)
    idx.add(xb)
    assert idx.ntotal == N
    _pq_search_and_check(idx, xb, xq, k, metric, M, nbits, nprobe, precomp)


@pytest.mark.parametrize("M,precomp,metric", [(32, False, L2), (32, True, L2), (32, False, IP), (8, False, L2)])
def test_ivfpq_integer_codebooks_bit_exact(res, M, precomp, metric):
    """integer coarse and PQ centroids and integer data: residuals, encode and every LUT / code sum are exact, so
    the codes are the first minimum and the distances bit-exact"""
    import faiss_b200 as fb

    d, nlist, N, nq, k = 512, 16, 4000, 8, 50
    dsub = d // M
    rs = np.random.RandomState(M + precomp)
    cent = rs.randint(-4, 5, (nlist, d)).astype(f32)
    pq = rs.randint(-3, 4, (M, 256, dsub)).astype(f32)
    xb = (cent[rs.randint(0, nlist, N)] + rs.randint(-3, 4, (N, d))).astype(f32)
    xq = (xb[rs.randint(0, N, nq)] + rs.randint(-1, 2, (nq, d))).astype(f32)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, metric)
    idx.setCoarseCentroids(cent)
    idx.setPQCentroids(pq)
    idx.setIsTrained(True)
    idx.setPrecomputedCodes(precomp)
    idx.add(xb)
    _pq_search_and_check(idx, xb, xq, k, metric, M, 8, 4, precomp, exact=True)


# ------------------------------------------------------------------ IVF-SQ
# (qtype, d, encodeResidual): 8bit d 384 and 6bit d 1000 take the generic scan, fp16 d 512 the fast path's 4 chunks,
# fp16 d 640 and 4bit d 768 the generic path past it; 8bit_direct on integers 0..15 without a residual is exact
IVFSQ_CASES = [
    (osq.QT_8bit, 384, True),
    (osq.QT_4bit, 512, True),
    (osq.QT_4bit, 768, True),
    (osq.QT_fp16, 512, True),
    (osq.QT_fp16, 640, True),
    (osq.QT_6bit, 1000, True),
    (osq.QT_8bit_direct, 2048, False),
]


@pytest.mark.parametrize("qtype,d,residual", IVFSQ_CASES)
def test_ivfsq_highdim_certified(res, qtype, d, residual):
    import faiss_b200 as fb

    N, nq, nlist, nprobe, k = 12000, 10, 32, 4, 100
    exact = qtype == osq.QT_8bit_direct
    if exact:
        rs = np.random.RandomState(d)
        xb = rs.randint(0, 16, (N, d)).astype(f32)
        xq = xb[rs.randint(0, N, nq)].copy()
        xq[1::2] = rs.randint(0, 16, (nq // 2, d))
    else:
        xb, xq = _data("clustered", N, nq, d, seed=d + qtype)
    idx = fb.GpuIndexIVFScalarQuantizer(res, d, nlist, qtype, L2, encodeResidual=residual)
    idx.setClustering(niter=4, seed=11)
    idx.train(xb)
    idx.add(xb)
    trained = idx.getTrained()
    cent = idx.getCoarseCentroids()
    probes, cdis = oc.probes(xq, cent, nprobe, L2)
    D, I = oc.search_preassigned(idx, xq, k, probes, cdis)
    for qi in range(nq):
        ids_all, t_all, b_all = [], [], []
        for l, li, raw in oc.probed_lists(idx, probes[qi]):
            X, vmin, vdiff = oc.sq_exact_decode(raw, qtype, trained, d)
            r = xq[qi].astype(np.float64) - (cent[l].astype(np.float64) if residual else 0.0)
            t, b = ob.sq_l2_truth(r, X, vmin, vdiff)
            ids_all.append(li)
            t_all.append(t)
            b_all.append(np.zeros_like(b) if exact else b)
            if exact:
                assert np.array_equal(X, xb[li]), "8bit_direct stores the value itself"
        ob.check_topk(D[qi], I[qi], np.concatenate(ids_all), np.concatenate(t_all), np.concatenate(b_all), k, L2,
                      what="ivfsq qtype=%d d=%d query %d" % (qtype, d, qi))


# ------------------------------------------------------------------ k-means update seam
@pytest.mark.parametrize("d", [1, 31, 127, 129, 300, 768])
def test_kmeans_accumulate_bit_exact(res, d):
    """the sorted update adds each centroid's points in index order in fp32: sums and counts must equal a
    sequential float32 sum in index order (np.cumsum, not the pairwise np.sum)"""
    import torch

    import faiss_b200 as fb

    n, k = 50000, 100
    rs = np.random.RandomState(d)
    x = (rs.randn(n, d) * 10 + 3).astype(f32)
    a = rs.randint(0, k, n).astype(np.int64)
    a[a == 17] = 18  # empty clusters
    a[a == 55] = 3
    a[rs.rand(n) < 0.5] = 42  # one cluster holds half the points
    a[rs.rand(n) < 0.02] = -1  # unassigned
    a[rs.rand(n) < 0.02] = k + rs.randint(0, 5)  # out of range
    sums, counts = fb.kmeans_accumulate(res, torch.from_numpy(x).cuda(), torch.from_numpy(a).cuda(), k)
    torch.cuda.synchronize()
    sums, counts = sums.cpu().numpy(), counts.cpu().numpy()
    for c in range(k):
        rows = np.nonzero(a == c)[0]  # index order
        assert counts[c] == rows.size, "count of centroid %d" % c
        want = np.cumsum(x[rows], axis=0, dtype=f32)[-1] if rows.size else np.zeros(d, f32)
        assert np.array_equal(sums[c], want), "centroid %d: max |diff| %g" % (c, float(np.abs(sums[c] - want).max()))


# ------------------------------------------------------------------ top-k merge seam
@pytest.mark.parametrize("nlists", [1, 7, 64])
@pytest.mark.parametrize("kin", [1, 33, 2048])
@pytest.mark.parametrize("k", [1, 64, 65, 1024, 2048])
@pytest.mark.parametrize("metric", [L2, IP])
def test_topk_merge_bit_exact(res, nlists, kin, k, metric):
    """merged [nq, k] == a lexsort of every valid input on (key, id): -1 holes skipped, keys duplicated across
    lists, negative stored ids, per-list id offsets"""
    import torch

    import faiss_b200 as fb

    nq = 3
    rs = np.random.RandomState(nlists * 10000 + kin * 10 + k + metric)
    Din = rs.randint(-50, 50, (nq, nlists, kin)).astype(f32) * f32(0.25)  # many equal keys within and across lists
    Iin = rs.randint(-1000, 10 ** 6, (nq, nlists, kin)).astype(np.int64)
    Iin[Iin == -1] = -2  # -1 only where planted
    Iin[rs.rand(nq, nlists, kin) < 0.15] = -1
    offs = (np.arange(nlists, dtype=np.int64) * 10 ** 7) if nlists > 1 else None
    # ids unique within a row after the offsets (what a merge of distinct shards sees)
    for q in range(nq):
        flat = Iin[q].reshape(-1)
        ok = flat != -1
        flat[ok] = np.arange(ok.sum()) * 7 - 500
        Iin[q] = flat.reshape(nlists, kin)
    Dt, It = torch.from_numpy(Din).cuda(), torch.from_numpy(Iin).cuda()
    Ot = torch.from_numpy(offs).cuda() if offs is not None else None
    D, I = fb.topk_merge(res, Dt, It, k, metric, id_offsets=Ot)
    torch.cuda.synchronize()
    D, I = D.cpu().numpy(), I.cpu().numpy()
    for q in range(nq):
        ids = Iin[q] + (offs[:, None] if offs is not None else 0)
        valid = Iin[q] != -1
        key = Din[q][valid].astype(np.float64)
        ids = ids[valid]
        o = np.lexsort((ids, key if metric == L2 else -key))[:k]
        wD = np.full(k, ob.FLT_MAX if metric == L2 else -ob.FLT_MAX, f32)
        wI = np.full(k, -1, np.int64)
        wD[: o.size], wI[: o.size] = key[o].astype(f32), ids[o]
        assert np.array_equal(D[q], wD), "query %d distances" % q
        assert np.array_equal(I[q], wI), "query %d ids" % q
