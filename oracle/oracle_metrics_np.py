"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the reference CPU's extra metrics (knn_extra_metrics,
faiss/utils/extra_distances.cpp:93-137, with VectorDistance<mt>, faiss/utils/simd_impl/distances_autovec-inl.h:181-304).

Distances accumulate in fp32, in dimension order, with the CPU's per-component expression.  Selection follows
the CPU heap: the k best by (distance, id), larger first for Jaccard; a NaN distance, or one not strictly better
than the sentinel (FLT_MAX, -FLT_MAX for Jaccard), never appears; empty slots are (-1, sentinel).
"""
import numpy as np

METRIC_INNER_PRODUCT = 0
METRIC_L2 = 1
METRIC_L1 = 2
METRIC_Linf = 3
METRIC_Lp = 4
METRIC_Canberra = 20
METRIC_BrayCurtis = 21
METRIC_JensenShannon = 22
METRIC_Jaccard = 23
METRIC_GOWER = 25

FLT_MAX = np.float32(np.finfo(np.float32).max)
EXTRA = [METRIC_L1, METRIC_Linf, METRIC_Lp, METRIC_Canberra, METRIC_BrayCurtis, METRIC_JensenShannon, METRIC_Jaccard,
         METRIC_GOWER]
NAMES = {METRIC_L1: "L1", METRIC_Linf: "Linf", METRIC_Lp: "Lp", METRIC_Canberra: "Canberra",
         METRIC_BrayCurtis: "BrayCurtis", METRIC_JensenShannon: "JensenShannon", METRIC_Jaccard: "Jaccard",
         METRIC_GOWER: "Gower"}


def is_similarity(metric):
    return metric in (METRIC_INNER_PRODUCT, METRIC_Jaccard)


def pairwise_extra(xq, xb, metric, metric_arg=0.0):
    """[nq, nb] fp32 distances, accumulated component by component in dimension order"""
    xq = np.asarray(xq, dtype=np.float32)
    xb = np.asarray(xb, dtype=np.float32)
    nq, d = xq.shape
    f32 = np.float32
    shape = (nq, xb.shape[0])
    acc = np.zeros(shape, dtype=f32)
    acc2 = np.zeros(shape, dtype=f32)
    with np.errstate(all="ignore"):
        for i in range(d):
            a = xq[:, i][:, None]
            b = xb[:, i][None, :]
            if metric == METRIC_L1:
                acc = acc + np.abs(a - b)
            elif metric == METRIC_Linf:
                acc = np.fmax(acc, np.abs(a - b))
            elif metric == METRIC_Lp:
                acc = acc + np.power(np.abs(a - b), f32(metric_arg))
            elif metric == METRIC_Canberra:
                acc = acc + np.abs(a - b) / (np.abs(a) + np.abs(b))
            elif metric == METRIC_BrayCurtis:
                acc = acc + np.abs(a - b)
                acc2 = acc2 + np.abs(a + b)
            elif metric == METRIC_JensenShannon:
                m = f32(0.5) * (a + b)
                acc = acc + ((-a) * np.log(m / a) + (-b) * np.log(m / b))
            elif metric == METRIC_Jaccard:
                acc = acc + np.fmin(a, b)
                acc2 = acc2 + np.fmax(a, b)
            elif metric == METRIC_GOWER:
                skip = np.isnan(a) | np.isnan(b)
                num = (a >= 0) & (b >= 0)
                cat = (a < 0) & (b < 0)
                step = np.where(num, np.where((a > 1) | (b > 1), f32(np.nan), np.abs(a - b)),
                                np.where(cat, (a != b).astype(f32), f32(np.nan)))
                step = np.broadcast_to(step, shape)
                acc = np.where(skip, acc, acc + step)
                acc2 = np.where(skip, acc2, acc2 + f32(1))
            else:
                raise ValueError("metric %d is not an extra metric" % metric)
        if metric in (METRIC_BrayCurtis, METRIC_Jaccard, METRIC_GOWER):
            acc = acc / acc2
        elif metric == METRIC_JensenShannon:
            acc = f32(0.5) * acc
    return acc.astype(f32)


def select(dis, k, metric):
    """the CPU heap's result over a [nq, nb] distance matrix"""
    nq, nb = dis.shape
    sim = is_similarity(metric)
    key = -dis if sim else dis
    sentinel = -FLT_MAX if sim else FLT_MAX
    D = np.full((nq, k), sentinel, dtype=np.float32)
    I = np.full((nq, k), -1, dtype=np.int64)
    ids = np.arange(nb, dtype=np.int64)
    for q in range(nq):
        ok = ~np.isnan(key[q]) & (key[q] < FLT_MAX)
        kk, ii = key[q][ok], ids[ok]
        order = np.lexsort((ii, kk))[:k]
        D[q, : order.size] = dis[q][ok][order]
        I[q, : order.size] = ii[order]
    return D, I


def knn_extra(xq, xb, k, metric, metric_arg=0.0, block=64):
    """knn_extra_metrics(xq, xb, k, metric, metric_arg): (D [nq, k], I [nq, k])"""
    xq = np.asarray(xq, dtype=np.float32)
    Ds, Is = [], []
    for q0 in range(0, xq.shape[0], block):
        D, I = select(pairwise_extra(xq[q0 : q0 + block], xb, metric, metric_arg), k, metric)
        Ds.append(D)
        Is.append(I)
    if not Ds:
        return np.zeros((0, k), np.float32), np.zeros((0, k), np.int64)
    return np.concatenate(Ds), np.concatenate(Is)


def assert_same_knn(refD, refI, D, I):
    """bit-exact distances, ids equal up to the order inside a group of equal distances, and up to which rows of
    the last group (the one cut at rank k) are kept.  The reference CPU's similarity heap (Jaccard) orders a tie
    group by decreasing id and keeps a scan-order-dependent part of the last group; every other result here,
    and the reference's distance heaps, use (distance, id)."""
    assert refD.shape == D.shape and refI.shape == I.shape
    assert np.array_equal((refI < 0), (I < 0)), "-1 placement differs"
    assert np.array_equal(refD.view(np.uint32), D.view(np.uint32)), "distances differ"
    for q in range(refI.shape[0]):
        valid = refI[q] >= 0
        if not valid.any():
            continue
        last = refD[q][valid][-1]
        for v in np.unique(refD[q][valid]):
            a = np.sort(refI[q][valid & (refD[q] == v)])
            b = np.sort(I[q][valid & (D[q] == v)])
            assert a.size == b.size, "query %d: tie group %r differs in size" % (q, v)
            if v != last:
                assert np.array_equal(a, b), "query %d: ids at distance %r differ" % (q, v)
        assert np.unique(I[q][valid]).size == int(valid.sum()), "duplicate ids in query %d" % q


# ---------------------------------------------------------------- test data
def positive(rs, n, d):
    """strictly positive floats (Canberra, JensenShannon and Jaccard without NaN components)"""
    return (rs.rand(n, d) + 0.05).astype(np.float32)


def integers(rs, n, d):
    """floor(16 u) + 1: every partial sum of L1, Linf, BrayCurtis and Jaccard is exact in fp32"""
    return (np.floor(16 * rs.rand(n, d)) + 1).astype(np.float32)


def gower_rows(rs, n, d):
    """mixed columns: even columns numeric in [0, 1], odd columns categorical in {-1, -2, -3}"""
    x = rs.rand(n, d).astype(np.float32)
    x[:, 1::2] = -np.floor(rs.rand(n, d // 2) * 3 + 1).astype(np.float32)
    return x


def metric_data(metric, rs, n, d, integer=False):
    if metric == METRIC_GOWER:
        return gower_rows(rs, n, d)
    if integer:
        return integers(rs, n, d)
    if metric in (METRIC_Canberra, METRIC_JensenShannon, METRIC_Jaccard):
        return positive(rs, n, d)
    return (rs.rand(n, d) * 2 - 1).astype(np.float32)
