"""CPU self-test of the certified top-k checker (oracle/oracle_bound_np.py).

Accept: numpy float32 emulations of the kernels' arithmetic -- sequential FMA chains, pairwise trees, the
32-lane strided sums with a butterfly, the IVF-PQ LUT / code sums, the precomputed-table decomposition and
the folded IVF-SQ decode -- never exceed the derived bounds, at d up to 2048.
Reject: every planted fault (a lost 16-dimension chunk, one dropped dimension, a swapped neighbour, a
duplicate id, tied ids out of order, a -1 before a valid entry) is caught.
"""
import numpy as np
import pytest

from oracle import oracle_bound_np as ob
from oracle.oracle_bound_np import METRIC_INNER_PRODUCT as IP, METRIC_L2 as L2

f32 = np.float32


def _fma(a, b, c):
    """fl(a * b + c) for float32 arrays: the product of two fp32 values is exact in float64"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def _terms(Q, Y, metric):
    """per-component fp32 operands (x, y) such that the kernel's term is x * y: [n, d] each"""
    if metric == L2:
        t = (Q[None, :] - Y).astype(f32)  # one rounding
        return t, t
    return np.broadcast_to(Q[None, :], Y.shape), Y


def emulate(q, Y, metric, order):
    """fp32 distance of query q [d] to each row of Y [n, d] in one summation order:
    'seq' an FMA chain in dimension order (flat_exact.cu), 'pair' a pairwise tree of rounded products,
    'warp' 32 lanes striding the dimension with FMA chains, then a 5-level xor butterfly (ivf.cu generic scan)."""
    a, b = _terms(q, Y, metric)
    n, d = Y.shape
    if order == "seq":
        acc = np.zeros(n, f32)
        for j in range(d):
            acc = _fma(a[:, j], b[:, j], acc)
        return acc
    if order == "pair":
        v = (a * b).astype(f32)
        while v.shape[1] > 1:
            if v.shape[1] % 2:
                v = np.concatenate([v, np.zeros((n, 1), f32)], 1)
            v = (v[:, 0::2] + v[:, 1::2]).astype(f32)
        return v[:, 0]
    assert order == "warp"
    lanes = np.zeros((n, 32), f32)
    for j in range(d):
        lanes[:, j % 32] = _fma(a[:, j], b[:, j], lanes[:, j % 32])
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(f32)
    return lanes[:, 0]


def _data(kind, n, d, seed):
    rs = np.random.RandomState(seed)
    if kind == "uniform":
        return rs.rand(n, d).astype(f32), rs.rand(d).astype(f32)
    if kind == "gauss":
        return rs.randn(n, d).astype(f32), rs.randn(d).astype(f32)
    # clustered: the query sits next to row 3
    Y = (rs.randn(n // 10 + 1, d)[rs.randint(0, n // 10 + 1, n)] + 0.3 * rs.randn(n, d)).astype(f32)
    return Y, (Y[3] + 0.01 * rs.randn(d)).astype(f32)


def _truth(q, Y, metric):
    return ob.l2_truth(q, Y) if metric == L2 else ob.ip_truth(q, Y)


def _select(dis, ids, k, metric):
    """top-k of fp32 distances by the (key, id) order"""
    key = dis if metric == L2 else -dis
    o = np.lexsort((ids, key.astype(np.float64)))[:k]
    D = np.full(k, ob.FLT_MAX if metric == L2 else -ob.FLT_MAX, f32)
    I = np.full(k, -1, np.int64)
    D[: o.size], I[: o.size] = dis[o], ids[o]
    return D, I


# ------------------------------------------------------------------ accept
@pytest.mark.parametrize("d", [17, 256, 1000, 2048])
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("kind", ["uniform", "gauss", "clustered"])
def test_accepts_every_summation_order(d, metric, kind):
    Y, q = _data(kind, 400, d, seed=d * 7 + metric)
    ids = np.arange(Y.shape[0], dtype=np.int64) * 3 + 11  # ids need not be row numbers
    t, beta = _truth(q, Y, metric)
    for order in ("seq", "pair", "warp"):
        dis = emulate(q, Y, metric, order)
        err = np.abs(dis.astype(np.float64) - t)
        assert np.all(err <= beta), (order, float((err / beta).max()))
        for k in (1, 10, 400, 512):
            D, I = _select(dis, ids, k, metric)
            ob.check_topk(D, I, ids, t, beta, k, metric, what=order)


def test_many_query_truth_matches_per_query_truth():
    rs = np.random.RandomState(3)
    Q, Y = rs.randn(4, 300).astype(f32), rs.randn(50, 300).astype(f32)
    for many, one in ((ob.l2_truth_many, ob.l2_truth), (ob.ip_truth_many, ob.ip_truth)):
        T, B = many(Q, Y)
        for i in range(4):
            t, b = one(Q[i], Y)
            assert np.all(np.abs(T[i] - t) <= 1e-9 * (1 + np.abs(t)))
            assert np.all(B[i] >= b * (1 - 1e-12))


def _pq_setup(d, M, seed):
    rs = np.random.RandomState(seed)
    dsub = d // M
    q = rs.randn(d).astype(f32)
    c = (3.0 * rs.randn(d)).astype(f32)  # a far centroid: the residual's rounding matters
    pq = rs.randn(M, 256, dsub).astype(f32)
    codes = rs.randint(0, 256, (300, M))
    Yd = pq[np.arange(M)[None, :], codes].reshape(300, d)
    return q, c, pq, codes, Yd, dsub


@pytest.mark.parametrize("d,M", [(768, 32), (1024, 4), (300, 20), (2048, 64)])
def test_accepts_pq_arithmetic(d, M):
    q, c, pq, codes, Yd, dsub = _pq_setup(d, M, d + M)
    r = (q - c).astype(f32)
    # L2: LUT entries are fma chains over the rounded residual, then M entries summed in two chains
    lut = np.zeros((M, 256), f32)
    for j in range(dsub):
        df = (r.reshape(M, dsub)[:, None, j] - pq[:, :, j]).astype(f32)
        lut = _fma(df, df, lut)
    ent = lut[np.arange(M)[None, :], codes]
    a0 = np.zeros(300, f32)
    a1 = np.zeros(300, f32)
    for m in range(M):
        if m & 1:
            a1 = (a1 + ent[:, m]).astype(f32)
        else:
            a0 = (a0 + ent[:, m]).astype(f32)
    dis = (a0 + a1).astype(f32)
    t, beta = ob.pq_l2_truth(q.astype(np.float64) - c, Yd, dsub, M)
    assert np.all(np.abs(dis - t) <= beta)
    # precomputed tables: T2 = ||y||^2 + 2<c|y>, t3 = -2<q|y>, t1 = ||q - c||^2 (fma chains)
    t2 = np.zeros((M, 256), f32)
    t3 = np.zeros((M, 256), f32)
    cs, qs = c.reshape(M, dsub), q.reshape(M, dsub)
    for j in range(dsub):
        y = pq[:, :, j]
        t2 = _fma(y, y, t2)
        t2 = _fma((2 * cs[:, None, j]).astype(f32), y, t2)
        t3 = _fma(qs[:, None, j], y, t3)
    tab = (t2 + (f32(-2) * t3).astype(f32)).astype(f32)
    t1 = emulate(q, c[None, :], L2, "warp")[0]
    acc = np.full(300, t1, f32)
    ent = tab[np.arange(M)[None, :], codes]
    for m in range(M):
        acc = (acc + ent[:, m]).astype(f32)
    t, beta = ob.pq_l2_precomp_truth(q, c, Yd, dsub, M)
    assert np.all(np.abs(acc - t) <= beta)
    # IP: coarse term rounded to fp32, LUT fma chains, code sum, one add
    qc = f32(float(q.astype(np.float64) @ c))
    lut = np.zeros((M, 256), f32)
    for j in range(dsub):
        lut = _fma(np.broadcast_to(qs[:, None, j], (M, 256)), pq[:, :, j], lut)
    ent = lut[np.arange(M)[None, :], codes]
    acc = np.zeros(300, f32)
    for m in range(M):
        acc = (acc + ent[:, m]).astype(f32)
    dis = (acc + qc).astype(f32)
    t, beta = ob.pq_ip_truth(q, c, Yd, dsub, M)
    assert np.all(np.abs(dis - t) <= beta)


@pytest.mark.parametrize("d,s", [(384, 255), (512, 15), (1000, 63)])
def test_accepts_sq_folded_decode(d, s):
    """x = m + b c with b = fl(vdiff / s), m = fl(vmin + b / 2); component fma(-b, c, fl(r - m))"""
    rs = np.random.RandomState(d)
    vmin = (rs.randn(d) * 4).astype(f32)
    vdiff = (rs.rand(d) * 8 + 0.1).astype(f32)
    codes = rs.randint(0, s + 1, (300, d)).astype(f32)
    q = (vmin + vdiff * rs.rand(d) + 5 * rs.randn(d)).astype(f32)
    cen = (5 * rs.randn(d)).astype(f32)
    b = (vdiff / f32(s)).astype(f32)
    m = (vmin + (f32(0.5) * b).astype(f32)).astype(f32)
    r = (q - cen).astype(f32)
    a = (r - m).astype(f32)
    comp = _fma(np.broadcast_to(-b, codes.shape), codes, np.broadcast_to(a, codes.shape))
    acc = np.zeros(300, f32)
    for j in range(d):
        acc = _fma(comp[:, j], comp[:, j], acc)
    X = vmin.astype(np.float64) + vdiff.astype(np.float64) * (codes + 0.5) / s
    t, beta = ob.sq_l2_truth(q.astype(np.float64) - cen, X, vmin, vdiff)
    assert np.all(np.abs(acc - t) <= beta)


def test_exact_mode_on_integer_data():
    """|values| <= 15, d = 2048: every fp32 sum is exact, so beta = 0 and the result must be the (key, id) order"""
    rs = np.random.RandomState(1)
    Y = rs.randint(-15, 16, (500, 2048)).astype(f32)
    Y[100] = Y[7]  # a tie
    q = Y[7].copy()
    ids = np.arange(500, dtype=np.int64)
    for metric in (L2, IP):
        dis = emulate(q, Y, metric, "warp")
        t, _ = _truth(q, Y, metric)
        assert np.array_equal(dis.astype(np.float64), t)
        D, I = _select(dis, ids, 20, metric)
        ob.check_topk(D, I, ids, t, 0.0, 20, metric)
        eD, eI = ob.exact_topk(t, ids, 20, metric)
        assert np.array_equal(D, eD) and np.array_equal(I, eI)


# ------------------------------------------------------------------ reject
def _good(kind, n, d, k, metric, seed, dims=None):
    Y, q = _data(kind, n, d, seed)
    ids = np.arange(n, dtype=np.int64)
    t, beta = _truth(q, Y, metric)
    return Y, q, ids, t, beta


def test_rejects_lost_last_chunk():
    for d in (300, 1000, 2048):
        for metric in (L2, IP):
            Y, q, ids, t, beta = _good("uniform", 500, d, 10, metric, d)
            D, I = _select(emulate(q, Y, metric, "seq"), ids, 10, metric)
            ob.check_topk(D, I, ids, t, beta, 10, metric)
            dis = emulate(q[: d - 16], Y[:, : d - 16], metric, "seq")  # the last kDK = 16 chunk never added
            D, I = _select(dis, ids, 10, metric)
            with pytest.raises(ob.CertificateError):
                ob.check_topk(D, I, ids, t, beta, 10, metric)


def test_rejects_one_dropped_dimension_of_2048():
    # dimension 1234 carries a large component, so losing it moves every distance far past the bound
    rs = np.random.RandomState(9)
    Y = rs.rand(500, 2048).astype(f32)
    Y[:, 1234] = f32(40) + rs.rand(500).astype(f32)
    q = rs.rand(2048).astype(f32)
    ids = np.arange(500, dtype=np.int64)
    for metric in (L2, IP):
        t, beta = _truth(q, Y, metric)
        keep = np.arange(2048) != 1234
        D, I = _select(emulate(q, Y, metric, "warp"), ids, 8, metric)
        ob.check_topk(D, I, ids, t, beta, 8, metric)
        D, I = _select(emulate(q[keep], Y[:, keep], metric, "warp"), ids, 8, metric)
        with pytest.raises(ob.CertificateError):
            ob.check_topk(D, I, ids, t, beta, 8, metric)


def test_rejects_swapped_neighbour():
    """the true #1 replaced by #(k+1), every reported distance itself correct: only completeness catches it"""
    k = 10
    for metric in (L2, IP):
        Y, q, ids, t, beta = _good("clustered", 600, 1024, k, metric, 5)
        key = t if metric == L2 else -t
        o = np.argsort(key, kind="stable")
        gap = abs(t[o[k]] - t[o[0]])
        assert gap > beta[o[0]] + beta[o[k]]
        pick = np.concatenate([o[1:k], o[k : k + 1]])
        dis = emulate(q, Y, metric, "seq")
        D, I = _select(dis[pick], ids[pick], k, metric)
        ob.check_topk(D, I, ids[pick], t[pick], beta[pick], k, metric)  # fine against the wrong candidate set
        with pytest.raises(ob.CertificateError, match="certainly better"):
            ob.check_topk(D, I, ids, t, beta, k, metric)


def test_rejects_duplicate_id():
    Y, q, ids, t, beta = _good("gauss", 300, 513, 10, L2, 2)
    D, I = _select(emulate(q, Y, L2, "seq"), ids, 10, L2)
    I[5], D[5] = I[4], D[4]
    with pytest.raises(ob.CertificateError, match="duplicate"):
        ob.check_topk(D, I, ids, t, beta, 10, L2)


def test_rejects_descending_ids_on_a_tie():
    Y, q, ids, t, beta = _good("gauss", 300, 768, 10, IP, 4)
    Y[200] = Y[50]  # identical rows: identical fp32 distances
    t, beta = _truth(q, Y, IP)
    dis = emulate(q, Y, IP, "seq")
    sel = np.array([50, 200] + [i for i in range(300) if i not in (50, 200)][:8])
    D, I = _select(dis[sel], ids[sel], 10, IP)
    j = int(np.where(I == 50)[0][0])
    assert I[j + 1] == 200 and D[j] == D[j + 1]
    I[j], I[j + 1] = 200, 50
    with pytest.raises(ob.CertificateError, match="must ascend"):
        ob.check_topk(D, I, ids[sel], t[sel], beta[sel], 10, IP)


def test_rejects_padding_before_a_valid_entry():
    Y, q, ids, t, beta = _good("uniform", 300, 257, 10, L2, 6)
    D, I = _select(emulate(q, Y, L2, "seq"), ids, 10, L2)
    D2, I2 = D.copy(), I.copy()
    I2[2:], D2[2:] = I[1:-1], D[1:-1]
    I2[1], D2[1] = -1, f32(ob.FLT_MAX)
    with pytest.raises(ob.CertificateError, match="is -1"):
        ob.check_topk(D2, I2, ids, t, beta, 10, L2)
    # and with fewer candidates than k, the padding must be -1 with the sentinel
    D, I = _select(emulate(q, Y[:4], L2, "seq"), ids[:4], 10, L2)
    ob.check_topk(D, I, ids[:4], t[:4], beta[:4], 10, L2)
    D[7] = f32(0)
    with pytest.raises(ob.CertificateError, match="padding"):
        ob.check_topk(D, I, ids[:4], t[:4], beta[:4], 10, L2)


@pytest.mark.parametrize("metric", [L2, IP])
def test_empty_candidate_set(metric):
    """a probe set with no vectors (empty lists, -1 probes): only padding is valid"""
    sentinel = ob.FLT_MAX if metric == L2 else -ob.FLT_MAX
    none = np.zeros(0)
    ob.check_topk(np.full(4, sentinel, f32), np.full(4, -1), np.zeros(0, np.int64), none, none, 4, metric)
    with pytest.raises(ob.CertificateError):
        ob.check_topk(np.array([1, sentinel], f32), np.array([5, -1]), np.zeros(0, np.int64), none, none, 2, metric)
