"""Every IVF list scan at d <= 256 against float64 truth, under the certified top-k check (oracle/oracle_bound_np.py).

The indexes are built from a payload (coarse centroids, PQ codebooks or SQ ranges, then setListSizes / setList with
random codes that cover every code value), so the list lengths are exact: 0, 1, 31, 32, 33, 127, 128, 129, 255,
256, 257 and a few thousand -- the edges of a 32-vector group, of a 4-group work unit and of the warp lists.  Ids
are shuffled in some cases, so user ids are not monotone in arena position and the (key, id) order is really
tested.  Queries sit next to stored vectors ('clustered': a well-separated top-k for the completeness clause) or
are small integers over integer codebooks ('int': every fp32 sum exact, so bound 0: bit-exact distances and the
exact top-k).

Each case certifies the first rows of its assign matrix with planted probe sets: an empty list paired with a
one-vector list, a -1 entry, a set of fewer than k candidates (-1 padding) and, where the list lengths allow it,
a set of exactly k.  Query regimes (ivfScanChunks): 'small' (nq 12: one probe per CTA), 'mid' (nq 300, nprobe 7:
two probes per CTA and an odd last chunk), 'big' (nq 1152: one CTA per query over all its probes, so the
interleaved L2 tables are built in pairs); of 'big' a fixed subset of 40 queries is certified.
"""
import itertools
import zlib

import numpy as np
import pytest

from oracle import oracle_bound_np as ob
from oracle import oracle_ivf_check_np as oc
from oracle import oracle_sq_np as osq

pytestmark = pytest.mark.gpu

L2, IP = ob.METRIC_L2, ob.METRIC_INNER_PRODUCT
f32 = np.float32

SIZES = np.array([0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 3001, 64, 65, 511, 1024], np.int64)
REGIMES = {"small": (12, 5), "mid": (300, 7), "big": (1152, 7)}
K_LADDER = [1, 32, 64, 65, 128, 129, 1024, 2048]
BIG_CERTIFIED = 40


# ------------------------------------------------------------------ payloads
def _ids(rs, shuffle):
    n = int(SIZES.sum())
    ids = rs.permutation(n).astype(np.int64) * 3 + 7 if shuffle else np.arange(n, dtype=np.int64)
    return np.split(ids, np.cumsum(SIZES)[:-1])


def _levels(rs, n, ksub, M):
    """[n, M] codes in [0, ksub); the longest lists hold every value of every sub-quantiser"""
    c = rs.randint(0, ksub, (n, M))
    if n >= ksub:
        c[:ksub] = np.stack([rs.permutation(ksub) for _ in range(M)], 1)
    return c


def _pack(codes, nbits, code_size):
    """[n, M] ints -> the CPU's LSB-first bitstring [n, code_size]"""
    if nbits == 8:
        return codes.astype(np.uint8)
    n, M = codes.shape
    bits = ((codes[:, :, None] >> np.arange(nbits)) & 1).reshape(n, M * nbits).astype(np.uint8)
    bits = np.concatenate([bits, np.zeros((n, code_size * 8 - M * nbits), np.uint8)], 1)
    return np.packbits(bits, axis=1, bitorder="little")


def _set_lists(idx, payload, ids):
    idx.setListSizes(SIZES)
    for l, (codes, li) in enumerate(zip(payload, ids)):
        if li.size:
            idx.setList(l, codes, li)


def _queries(rs, kind, decoded, nq, d):
    """queries next to stored vectors ('clustered') or integers around them ('int')"""
    allv = np.concatenate([x for x in decoded if x.shape[0]])
    base = allv[rs.randint(0, allv.shape[0], nq)]
    if kind == "int":
        return (np.rint(base) + rs.randint(-1, 2, base.shape)).astype(f32)
    return (base + 0.05 * rs.randn(*base.shape)).astype(f32)


def _probe_rows(xq, cent, nprobe, metric, k):
    """float64 probes, with planted rows 0..3: an empty list paired with a one-vector list, a -1 entry, fewer than
    k candidates, exactly k candidates (where a subset of the list lengths adds up to k)"""
    probes, _ = oc.probes(xq, cent, nprobe, metric)
    e0, e1 = int(np.nonzero(SIZES == 0)[0][0]), int(np.nonzero(SIZES == 1)[0][0])
    rest = [l for l in probes[0] if l not in (e0, e1)]
    probes[0] = [e0, e1] + rest[: nprobe - 2]
    probes[1, 1] = -1
    few, tot = [], 0
    for l in np.argsort(SIZES, kind="stable"):
        if len(few) < nprobe and tot + SIZES[l] < k:
            few.append(int(l))
            tot += int(SIZES[l])
    probes[2] = few + [-1] * (nprobe - len(few))
    for r in range(1, nprobe + 1):
        hit = next((c for c in itertools.combinations(range(len(SIZES)), r) if SIZES[list(c)].sum() == k), None)
        if hit is not None:
            probes[3] = list(hit) + [-1] * (nprobe - r)
            break
    q, c = xq.astype(np.float64), cent.astype(np.float64)
    full = (q * q).sum(1)[:, None] + (c * c).sum(1)[None, :] - 2 * q @ c.T if metric == L2 else q @ c.T
    cdis = np.where(probes >= 0, np.take_along_axis(full, np.maximum(probes, 0), 1), 0).astype(f32)
    return probes, cdis


def _certify(D, I, probes, rows, k, metric, list_truth, exact, what):
    """check_topk of each certified row over the union of its probed lists; list_truth(qi, l) -> (t, beta)"""
    for qi in rows:
        ls = [int(l) for l in probes[qi] if l >= 0 and SIZES[l] > 0]
        ids = np.concatenate([list_truth.ids[l] for l in ls]) if ls else np.zeros(0, np.int64)
        tb = [list_truth(qi, l) for l in ls]
        t = np.concatenate([x[0] for x in tb]) if ls else np.zeros(0)
        b = np.zeros_like(t) if exact else (np.concatenate([x[1] for x in tb]) if ls else np.zeros(0))
        ob.check_topk(D[qi], I[qi], ids, t, b, k, metric, what="%s query %d" % (what, qi))


class _Truth:
    def __init__(self, ids, fn):
        self.ids, self.fn = ids, fn

    def __call__(self, qi, l):
        return self.fn(qi, l)


# ------------------------------------------------------------------ builders: (index, decoded lists, truth factory)
def _build_pq(res, fb, d, M, nbits, variant, kind, rs, shuffle):
    nlist, dsub, ksub = len(SIZES), d // M, 1 << nbits
    metric = IP if variant == "ip" else L2
    if kind == "int":
        cent = rs.randint(-4, 5, (nlist, d)).astype(f32)
        pq = rs.randint(-3, 4, (M, ksub, dsub)).astype(f32)
    else:
        cent = (rs.randn(nlist, d) * 2).astype(f32)
        pq = (rs.randn(M, ksub, dsub) * 0.5).astype(f32)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, nbits, metric, interleaved_layout=nbits != 8)
    idx.setCoarseCentroids(cent)
    idx.setPQCentroids(pq)
    idx.setIsTrained(True)
    idx.setPrecomputedCodes(variant == "precomp")
    ids = _ids(rs, shuffle)
    codes = [_levels(rs, int(n), ksub, M) for n in SIZES]
    _set_lists(idx, [_pack(c, nbits, idx._code_size()) for c in codes], ids)
    # the index's own lists, decoded (and its codes equal to what was set)
    Yd = []
    for l in range(nlist):
        li, raw = idx.getListIndices(l), idx.getListVectorData(l)
        assert np.array_equal(li, ids[l]), "list %d ids" % l
        got = oc.unpack(raw.reshape(li.size, idx._code_size()), M, nbits)
        assert np.array_equal(got, codes[l]), "list %d codes" % l
        Yd.append(pq[np.arange(M)[None, :], got].reshape(li.size, d).astype(np.float64))
    decoded = [cent[l][None, :].astype(np.float64) + Yd[l] for l in range(nlist)]

    def truth(xq):
        def fn(qi, l):
            if variant == "precomp":
                return ob.pq_l2_precomp_truth(xq[qi], cent[l], Yd[l], dsub, M)
            if variant == "direct":
                return ob.pq_l2_truth(xq[qi].astype(np.float64) - cent[l], Yd[l], dsub, M)
            return ob.pq_ip_truth(xq[qi], cent[l], Yd[l], dsub, M)

        return _Truth(ids, fn)

    return idx, metric, cent, decoded, truth


def _build_flat(res, fb, d, variant, kind, rs, shuffle):
    nlist = len(SIZES)
    metric = IP if variant == "ip" else L2
    cent = (rs.randn(nlist, d) * 2).astype(f32)
    if kind == "int":
        cent = np.rint(cent * 2).astype(f32)
        X = [(cent[l] + rs.randint(-3, 4, (int(n), d))).astype(f32) for l, n in enumerate(SIZES)]
    else:
        X = [(cent[l] + rs.randn(int(n), d)).astype(f32) for l, n in enumerate(SIZES)]
    idx = fb.GpuIndexIVFFlat(res, d, nlist, metric)
    idx.setCoarseCentroids(cent)
    idx.setIsTrained(True)
    ids = _ids(rs, shuffle)
    _set_lists(idx, [x.view(np.uint8) for x in X], ids)
    for l in range(nlist):
        assert np.array_equal(idx.getListVectorData(l).view(f32).reshape(-1, d), X[l]), "list %d vectors" % l

    def truth(xq):
        def fn(qi, l):
            return ob.l2_truth(xq[qi], X[l]) if metric == L2 else ob.ip_truth(xq[qi], X[l])

        return _Truth(ids, fn)

    return idx, metric, cent, [x.astype(np.float64) for x in X], truth


def _build_sq(res, fb, d, qtype, residual, variant, kind, rs, shuffle):
    nlist = len(SIZES)
    metric = IP if variant == "ip" else L2
    cent = (rs.randn(nlist, d) * 2).astype(f32)
    if kind == "int":
        cent = np.rint(cent).astype(f32)
    cs = osq.code_size(qtype, d)
    if qtype in osq.UNIFORM:
        trained = np.array([-3.0, 6.5], f32)
    elif qtype in osq.NON_UNIFORM:
        trained = np.concatenate([rs.randn(d) * 2 - 2, np.abs(rs.randn(d)) * 3 + 0.1]).astype(f32)
    else:
        trained = np.zeros(0, f32)
    payload = []
    for n in SIZES:
        n = int(n)
        if qtype == osq.QT_fp16:
            v = rs.randint(-8, 9, (n, d)) if kind == "int" else rs.randn(n, d) * 2
            payload.append(np.ascontiguousarray(v.astype(np.float16)).view(np.uint8).reshape(n, cs))
        elif qtype == osq.QT_8bit_direct:
            payload.append(rs.randint(0, 256 if kind != "int" else 16, (n, cs)).astype(np.uint8))
        else:
            c = rs.randint(0, 256, (n, cs)).astype(np.uint8)
            if n >= 256:
                c[:256] = np.arange(256, dtype=np.uint8)[:, None]
            payload.append(c)
    idx = fb.GpuIndexIVFScalarQuantizer(res, d, nlist, qtype, metric, encodeResidual=residual)
    idx.setCoarseCentroids(cent)
    idx.setTrained(trained)
    idx.setIsTrained(True)
    ids = _ids(rs, shuffle)
    _set_lists(idx, payload, ids)
    s = oc.sq_levels(qtype)
    dec = []
    for l in range(nlist):
        raw = idx.getListVectorData(l)
        assert np.array_equal(raw.reshape(-1, cs), payload[l]), "list %d codes" % l
        dec.append(oc.sq_exact_decode(raw, qtype, trained, d))
    decoded = [x + (cent[l].astype(np.float64) if residual else 0.0) for l, (x, _, _) in enumerate(dec)]

    def truth(xq):
        def fn(qi, l):
            X, vmin, vdiff = dec[l]
            c = cent[l].astype(np.float64) if residual else np.zeros(d)
            if metric == L2:
                return ob.sq_l2_truth(xq[qi].astype(np.float64) - c, X, vmin, vdiff)
            return ob.sq_ip_truth(xq[qi], X, vmin, vdiff, s, float(xq[qi].astype(np.float64) @ c))

        return _Truth(ids, fn)

    return idx, metric, cent, decoded, truth


# ------------------------------------------------------------------ the case matrix
PQ_ILV = [(128, 32), (96, 32), (64, 16), (64, 32), (32, 32), (48, 16), (256, 32)]  # dsub 4, 3, 4, 2, 1, 3, 8
PQ_NIB = [(128, 32), (128, 64), (192, 64)]
PQ_VEC = [(128, 8), (96, 12), (192, 48), (128, 64), (120, 24), (7, 7)]  # vec16: 48, 64; dsub 5: (120, 24)
PQ_PACKED = [(64, 16, 5), (96, 16, 6), (64, 8, 4), (120, 20, 6)]  # (64, 8, 4): M / 2 = 4 bytes, packed
FLAT_D = [128, 256, 3, 31, 33, 64, 96, 100, 129, 200]  # 128 / 256: the fast path
# (qtype, d): fast paths (8-bit 128 / 256, 4-bit 256, fp16 64..256), generic 8-bit 100, odd 4-bit 33, 6-bit 17
# and 64, fp16 40
SQ_SHAPES = [(osq.QT_8bit, 128), (osq.QT_8bit, 256), (osq.QT_8bit_uniform, 128), (osq.QT_4bit, 256),
             (osq.QT_4bit_uniform, 256), (osq.QT_fp16, 64), (osq.QT_fp16, 128), (osq.QT_fp16, 256),
             (osq.QT_8bit, 100), (osq.QT_4bit, 33), (osq.QT_6bit, 17), (osq.QT_6bit, 64), (osq.QT_fp16, 40),
             (osq.QT_8bit_direct, 128), (osq.QT_4bit_uniform, 33)]
REG = ["small", "mid", "big"]


def _cases():
    out = []
    n = itertools.count()

    def add(*c):
        i = next(n)
        # the regime turns one step slower than the three variants of a shape, so no variant keeps one regime
        out.append(c + (K_LADDER[i % len(K_LADDER)], REG[(i + i // 3) % 3], i % 2 == 1))

    # interleaved 8-bit: every shape x {direct, precomputed, IP} on integers, and once more on clustered data
    for (d, M), v in itertools.product(PQ_ILV, ["direct", "precomp", "ip"]):
        add("pq", d, M, 8, v, "int")
    for i, (d, M) in enumerate(PQ_ILV):
        add("pq", d, M, 8, ["direct", "precomp", "ip"][i % 3], "clustered")
    for (d, M), v in itertools.product(PQ_NIB, ["direct", "ip"]):
        add("pq", d, M, 4, v, "clustered")
    for (d, M), v in itertools.product(PQ_VEC, ["direct", "ip"]):
        add("pq", d, M, 8, v, "clustered" if d != 7 else "int")
    for (d, M, nb), v in itertools.product(PQ_PACKED, ["direct", "ip"]):
        add("pq", d, M, nb, v, "clustered")
    for i, (d, v) in enumerate(itertools.product(FLAT_D, ["l2", "ip"])):
        add("flat", d, None, None, v, "int" if i % 3 == 0 else "clustered")
    for i, ((qt, d), v) in enumerate(itertools.product(SQ_SHAPES, ["l2", "ip"])):
        exact = qt == osq.QT_8bit_direct or (qt == osq.QT_fp16 and d == 128)
        add("sq", d, qt, (i // 2 + i) % 2 == 0, v, "int" if exact else "clustered")
    return out


CASES = _cases()


def _case_id(c):
    fam, d, a, b, v, kind, k, reg, sh = c
    shape = "d%d_M%d_b%d" % (d, a, b) if fam == "pq" else "d%d" % d if fam == "flat" else "d%d_qt%d_res%d" % (d, a, b)
    return "%s-%s-%s-%s-k%d-%s%s" % (fam, shape, v, kind, k, reg, "-shuf" if sh else "")


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_ivf_scan_certified(res, case):
    import faiss_b200 as fb

    fam, d, a, b, variant, kind, k, regime, shuffle = case
    rs = np.random.RandomState(zlib.crc32(_case_id(case).encode()))
    if fam == "pq":
        idx, metric, cent, decoded, truth = _build_pq(res, fb, d, a, b, variant, kind, rs, shuffle)
    elif fam == "flat":
        idx, metric, cent, decoded, truth = _build_flat(res, fb, d, variant, kind, rs, shuffle)
    else:
        idx, metric, cent, decoded, truth = _build_sq(res, fb, d, a, b, variant, kind, rs, shuffle)
    nq, nprobe = REGIMES[regime]
    xq = _queries(rs, kind, decoded, nq, d)
    probes, cdis = _probe_rows(xq, cent, nprobe, metric, k)
    D, I = oc.search_preassigned(idx, xq, k, probes, cdis)
    rows = range(BIG_CERTIFIED) if regime == "big" else range(nq)
    _certify(D, I, probes, rows, k, metric, truth(xq), kind == "int", _case_id(case))


def test_case_matrix_covers_the_ladder_and_regimes():
    """every k of the ladder and every query regime appears for each scan family"""
    for fam in ("pq", "flat", "sq"):
        ks = {c[6] for c in CASES if c[0] == fam}
        regs = {c[7] for c in CASES if c[0] == fam}
        assert ks == set(K_LADDER), (fam, ks)
        assert regs == set(REG), (fam, regs)


# ------------------------------------------------------------------ add-built PQ: the device's encoding
# (d, M): dsub 1, 2, 3, 4, 5 (the encode kernel's runtime branch), 6
ENCODE_SHAPES = [(32, 32), (64, 32), (96, 32), (128, 32), (120, 24), (96, 16)]


@pytest.mark.parametrize("d,M", ENCODE_SHAPES)
@pytest.mark.parametrize("kind", ["int", "clustered"])
def test_ivfpq_add_encodes_nearest_code(res, d, M, kind):
    """codes of add() are the first float64 minimum of every residual sub-vector (integers: exactly; float data:
    a different pick only within the two sub-distances' bounds), and the search over them certifies"""
    import faiss_b200 as fb

    nlist, N, dsub = 16, 6000, d // M
    rs = np.random.RandomState(d * 100 + M + len(kind))
    if kind == "int":
        cent = rs.randint(-4, 5, (nlist, d)).astype(f32)
        pq = rs.randint(-3, 4, (M, 256, dsub)).astype(f32)
        xb = (cent[rs.randint(0, nlist, N)] + rs.randint(-3, 4, (N, d))).astype(f32)
    else:
        cent = (rs.randn(nlist, d) * 2).astype(f32)
        pq = (rs.randn(M, 256, dsub) * 0.5).astype(f32)
        xb = (cent[rs.randint(0, nlist, N)] + 0.5 * rs.randn(N, d)).astype(f32)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, L2)
    idx.setCoarseCentroids(cent)
    idx.setPQCentroids(pq)
    idx.setIsTrained(True)
    idx.setPrecomputedCodes(False)
    idx.add_with_ids(xb, np.arange(N, dtype=np.int64)[::-1].copy())
    for l in range(nlist):
        li, raw = idx.getListIndices(l), idx.getListVectorData(l)
        oc.pq_check_codes(xb[N - 1 - li], cent[l], pq, oc.unpack(raw.reshape(li.size, -1), M, 8), M, kind == "int")


# ------------------------------------------------------------------ search == search_preassigned
# (family, d, M or qtype, nbits or residual): PQ interleaved, vector-major, packed and nibble layouts; SQ with and
# without residuals
SAME_CASES = [("pq", 128, 32, 8), ("pq", 128, 8, 8), ("pq", 64, 16, 5), ("pq", 128, 32, 4),
              ("sq", 128, osq.QT_8bit, True), ("sq", 128, osq.QT_8bit, False), ("sq", 100, osq.QT_6bit, True)]


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("fam,d,a,b", SAME_CASES)
def test_search_equals_search_preassigned(res, fam, d, a, b, metric):
    """search(xq, k) == search_preassigned with the coarse result of the index's own shared quantizer, bit for bit
    (for IP the coarse distance enters the key)"""
    import faiss_b200 as fb

    nlist, N, nq, nprobe, k = 32, 20000, 300, 7, 50
    rs = np.random.RandomState(d + a + int(b) + metric)
    cent = (rs.randn(nlist, d) * 2).astype(f32)
    xb = (cent[rs.randint(0, nlist, N)] + rs.randn(N, d)).astype(f32)
    xq = (xb[rs.randint(0, N, nq)] + 0.1 * rs.randn(nq, d)).astype(f32)
    cq = fb.GpuIndexFlat(res, d, metric)
    cq.add(cent)
    if fam == "pq":
        idx = fb.GpuIndexIVFPQ(res, d, nlist, a, b, metric, quantizer=cq, interleaved_layout=b != 8)
        idx.setPQCentroids((rs.randn(a, 1 << b, d // a) * 0.5).astype(f32))
    else:
        idx = fb.GpuIndexIVFScalarQuantizer(res, d, nlist, a, metric, encodeResidual=b, quantizer=cq)
        idx.setTrained(osq.train_minmax(xb - (cent[0] if b else 0), a))
    idx.setIsTrained(True)
    idx.add(xb)
    idx.nprobe = nprobe
    D, I = idx.search(xq, k)
    cD, cI = cq.search(xq, nprobe)
    D2, I2 = idx.search_preassigned(xq, k, cI, cD)
    assert np.array_equal(I, I2), "ids differ in %d rows" % int((I != I2).any(1).sum())
    assert np.array_equal(D, D2), "distances differ in %d rows" % int((D != D2).any(1).sum())
