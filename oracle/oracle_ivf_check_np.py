"""TEST INFRASTRUCTURE ONLY -- what the certified IVF tests need besides the bounds of oracle_bound_np: float64
probes from an index's own centroids, its probed lists, PQ code unpacking and checking, and the exact SQ decode.

numpy only; it does not import the product (the functions that take an index only call its methods).
"""
import numpy as np

from oracle import oracle_bound_np as ob
from oracle import oracle_sq_np as osq

f32 = np.float32


def probes(xq, cent, nprobe, metric):
    """probes and coarse distances in float64 from the index's own centroids; ties by ascending list number"""
    q, c = xq.astype(np.float64), cent.astype(np.float64)
    if metric == ob.METRIC_L2:
        dis = (q * q).sum(1)[:, None] + (c * c).sum(1)[None, :] - 2 * q @ c.T
        order = np.argsort(dis, 1, kind="stable")[:, :nprobe]
    else:
        dis = q @ c.T
        order = np.argsort(-dis, 1, kind="stable")[:, :nprobe]
    return order.astype(np.int64), np.take_along_axis(dis, order, 1).astype(f32)


def search_preassigned(idx, xq, k, assign, cdis):
    """IndexIVF::search_preassigned reads nprobe entries of every assign row, nprobe being the index's"""
    idx.nprobe = assign.shape[1]
    return idx.search_preassigned(xq, k, assign, cdis)


def probed_lists(idx, probes_row):
    """(list number, ids, raw codes) of every probed list of one query; -1 entries probe nothing"""
    return [(int(l), idx.getListIndices(int(l)), idx.getListVectorData(int(l))) for l in probes_row if l >= 0]


def unpack(codes, M, nbits):
    """ProductQuantizer codes [n, code_size] (LSB-first bitstring) -> [n, M] ints"""
    if nbits == 8:
        return codes.astype(np.int64)
    bits = np.unpackbits(codes, axis=1, bitorder="little")
    w = 1 << np.arange(nbits)
    return (bits[:, : M * nbits].reshape(-1, M, nbits) * w).sum(2).astype(np.int64)


def pq_check_codes(x, cent_l, pq, codes, M, exact):
    """codes against the float64 argmin of the residual sub-vectors; a different pick is allowed only where
    the two sub-distances lie within their bounds (exact: never -- the first minimum wins)"""
    dsub = pq.shape[2]
    r = x.astype(np.float64) - cent_l.astype(np.float64)[None, :]
    for m in range(M):
        rm = r[:, m * dsub : (m + 1) * dsub]
        y = pq[m].astype(np.float64)
        dist = (rm * rm).sum(1)[:, None] + (y * y).sum(1)[None, :] - 2 * rm @ y.T  # exact on integers
        best = np.argmin(dist, 1)
        got = codes[:, m]
        bad = np.nonzero(got != best)[0]
        if bad.size == 0:
            continue
        assert not exact, "sub-quantiser %d: codes %s, first minimum %s" % (m, got[bad][:5], best[bad][:5])
        for i in bad:
            pair = np.array([got[i], best[i]])
            diff = rm[i][None, :] - y[pair]
            t = (diff * diff).sum(1)
            e = np.broadcast_to(2 * ob.U * np.abs(rm[i])[None, :], diff.shape)
            beta = ob.perturbed_l2_bound(diff, e, dsub + 3) + ob.slack((rm[i] ** 2).sum() + (y[pair] ** 2).sum(1), 4 * dsub)
            assert t[0] - t[1] <= beta.sum(), "sub-quantiser %d, vector %d: code %d is %.3e worse than %d (bound %.3e)" % (
                m, i, got[i], t[0] - t[1], best[i], beta.sum())


def sq_levels(qtype):
    """s of the decode vmin + vdiff (c + 1/2) / s; 1 for fp16 / 8bit_direct (the code is the value)"""
    return 1 if qtype in (osq.QT_fp16, osq.QT_8bit_direct) else osq._levels(qtype)


def sq_exact_decode(codes, qtype, trained, d):
    """float64 decode vmin + vdiff (c + 1/2) / s of the index's codes (the kernel's reference value), vmin, vdiff"""
    x32 = osq.sq_decode(codes, qtype, trained, d)
    if qtype in (osq.QT_fp16, osq.QT_8bit_direct):
        return x32.astype(np.float64), np.zeros(d), np.zeros(d)
    s = osq._levels(qtype)
    unit = osq.sq_decode(codes, qtype, np.concatenate([np.zeros(d), np.ones(d)]).astype(f32)
                         if qtype in osq.NON_UNIFORM else np.array([0, 1], f32), d)
    lev = np.rint(unit.astype(np.float64) * s - 0.5)  # (c + 1/2) / s rounded to fp32 still names c
    vmin, vdiff = osq._ranges(qtype, trained, d)
    vmin, vdiff = vmin.astype(np.float64), vdiff.astype(np.float64)
    return vmin[None, :] + vdiff[None, :] * (lev + 0.5) / s, vmin, vdiff
