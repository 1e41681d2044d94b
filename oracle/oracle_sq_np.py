"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the reference CPU scalar quantiser and of
IndexIVFScalarQuantizer search, for the parity tests of GpuIndexIVFScalarQuantizer.

Sources restated (reference tree):
  faiss/impl/ScalarQuantizer.cpp:451-520     code_size per type
  faiss/impl/scalar_quantizer/training.cpp:209-383   RS_minmax ranges (uniform / per dimension)
  faiss/impl/scalar_quantizer/quantizers.h:66-150    encode (x - vmin) / vdiff, clamp; decode vmin + xi * vdiff
  faiss/impl/scalar_quantizer/quantizers.h:238-341   fp16 and 8bit_direct
  faiss/impl/scalar_quantizer/codecs.h:25-120        8-, 4- and 6-bit component codecs and bit layouts
  faiss/utils/fp16-fp16c.h                           fp16 encode rounds to nearest even (avx2 build)
  faiss/impl/scalar_quantizer/scanners.h:44-135      IVF scanners: L2 on q - c_list when by_residual,
                                                     IP adds the coarse distance when by_residual
"""
import numpy as np

from oracle.oracle_np import METRIC_L2, METRIC_INNER_PRODUCT, _finish, _topk_sorted, knn_flat  # noqa: F401

QT_8bit, QT_4bit, QT_8bit_uniform, QT_4bit_uniform, QT_fp16, QT_8bit_direct, QT_6bit = range(7)
UNIFORM = (QT_8bit_uniform, QT_4bit_uniform)
NON_UNIFORM = (QT_8bit, QT_4bit, QT_6bit)


def code_size(qtype, d):
    if qtype in (QT_4bit, QT_4bit_uniform):
        return (d + 1) // 2
    if qtype == QT_6bit:
        return (d * 6 + 7) // 8
    if qtype == QT_fp16:
        return 2 * d
    return d


def _levels(qtype):
    return 15 if qtype in (QT_4bit, QT_4bit_uniform) else 63 if qtype == QT_6bit else 255


def train_minmax(x, qtype, rangestat_arg=0.0):
    """ScalarQuantizer::train with RS_minmax: [vmin, vdiff] over all values (uniform types) or
    [vmin[d], vdiff[d]] per dimension (non-uniform); empty for fp16 / 8bit_direct."""
    x = np.asarray(x, dtype=np.float32)
    arg = np.float32(rangestat_arg)
    if qtype in UNIFORM:
        vmin, vmax = np.float32(x.min()), np.float32(x.max())
        vexp = np.float32((vmax - vmin) * arg)
        vmin, vmax = np.float32(vmin - vexp), np.float32(vmax + vexp)
        return np.array([vmin, np.float32(vmax - vmin)], dtype=np.float32)
    if qtype in NON_UNIFORM:
        vmin, vmax = x.min(0), x.max(0)
        vexp = ((vmax - vmin) * arg).astype(np.float32)
        vmin, vmax = (vmin - vexp).astype(np.float32), (vmax + vexp).astype(np.float32)
        return np.concatenate([vmin, (vmax - vmin).astype(np.float32)])
    return np.zeros(0, dtype=np.float32)


def _ranges(qtype, trained, d):
    trained = np.asarray(trained, dtype=np.float32)
    if qtype in UNIFORM:
        return np.full(d, trained[0], np.float32), np.full(d, trained[1], np.float32)
    return trained[:d], trained[d : 2 * d]


def sq_encode(x, qtype, trained):
    """Codes [n, code_size] of the rows of x, byte for byte the CPU's encode_vector."""
    x = np.asarray(x, dtype=np.float32)
    n, d = x.shape
    if qtype == QT_fp16:
        return np.ascontiguousarray(x.astype(np.float16)).view(np.uint8).reshape(n, 2 * d)
    if qtype == QT_8bit_direct:
        # (uint8_t)x: the low byte of the truncated integer
        return (np.trunc(x).astype(np.int64) & 0xFF).astype(np.uint8)
    vmin, vdiff = _ranges(qtype, trained, d)
    with np.errstate(divide="ignore", invalid="ignore"):
        xi = ((x - vmin[None, :]) / vdiff[None, :]).astype(np.float32)
    xi = np.where(vdiff[None, :] != 0, xi, np.float32(0))
    xi = np.clip(xi, np.float32(0), np.float32(1))
    if qtype in (QT_8bit, QT_8bit_uniform):
        return (np.float32(255) * xi).astype(np.float32).astype(np.int64).astype(np.uint8)  # fp32 product, truncated
    # 4- and 6-bit: (int)(xi * 15.0) / (int)(xi * 63.0) are double products, truncated
    lev = (xi.astype(np.float64) * float(_levels(qtype))).astype(np.int64)
    cs = code_size(qtype, d)
    codes = np.zeros((n, cs), dtype=np.int64)
    if qtype in (QT_4bit, QT_4bit_uniform):
        for i in range(d):
            codes[:, i // 2] |= lev[:, i] << ((i & 1) * 4)
        return (codes & 0xFF).astype(np.uint8)
    for i in range(d):  # 6-bit: codecs.h:64-92, 4 components in 3 bytes
        g, b = (i >> 2) * 3, lev[:, i]
        r = i & 3
        if r == 0:
            codes[:, g] |= b
        elif r == 1:
            codes[:, g] |= b << 6
            codes[:, g + 1] |= b >> 2
        elif r == 2:
            codes[:, g + 1] |= b << 4
            codes[:, g + 2] |= b >> 4
        else:
            codes[:, g + 2] |= b << 2
    return (codes & 0xFF).astype(np.uint8)


def sq_decode(codes, qtype, trained, d):
    """decode_vector: [n, d] float32"""
    codes = np.asarray(codes, dtype=np.uint8).reshape(-1, code_size(qtype, d))
    n = codes.shape[0]
    if qtype == QT_fp16:
        return np.ascontiguousarray(codes).view(np.float16).reshape(n, d).astype(np.float32)
    if qtype == QT_8bit_direct:
        return codes.astype(np.float32)
    c = codes.astype(np.int64)
    if qtype in (QT_8bit, QT_8bit_uniform):
        lev = c
    elif qtype in (QT_4bit, QT_4bit_uniform):
        i = np.arange(d)
        lev = (c[:, i // 2] >> ((i & 1) * 4)) & 0xF
    else:
        lev = np.empty((n, d), dtype=np.int64)
        for i in range(d):
            g, r = (i >> 2) * 3, i & 3
            if r == 0:
                lev[:, i] = c[:, g] & 0x3F
            elif r == 1:
                lev[:, i] = (c[:, g] >> 6) | ((c[:, g + 1] & 0xF) << 2)
            elif r == 2:
                lev[:, i] = (c[:, g + 1] >> 4) | ((c[:, g + 2] & 3) << 4)
            else:
                lev[:, i] = c[:, g + 2] >> 2
    xi = ((lev.astype(np.float32) + np.float32(0.5)) / np.float32(_levels(qtype))).astype(np.float32)
    vmin, vdiff = _ranges(qtype, trained, d)
    return (vmin[None, :] + xi * vdiff[None, :]).astype(np.float32)


def ivfsq_search(xq, k, nprobe, centroids, qtype, trained, lists_codes, lists_ids, metric=METRIC_L2, by_residual=True,
                 probes=None, centroid_dis=None):
    """IndexIVFScalarQuantizer::search / search_preassigned: decode each probed list, L2 against q - c_list
    (by_residual) or q; IP q . x plus the coarse distance (by_residual).  Distances in float64, rounded."""
    xq = np.asarray(xq, dtype=np.float32)
    nq, d = xq.shape
    if probes is None:
        centroid_dis, probes = knn_flat(xq, centroids, nprobe, metric)
    D = np.empty((nq, k), dtype=np.float32)
    I = np.empty((nq, k), dtype=np.int64)
    for qi in range(nq):
        keys, ids = [], []
        for p in range(probes.shape[1]):
            l = probes[qi, p]
            if l < 0 or np.asarray(lists_ids[l]).size == 0:
                continue
            x = sq_decode(lists_codes[l], qtype, trained, d).astype(np.float64)
            q = xq[qi].astype(np.float64)
            if metric == METRIC_L2:
                r = (xq[qi] - centroids[l]).astype(np.float64) if by_residual else q
                dis = ((x - r[None, :]) ** 2).sum(1)
                keys.append(dis.astype(np.float32))
            else:
                dis = x @ q + (float(centroid_dis[qi, p]) if by_residual else 0.0)
                keys.append(-dis.astype(np.float32))
            ids.append(np.asarray(lists_ids[l], dtype=np.int64))
        if keys:
            kk, ii = _topk_sorted(np.concatenate(keys)[None, :], np.concatenate(ids)[None, :], k)
        else:
            kk = np.full((1, k), np.inf, dtype=np.float32)
            ii = np.full((1, k), -1, dtype=np.int64)
        D[qi], I[qi] = _finish(kk, ii, metric)
    return D, I
