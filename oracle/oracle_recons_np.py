"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the reference CPU IndexIVF retrieval, for the parity tests of
reconstruct_n / reconstruct_batch / search_and_reconstruct / search_and_return_codes.

Sources restated (reference tree):
  faiss/IndexIVF.cpp:1073-1090            reconstruct_n: every stored entry with i0 <= id < i0 + ni, lists in order, so
                                          the entry last in (list, offset) order wins
  faiss/IndexIVF.cpp:1183-1248            search_and_return_codes; encode_listno (little-endian, coarse_code_size bytes)
  faiss/IndexIVFPQ.cpp:358-372            reconstruct_from_offset: pq.decode(code), then + centroid[list]
  faiss/IndexScalarQuantizer.cpp:400-425  reconstruct_from_offset: sq.decode(code), then + centroid[list] if by_residual
  faiss/impl/ProductQuantizer-inl.h       PQDecoderGeneric: codes of nbits bits, LSB first
  faiss/impl/scalar_quantizer/quantizers.h:92-146  decode_vector: xi = (c + 0.5f) / s, then vmin + xi * vdiff.
      decode_vector is final in the scalar QuantizerTemplate, so the AVX2 quantizer (d % 8 == 0) decodes with it too;
      the oracle's g++ -O3 -mfma build contracts vmin + xi * vdiff into one fused multiply-add (checked in its
      object code), restated here as one rounding of the exact value.
"""
import numpy as np

from oracle import oracle_sq_np as sq

FLAT, SQ, PQ = 0, 1, 2


def _fma32(a, b, c):
    """round_to_float32(a * b + c) for float32 arrays: the product is exact in float64, the sum is rounded once in
    the 64-bit-mantissa long double and once to float32 (the first rounding cannot reach a float32 tie here: the
    exact sum has at most 24 + 24 + |exponent gap| significant bits, within long double's 64 for the ranges used)"""
    ld = np.longdouble
    return (a.astype(ld) * b.astype(ld) + c.astype(ld)).astype(np.float32)


def sq_decode(codes, qtype, trained, d):
    """ScalarQuantizer::decode of the oracle build: [n, d] float32"""
    codes = np.asarray(codes, dtype=np.uint8).reshape(-1, sq.code_size(qtype, d))
    if qtype in (sq.QT_fp16, sq.QT_8bit_direct):
        return sq.sq_decode(codes, qtype, trained, d)
    n = codes.shape[0]
    c = codes.astype(np.int64)
    if qtype in (sq.QT_8bit, sq.QT_8bit_uniform):
        lev = c
    elif qtype in (sq.QT_4bit, sq.QT_4bit_uniform):
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
    xi = ((lev.astype(np.float32) + np.float32(0.5)) / np.float32(sq._levels(qtype))).astype(np.float32)
    vmin, vdiff = sq._ranges(qtype, trained, d)
    return _fma32(xi, np.broadcast_to(vdiff, xi.shape), np.broadcast_to(vmin, xi.shape))


def pq_codes(codes, M, nbits):
    """the M sub-quantiser indices of each packed code row: [n, M] int64"""
    cs = (M * nbits + 7) // 8
    b = np.asarray(codes, dtype=np.uint8).reshape(-1, cs).astype(np.int64)
    b = np.concatenate([b, np.zeros((b.shape[0], 1), np.int64)], axis=1)
    out = np.empty((b.shape[0], M), dtype=np.int64)
    for m in range(M):
        bit = m * nbits
        w = b[:, bit >> 3] | (b[:, (bit >> 3) + 1] << 8)
        out[:, m] = (w >> (bit & 7)) & ((1 << nbits) - 1)
    return out


def pq_decode(codes, M, nbits, pq_centroids):
    """ProductQuantizer::decode: [n, d]; pq_centroids [M, 2^nbits, dsub]"""
    pqc = np.asarray(pq_centroids, dtype=np.float32).reshape(M, 1 << nbits, -1)
    c = pq_codes(codes, M, nbits)
    return np.concatenate([pqc[m][c[:, m]] for m in range(M)], axis=1).astype(np.float32)


def reconstruct_list(kind, codes, l, d, centroids=None, **kw):
    """reconstruct_from_offset of every entry of list l ([len, d] float32)"""
    if kind == FLAT:
        return np.asarray(codes, dtype=np.uint8).view(np.float32).reshape(-1, d)
    if kind == PQ:
        x = pq_decode(codes, kw["M"], kw["nbits"], kw["pq"])
        return (x + centroids[l][None, :]).astype(np.float32)
    x = sq_decode(codes, kw["qtype"], kw["trained"], d)
    if kw.get("by_residual", True):
        x = (x + centroids[l][None, :]).astype(np.float32)
    return x


def reconstruct_n(kind, lists_codes, lists_ids, i0, ni, d, out, centroids=None, **kw):
    """IndexIVF::reconstruct_n into out [ni, d] (rows of ids not stored are left as they are)"""
    for l, (codes, ids) in enumerate(zip(lists_codes, lists_ids)):
        ids = np.asarray(ids, dtype=np.int64)
        if ids.size == 0:
            continue
        x = reconstruct_list(kind, codes, l, d, centroids, **kw)
        for off, i in enumerate(ids):
            if i0 <= i < i0 + ni:
                out[i - i0] = x[off]
    return out


def coarse_code_size(nlist):
    nbyte, nl = 0, nlist - 1
    while nl > 0:
        nbyte += 1
        nl >>= 8
    return nbyte


def encode_listno(l, nlist):
    return np.array([(l >> (8 * b)) & 0xFF for b in range(coarse_code_size(nlist))], dtype=np.uint8)
