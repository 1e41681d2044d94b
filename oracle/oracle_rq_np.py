"""TEST INFRASTRUCTURE ONLY -- numpy restatement of ResidualQuantizer's beam-search encoding
(faiss/impl/residual_quantizer_encode_steps.cpp, faiss/impl/AdditiveQuantizer.cpp:241-315).

Every fp32 operation the CPU rounds separately is rounded separately here, in the CPU's order:
  refine_beam      dis = (‖r‖² + ‖c‖²) + (−2·⟨r, c⟩)  (pairwise_L2sqr: the norms, then the sgemm with beta = 1);
                   children r − c
  refine_beam_lut  cd[k] = ‖c_k‖² − 2·qcp[k]; dp = Σ_{m1<m} cross_m[off[m1] + code[m1], k] in m1 order, in chunks of
                   8 added one after another; the value is dist + cd at m = 0, (cd + 2·dp) + dist at 1 <= m <= 7 with
                   K >= 32 (the AVX2 finalize), (dist + cd) + 2·dp otherwise
  selection        the B_out smallest by (value, j = b·K + k)
The dot products and squared norms (which the CPU computes with sgemm / SIMD sums) are rounded once from float64, so
the restatement equals the CPU wherever those sums are exact in fp32: integer data and codebooks.
"""
import numpy as np

ST_decompress, ST_LUT_nonorm, ST_norm_from_LUT, ST_norm_float, ST_norm_qint8, ST_norm_qint4 = range(6)
DEVICE_PACKED = (ST_decompress, ST_LUT_nonorm, ST_norm_from_LUT, ST_norm_float, ST_norm_qint8, ST_norm_qint4)
_NORM_BITS = {ST_norm_float: 32, ST_norm_qint8: 8, ST_norm_qint4: 4}

f32 = np.float32


def offsets(nbits):
    return np.concatenate([[0], np.cumsum([1 << int(b) for b in nbits])]).astype(np.int64)


def final_beam(nbits, beam_in, out_beam):
    b = beam_in
    for nb in nbits:
        b = min(b << int(nb), out_beam)
    return b


def _norms(x):
    return (x.astype(np.float64) ** 2).sum(-1).astype(f32)


def _ip(a, b):
    return (a.astype(np.float64) @ b.astype(np.float64).T).astype(f32)


def tables(cb, nbits):
    """(centroid_norms [total_K], [cross_m [off_m, K_m] for m in 0..M-1]) -- compute_codebook_tables"""
    off = offsets(nbits)
    cross = [_ip(cb[: off[m]], cb[off[m]:off[m + 1]]) for m in range(len(nbits))]
    return _norms(cb), cross


def _select(v, out):
    """rows of candidate values [n, C] -> (ids [n, out], values [n, out]) by (value asc, id asc)"""
    order = np.argsort(v, axis=1, kind="stable")[:, :out]
    return order, np.take_along_axis(v, order, 1)


def refine_beam(cb, nbits, residuals, out_beam):
    """ResidualQuantizer::refine_beam: residuals [n, B_in, d] -> (codes [n, B, M], residuals [n, B, d], dis [n, B])"""
    cb = np.asarray(cb, f32)
    r = np.asarray(residuals, f32)
    n, B, d = r.shape
    off = offsets(nbits)
    cnorm = _norms(cb)
    codes = np.zeros((n, B, 0), np.int32)
    dis = None
    for m, nb in enumerate(nbits):
        K = 1 << int(nb)
        cbm = cb[off[m]:off[m + 1]]
        rn = _norms(r.reshape(-1, d)).reshape(n, B)
        ip = _ip(r.reshape(-1, d), cbm).reshape(n, B, K)
        v = (rn[:, :, None] + cnorm[off[m]:off[m + 1]][None, None]) + f32(-2) * ip
        Bo = min(B * K, out_beam)
        ids, dis = _select(v.reshape(n, B * K), Bo)
        js, ls = ids // K, ids % K
        codes = np.concatenate([np.take_along_axis(codes, js[:, :, None], 1), ls[:, :, None].astype(np.int32)], 2)
        r = np.take_along_axis(r, js[:, :, None], 1) - cbm[ls]
        B = Bo
    return codes, r, dis


def refine_beam_lut(cb, nbits, x, out_beam):
    """ResidualQuantizer::refine_beam_LUT on x [n, d] (query_norms and query_cp made from x) -> (codes, dis)"""
    cb = np.asarray(cb, f32)
    x = np.asarray(x, f32)
    n = x.shape[0]
    off = offsets(nbits)
    cnorm, cross = tables(cb, nbits)
    qcp = _ip(x, cb)
    dist = _norms(x)[:, None]
    codes = np.zeros((n, 1, 0), np.int32)
    B = 1
    for m, nb in enumerate(nbits):
        K = 1 << int(nb)
        cd = cnorm[None, off[m]:off[m + 1]] - f32(2) * qcp[:, off[m]:off[m + 1]]  # [n, K]
        if m == 0:
            v = dist[:, :, None] + cd[:, None, :]
        else:
            dp = None
            for c0 in range(0, m, 8):
                s = None
                for m1 in range(c0, min(c0 + 8, m)):
                    row = cross[m][off[m1] + codes[:, :, m1]]  # [n, B, K]
                    s = row if s is None else s + row
                dp = s if dp is None else dp + s
            if m <= 7 and K >= 32:
                v = (cd[:, None, :] + f32(2) * dp) + dist[:, :, None]
            else:
                v = (dist[:, :, None] + cd[:, None, :]) + f32(2) * dp
        Bo = min(B * K, out_beam)
        ids, dist = _select(v.reshape(n, B * K), Bo)
        js, ls = ids // K, ids % K
        codes = np.concatenate([np.take_along_axis(codes, js[:, :, None], 1), ls[:, :, None].astype(np.int32)], 2)
        B = Bo
    return codes, dist


def decode_unpacked(cb, nbits, codes):
    """codes [n, M] -> x [n, d]: C_0[c_0] + C_1[c_1] + ... in m order"""
    off = offsets(nbits)
    x = cb[off[0] + codes[:, 0]].copy()
    for m in range(1, len(nbits)):
        x = x + cb[off[m] + codes[:, m]]
    return x


def _encode_qint(x, amin, amax, levels):
    x1 = (x - f32(amin)) / (f32(amax) - f32(amin)) * f32(levels)
    with np.errstate(invalid="ignore"):
        f = np.floor(x1).astype(np.float64)
        ok = (f >= -2.0 ** 31) & (f < 2.0 ** 31)
        xi = np.where(ok, np.nan_to_num(f), -2.0 ** 31).astype(np.int64)  # x86: 0x80000000 when out of range
    return np.clip(xi, 0, levels - 1).astype(np.uint64)


def encode_norm(norms, search_type, norm_min, norm_max):
    norms = np.asarray(norms, f32)
    if search_type == ST_norm_float:
        return norms.view(np.uint32).astype(np.uint64)
    if search_type == ST_norm_qint8:
        return _encode_qint(norms, norm_min, norm_max, 256)
    if search_type == ST_norm_qint4:
        return _encode_qint(norms, norm_min, norm_max, 16)
    return np.zeros(norms.shape, np.uint64)


def code_size(nbits, search_type):
    return (sum(int(b) for b in nbits) + _NORM_BITS.get(search_type, 0) + 7) // 8


def pack_codes(codes, nbits, search_type=ST_decompress, norms=None, norm_min=0.0, norm_max=0.0):
    """AdditiveQuantizer::pack_codes: each code LSB-first with nbits[m] bits, then encode_norm(norm)"""
    codes = np.asarray(codes)
    n = codes.shape[0]
    fields = [(codes[:, m].astype(np.uint64), int(nb)) for m, nb in enumerate(nbits)]
    if search_type in _NORM_BITS:
        fields.append((encode_norm(norms, search_type, norm_min, norm_max), _NORM_BITS[search_type]))
    bits = np.concatenate([((v[:, None] >> np.arange(nb, dtype=np.uint64)) & 1).astype(np.uint8) for v, nb in fields], 1)
    cs = code_size(nbits, search_type)
    bits = np.concatenate([bits, np.zeros((n, cs * 8 - bits.shape[1]), np.uint8)], 1)
    return np.packbits(bits, axis=1, bitorder="little")


def compute_codes(cb, nbits, x, use_beam_lut, max_beam, search_type=ST_decompress, norm_min=0.0, norm_max=0.0,
                  centroids=None):
    """ResidualQuantizer::compute_codes_add_centroids -> packed [n, code_size]"""
    x = np.asarray(x, f32)
    norms = None
    if use_beam_lut:
        codes, _ = refine_beam_lut(cb, nbits, x, max_beam)
    else:
        codes, r, _ = refine_beam(cb, nbits, x[:, None, :], max_beam)
        norms = _norms(x - r[:, 0])  # ‖x − residual‖²
    c0 = codes[:, 0]
    if search_type in _NORM_BITS and (norms is None or centroids is not None):
        rec = decode_unpacked(np.asarray(cb, f32), nbits, c0)
        if centroids is not None:
            rec = rec + np.asarray(centroids, f32)
        norms = _norms(rec)
    return pack_codes(c0, nbits, search_type, norms, norm_min, norm_max)
