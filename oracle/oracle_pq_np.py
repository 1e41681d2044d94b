"""Numpy restatement of the reference's packed PQ codes (nbits < 8) and an IVF-PQ search over them.

ProductQuantizer::code_size = ceil(M * nbits / 8) bytes per vector (faiss/impl/ProductQuantizer.cpp
set_derived_values).  The codes of a vector form one LSB-first bitstring: code m occupies bits
[m * nbits, (m + 1) * nbits), bit b of the string being bit (b % 8) of byte b // 8; the last byte is padded
with zero bits.  That is what PQEncoderGeneric writes and PQDecoderGeneric reads
(faiss/impl/ProductQuantizer-inl.h:12-59 and :67-101).  For nbits = 8 the string is the codes themselves.
"""
import numpy as np

from oracle import oracle_np as o


def pq_code_size(M, nbits):
    return (M * nbits + 7) // 8


def pq_pack_codes(codes, nbits):
    """codes [n, M] (values < 2^nbits) -> packed [n, ceil(M * nbits / 8)] uint8 (PQEncoderGeneric::encode,
    ProductQuantizer-inl.h:23-40, flushed by ~PQEncoderGeneric, :42-46)"""
    codes = np.asarray(codes, dtype=np.uint64)
    n, M = codes.shape
    cs = pq_code_size(M, nbits)
    bits = ((codes[:, :, None] >> np.arange(nbits, dtype=np.uint64)[None, None, :]) & 1).astype(np.uint8)
    bits = bits.reshape(n, M * nbits)
    bits = np.concatenate([bits, np.zeros((n, cs * 8 - M * nbits), np.uint8)], axis=1)
    return np.packbits(bits.reshape(n, cs, 8), axis=2, bitorder="little").reshape(n, cs)


def pq_unpack_codes(packed, M, nbits):
    """packed [n, code_size] (or flat bytes) -> codes [n, M] uint8 (PQDecoderGeneric::decode, ProductQuantizer-inl.h:76-101)"""
    cs = pq_code_size(M, nbits)
    packed = np.asarray(packed, dtype=np.uint8).reshape(-1, cs)
    n = packed.shape[0]
    bits = np.unpackbits(packed, axis=1, bitorder="little")[:, : M * nbits].reshape(n, M, nbits).astype(np.uint16)
    return (bits << np.arange(nbits, dtype=np.uint16)[None, None, :]).sum(-1).astype(np.uint8)


def ivfpq_search(xq, k, nprobe, centroids, pq_centroids, lists_codes, lists_ids, metric=o.METRIC_L2, probes=None, nbits=8):
    """oracle_np.ivfpq_search over lists holding ProductQuantizer codes of `nbits` bits (the CPU's
    ArrayInvertedLists bytes), unpacked first"""
    M = pq_centroids.shape[0]
    assert pq_centroids.shape[1] == 1 << nbits
    if nbits != 8:
        lists_codes = [pq_unpack_codes(c, M, nbits) for c in lists_codes]
    return o.ivfpq_search(xq, k, nprobe, centroids, pq_centroids, lists_codes, lists_ids, metric, probes=probes)
