"""The reference IndexIVFPQ with any nbits: ref.IndexIVFPQ sized from ProductQuantizer's ksub = 2^nbits and
code_size = ceil(M * nbits / 8) (ref.IndexIVFPQ sizes these for nbits = 8).  Same shim entry points."""
import ctypes

import numpy as np

from oracle import ref
from oracle.ref import _ck, _f, _p, _u8


class IndexIVFPQ(ref.IndexIVFPQ):
    def __init__(self, d, nlist, M, nbits=8, metric=1):
        super().__init__(d, nlist, M, nbits, metric)
        self.nbits = nbits
        self.pq_code_size = (M * nbits + 7) // 8

    def pq_centroids(self):
        out = np.empty((self.M, 1 << self.nbits, self.d // self.M), dtype=np.float32)
        _ck(ref.lib().ref_ivfpq_get_pq_centroids(self.h, _p(out, _f)))
        return out

    def pq_compute_codes(self, x):
        """ProductQuantizer::compute_codes: [n, code_size] packed bytes"""
        x = np.ascontiguousarray(x, dtype=np.float32)
        codes = np.empty((x.shape[0], self.pq_code_size), dtype=np.uint8)
        _ck(ref.lib().ref_pq_compute_codes(self.h, _p(x, _f), _p(codes, _u8), ctypes.c_int64(x.shape[0])))
        return codes
