"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's LocalSearchQuantizer encoding:
oracle/_ref/libfaiss_ref_lsq.so (oracle/ref_lsq_shim.cpp, built by oracle/Makefile) over the UNMODIFIED reference CPU
library of oracle/ref.py.

Only tests/, tests/golden/ and bench_icm.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes

import numpy as np

from oracle import ref

_f = ctypes.POINTER(ctypes.c_float)
_i32 = ctypes.POINTER(ctypes.c_int32)
_u32 = ctypes.POINTER(ctypes.c_uint32)


def _declare(L):
    L.ref_lsq_new.restype = ctypes.c_void_p
    L.ref_lsq_new.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, _f, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    L.ref_lsq_free.argtypes = [ctypes.c_void_p]
    L.ref_lsq_free.restype = None
    L.ref_lsq_compute_codes.argtypes = [ctypes.c_void_p, _f, ctypes.c_int64, _i32]
    L.ref_lsq_icm_encode.argtypes = [ctypes.c_void_p, _i32, _f, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32, _u32]
    L.ref_lsq_draws.argtypes = [ctypes.c_int64] * 5 + [ctypes.c_uint32, ctypes.c_int64, _i32, _u32]


_shim = ref.Shim("lsq", _declare)
LIB_PATH, build, available, lib, _ck = _shim.path, _shim.build, _shim.available, _shim.lib, _shim.ck


class LSQ:
    """a reference LocalSearchQuantizer(d, M, nbits) with the given codebooks [M, K, d], marked trained"""

    def __init__(self, codebooks, nperts=4, icm_iters=4, encode_ils_iters=16, random_seed=0x12345):
        cb = np.ascontiguousarray(codebooks, np.float32)
        self.M, self.K, self.d = cb.shape
        nbits = int(self.K).bit_length() - 1
        assert 1 << nbits == self.K, "the reference LSQ takes K = 2^nbits"
        self.h = lib().ref_lsq_new(self.d, self.M, nbits, cb.ctypes.data_as(_f), nperts, icm_iters, encode_ils_iters, random_seed)
        if not self.h:
            _ck(-1)

    def __del__(self):
        if getattr(self, "h", None):
            lib().ref_lsq_free(self.h)
            self.h = None

    def compute_codes(self, x):
        """LocalSearchQuantizer::compute_codes, unpacked -> int32 [n, M]"""
        x = np.ascontiguousarray(x, np.float32)
        out = np.empty((x.shape[0], self.M), np.int32)
        _ck(lib().ref_lsq_compute_codes(self.h, x.ctypes.data_as(_f), x.shape[0], out.ctypes.data_as(_i32)))
        return out

    def icm_encode(self, codes, x, ils_iters, seed):
        """lsq::IcmEncoder::encode with std::mt19937(seed) -> (codes [n, M], the generator's next output)"""
        x = np.ascontiguousarray(x, np.float32)
        c = np.array(codes, np.int32, order="C")
        nxt = ctypes.c_uint32()
        _ck(lib().ref_lsq_icm_encode(self.h, c.ctypes.data_as(_i32), x.ctypes.data_as(_f), x.shape[0], ils_iters, seed, ctypes.byref(nxt)))
        return c, nxt.value


def draws(M, K, nperts, n, ils_iters, seed, skip=0):
    """perturb_codes' draws from std::mt19937(seed) after `skip` outputs -> ([ils_iters, n, nperts, 2] int32, next output)"""
    out = np.empty((ils_iters, n, nperts, 2), np.int32)
    nxt = ctypes.c_uint32()
    _ck(lib().ref_lsq_draws(M, K, nperts, n, ils_iters, seed, skip, out.ctypes.data_as(_i32), ctypes.byref(nxt)))
    return out, nxt.value
