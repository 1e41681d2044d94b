"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's LocalSearchQuantizer encoding:
oracle/_ref/libfaiss_ref_lsq.so (oracle/ref_lsq_shim.cpp, built by oracle/lsq.mk) over the UNMODIFIED reference CPU
library of oracle/ref.py.

Only tests/, tests/golden/ and bench_icm.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref_lsq.so")

_f = ctypes.POINTER(ctypes.c_float)
_i32 = ctypes.POINTER(ctypes.c_int32)
_u32 = ctypes.POINTER(ctypes.c_uint32)


def build(verbose=False):
    """Compile oracle/_ref/libfaiss_ref_lsq.so (only where the reference sources are mounted)."""
    if not os.path.isdir("/root/reference/faiss") or not ref.available():
        return available()
    r = subprocess.run(["make", "-C", _HERE, "-f", "lsq.mk"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref LSQ shim build failed:\n" + (r.stdout or "")[-3000:] + (r.stderr or "")[-3000:])
    return True


def available():
    return ref.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        ref.lib()
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref_lsq.so missing: run `make -C oracle -f lsq.mk`")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_lsq_last_error.restype = ctypes.c_char_p
        L.ref_lsq_new.restype = ctypes.c_void_p
        L.ref_lsq_new.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, _f, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.ref_lsq_set_threads.argtypes = [ctypes.c_int]
        L.ref_lsq_set_threads.restype = None
        L.ref_lsq_free.argtypes = [ctypes.c_void_p]
        L.ref_lsq_free.restype = None
        L.ref_lsq_compute_codes.argtypes = [ctypes.c_void_p, _f, ctypes.c_int64, _i32]
        L.ref_lsq_icm_encode.argtypes = [ctypes.c_void_p, _i32, _f, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32, _u32]
        L.ref_lsq_draws.argtypes = [ctypes.c_int64] * 5 + [ctypes.c_uint32, ctypes.c_int64, _i32, _u32]
        _lib = L
    return _lib


def _ck(rc):
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_lsq_last_error().decode(errors="replace"))


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
        if getattr(self, "h", None) and _lib is not None:
            _lib.ref_lsq_free(self.h)
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


def set_threads(n):
    """the OpenMP thread count of the reference encoder"""
    lib().ref_lsq_set_threads(int(n))


def draws(M, K, nperts, n, ils_iters, seed, skip=0):
    """perturb_codes' draws from std::mt19937(seed) after `skip` outputs -> ([ils_iters, n, nperts, 2] int32, next output)"""
    out = np.empty((ils_iters, n, nperts, 2), np.int32)
    nxt = ctypes.c_uint32()
    _ck(lib().ref_lsq_draws(M, K, nperts, n, ils_iters, seed, skip, out.ctypes.data_as(_i32), ctypes.byref(nxt)))
    return out, nxt.value
