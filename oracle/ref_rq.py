"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's ResidualQuantizer encoding:
oracle/_ref/libfaiss_ref_rq.so (oracle/ref_rq_shim.cpp, built by oracle/rq.mk) over the UNMODIFIED reference CPU
library of oracle/ref.py.

Only tests/, tests/golden/ and bench_rq.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref_rq.so")

_f = ctypes.POINTER(ctypes.c_float)
_i32 = ctypes.POINTER(ctypes.c_int32)
_u8 = ctypes.POINTER(ctypes.c_uint8)

# AdditiveQuantizer::Search_type_t
ST_decompress, ST_LUT_nonorm, ST_norm_from_LUT, ST_norm_float, ST_norm_qint8, ST_norm_qint4 = range(6)
ST_norm_cqint8, ST_norm_cqint4, ST_norm_lsq2x4, ST_norm_rq2x4 = range(6, 10)
Train_default, Train_progressive_dim, Train_refine_codebook = 0, 1, 2


def build(verbose=False):
    """Compile oracle/_ref/libfaiss_ref_rq.so (only where the reference sources are mounted)."""
    if not os.path.isdir("/root/reference/faiss") or not ref.available():
        return available()
    r = subprocess.run(["make", "-C", _HERE, "-f", "rq.mk"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref RQ shim build failed:\n" + (r.stdout or "")[-3000:] + (r.stderr or "")[-3000:])
    return True


def available():
    return ref.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        ref.lib()
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref_rq.so missing: run `make -C oracle -f rq.mk`")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_rq_last_error.restype = ctypes.c_char_p
        L.ref_rq_new.restype = ctypes.c_void_p
        L.ref_rq_new.argtypes = [ctypes.c_int, ctypes.c_int, _i32, ctypes.c_int, _f]
        L.ref_rq_free.argtypes = [ctypes.c_void_p]
        L.ref_rq_free.restype = None
        L.ref_rq_set_threads.argtypes = [ctypes.c_int]
        L.ref_rq_set_threads.restype = None
        L.ref_rq_set_params.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float]
        L.ref_rq_code_size.argtypes = [ctypes.c_void_p]
        L.ref_rq_code_size.restype = ctypes.c_int64
        L.ref_rq_cross_size.argtypes = [ctypes.c_void_p]
        L.ref_rq_cross_size.restype = ctypes.c_int64
        L.ref_rq_train.argtypes = [ctypes.c_void_p, ctypes.c_int64, _f, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.ref_rq_tables.argtypes = [ctypes.c_void_p, _f, _f, _f]
        L.ref_rq_refine_beam.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, _f, ctypes.c_int, _i32, _f, _f]
        L.ref_rq_refine_beam_lut.argtypes = [ctypes.c_void_p, ctypes.c_int64, _f, ctypes.c_int, _i32, _f]
        L.ref_rq_compute_codes.argtypes = [ctypes.c_void_p, _f, ctypes.c_int64, _f, _u8]
        L.ref_rq_decode.argtypes = [ctypes.c_void_p, _u8, ctypes.c_int64, _f]
        _lib = L
    return _lib


def _ck(rc):
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_rq_last_error().decode(errors="replace"))


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def final_beam(nbits, beam_in, out_beam):
    b = beam_in
    for nb in nbits:
        b = min(b << nb, out_beam)
    return b


class RQ:
    """a reference ResidualQuantizer(d, nbits); with codebooks [total_K, d] it is trained and has its tables"""

    def __init__(self, d, nbits, codebooks=None, search_type=ST_decompress, max_beam_size=5, use_beam_LUT=0,
                 norm_min=0.0, norm_max=0.0):
        self.d, self.nbits = int(d), [int(b) for b in nbits]
        self.M = len(self.nbits)
        nb = np.array(self.nbits, np.int32)
        cb = None if codebooks is None else np.ascontiguousarray(codebooks, np.float32)
        self.h = lib().ref_rq_new(self.d, self.M, _p(nb, _i32), int(search_type), _p(cb, _f))
        if not self.h:
            _ck(-1)
        self.set_params(max_beam_size, use_beam_LUT, norm_min, norm_max)

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.ref_rq_free(self.h)
            self.h = None

    def set_params(self, max_beam_size, use_beam_LUT, norm_min=0.0, norm_max=0.0):
        _ck(lib().ref_rq_set_params(self.h, int(max_beam_size), int(use_beam_LUT), float(norm_min), float(norm_max)))

    @property
    def code_size(self):
        return int(lib().ref_rq_code_size(self.h))

    @property
    def total_k(self):
        return sum(1 << b for b in self.nbits)

    def train(self, x, train_type=Train_progressive_dim, max_beam_size=5, niter=25):
        x = np.ascontiguousarray(x, np.float32)
        _ck(lib().ref_rq_train(self.h, x.shape[0], _p(x, _f), int(train_type), int(max_beam_size), int(niter)))

    def tables(self):
        """(codebooks [total_K, d], centroid_norms [total_K], codebook_cross_products [flat])"""
        cb = np.empty((self.total_k, self.d), np.float32)
        norms = np.empty(self.total_k, np.float32)
        cross = np.empty(int(lib().ref_rq_cross_size(self.h)), np.float32)
        _ck(lib().ref_rq_tables(self.h, _p(cb, _f), _p(norms, _f), _p(cross, _f)))
        return cb, norms, cross

    def refine_beam(self, residuals, beam_in, out_beam):
        """residuals [n, beam_in, d] -> (codes [n, B, M], residuals [n, B, d], distances [n, B])"""
        r = np.ascontiguousarray(residuals, np.float32)
        n = r.shape[0]
        B = final_beam(self.nbits, beam_in, out_beam)
        codes = np.empty((n, B, self.M), np.int32)
        ro = np.empty((n, B, self.d), np.float32)
        dis = np.empty((n, B), np.float32)
        _ck(lib().ref_rq_refine_beam(self.h, n, beam_in, _p(r, _f), out_beam, _p(codes, _i32), _p(ro, _f), _p(dis, _f)))
        return codes, ro, dis

    def refine_beam_lut(self, x, out_beam):
        """x [n, d] -> (codes [n, B, M], distances [n, B]) on the CPU's own query_norms and query_cp"""
        x = np.ascontiguousarray(x, np.float32)
        n = x.shape[0]
        B = final_beam(self.nbits, 1, out_beam)
        codes = np.empty((n, B, self.M), np.int32)
        dis = np.empty((n, B), np.float32)
        _ck(lib().ref_rq_refine_beam_lut(self.h, n, _p(x, _f), out_beam, _p(codes, _i32), _p(dis, _f)))
        return codes, dis

    def compute_codes(self, x, centroids=None):
        """compute_codes_add_centroids -> packed [n, code_size] uint8"""
        x = np.ascontiguousarray(x, np.float32)
        c = None if centroids is None else np.ascontiguousarray(centroids, np.float32)
        out = np.empty((x.shape[0], self.code_size), np.uint8)
        _ck(lib().ref_rq_compute_codes(self.h, _p(x, _f), x.shape[0], _p(c, _f), _p(out, _u8)))
        return out

    def decode(self, packed):
        packed = np.ascontiguousarray(packed, np.uint8)
        out = np.empty((packed.shape[0], self.d), np.float32)
        _ck(lib().ref_rq_decode(self.h, _p(packed, _u8), packed.shape[0], _p(out, _f)))
        return out


def set_threads(n):
    """the OpenMP thread count of the reference encoder"""
    lib().ref_rq_set_threads(int(n))
