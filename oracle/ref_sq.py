"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's IndexIVFScalarQuantizer:
oracle/_ref/libfaiss_ref_sq.so (oracle/ref_sq_shim.cpp, built by oracle/Makefile) over the UNMODIFIED
reference CPU library of oracle/ref.py.  The handles are reference IndexIVF objects, so every generic
Index / IVF call of oracle.ref applies to them.

Only tests/ and tests/golden/ import this module.  Nothing under faiss_b200/ does.
"""
import ctypes

import numpy as np

from oracle import ref

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)
_u8 = ctypes.POINTER(ctypes.c_uint8)

# faiss::ScalarQuantizer::QuantizerType (faiss/impl/ScalarQuantizer.h:27-34)
QT_8bit, QT_4bit, QT_8bit_uniform, QT_4bit_uniform, QT_fp16, QT_8bit_direct, QT_6bit = range(7)
QT_NAMES = ["8bit", "4bit", "8bit_uniform", "4bit_uniform", "fp16", "8bit_direct", "6bit"]


def _declare(L):
    L.ref_ivfsq_new.restype = ctypes.c_void_p
    L.ref_ivfsq_trained_size.restype = ctypes.c_int64
    L.ref_ivfsq_code_size.restype = ctypes.c_int64


_shim = ref.Shim("sq", _declare)
LIB_PATH, build, available, lib, _ck = _shim.path, _shim.build, _shim.available, _shim.lib, _shim.ck


class IndexIVFScalarQuantizer(ref._IVF):
    """faiss::IndexIVFScalarQuantizer (faiss/IndexScalarQuantizer.h) over an IndexFlat coarse quantizer."""

    def __init__(self, d, nlist, qtype, metric=1, by_residual=True):
        h = lib().ref_ivfsq_new(int(d), ctypes.c_int64(nlist), int(qtype), int(metric), int(bool(by_residual)))
        if not h:
            _ck(-1)
        super().__init__(h)
        self.d, self.qtype, self.by_residual = d, int(qtype), bool(by_residual)

    def trained(self):
        n = lib().ref_ivfsq_trained_size(self.h)
        out = np.empty(n, dtype=np.float32)
        _ck(lib().ref_ivfsq_get_trained(self.h, out.ctypes.data_as(_f)))
        return out

    def set_trained(self, t):
        t = np.ascontiguousarray(t, dtype=np.float32).reshape(-1)
        _ck(lib().ref_ivfsq_set_trained(self.h, t.ctypes.data_as(_f), ctypes.c_int64(t.size)))

    def sq_code_size(self):
        return lib().ref_ivfsq_code_size(self.h)

    def set_rangestat(self, rangestat, arg=0.0):
        _ck(lib().ref_ivfsq_set_rangestat(self.h, int(rangestat), ctypes.c_float(arg)))

    def encode(self, x, list_nos):
        """encode_vectors(n, x, list_nos, codes): residuals against list_nos when by_residual; rows whose
        list number is < 0 stay zero"""
        x = np.ascontiguousarray(x, dtype=np.float32)
        list_nos = np.ascontiguousarray(list_nos, dtype=np.int64).reshape(-1)
        codes = np.zeros((x.shape[0], self.sq_code_size()), dtype=np.uint8)
        _ck(lib().ref_ivfsq_encode(self.h, ctypes.c_int64(x.shape[0]), x.ctypes.data_as(_f), list_nos.ctypes.data_as(_i64),
                                   codes.ctypes.data_as(_u8)))
        return codes
