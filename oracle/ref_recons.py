"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's IndexIVF retrieval calls (search_and_reconstruct,
search_and_return_codes, a direct map + reconstruct): oracle/_ref/libfaiss_ref_recons.so (oracle/ref_recons_shim.cpp,
built by oracle/Makefile) over the UNMODIFIED reference CPU library of oracle/ref.py.  The functions take the IVF
handles of oracle.ref / oracle.ref_sq.

Only tests/, tests/golden/ and bench_reconstruct.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes

import numpy as np

from oracle import ref

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)
_u8 = ctypes.POINTER(ctypes.c_uint8)


def _declare(L):
    L.ref_ivf_coarse_code_size.restype = ctypes.c_int64
    L.ref_ivf_coarse_code_size.argtypes = [ctypes.c_void_p]


_shim = ref.Shim("recons", _declare)
LIB_PATH, build, available, lib, _ck = _shim.path, _shim.build, _shim.available, _shim.lib, _shim.ck


def _x(x):
    return np.ascontiguousarray(x, dtype=np.float32)


def search_and_reconstruct(idx, x, k, nprobe):
    """IndexIVF::search_and_reconstruct -> D [n, k], I [n, k], R [n, k, d]"""
    x = _x(x)
    n, d = x.shape
    D = np.empty((n, k), np.float32)
    I = np.empty((n, k), np.int64)
    R = np.empty((n, k, d), np.float32)
    _ck(lib().ref_ivf_search_and_reconstruct(idx.h, ctypes.c_int64(n), x.ctypes.data_as(_f), ctypes.c_int64(k),
                                             ctypes.c_int64(nprobe), D.ctypes.data_as(_f), I.ctypes.data_as(_i64),
                                             R.ctypes.data_as(_f)))
    return D, I, R


def search_and_return_codes(idx, x, k, nprobe, include_listno=False):
    """IndexIVF::search_and_return_codes -> D, I, codes [n, k, (coarse_code_size if include_listno) + code_size]"""
    x = _x(x)
    n = x.shape[0]
    width = idx.code_size() + (coarse_code_size(idx) if include_listno else 0)
    D = np.empty((n, k), np.float32)
    I = np.empty((n, k), np.int64)
    C = np.empty((n, k, width), np.uint8)
    _ck(lib().ref_ivf_search_and_return_codes(idx.h, ctypes.c_int64(n), x.ctypes.data_as(_f), ctypes.c_int64(k),
                                              ctypes.c_int64(nprobe), D.ctypes.data_as(_f), I.ctypes.data_as(_i64),
                                              C.ctypes.data_as(_u8), int(bool(include_listno))))
    return D, I, C


def coarse_code_size(idx):
    return int(lib().ref_ivf_coarse_code_size(idx.h))


def reconstruct(idx, keys, d):
    """a hash-table direct map + IndexIVF::reconstruct per key (ids must be unique) -> [n, d]"""
    keys = np.ascontiguousarray(keys, dtype=np.int64).reshape(-1)
    out = np.empty((keys.size, d), np.float32)
    _ck(lib().ref_ivf_reconstruct_keys(idx.h, ctypes.c_int64(keys.size), keys.ctypes.data_as(_i64), out.ctypes.data_as(_f)))
    return out
