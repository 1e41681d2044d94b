"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's IndexIVF retrieval calls (search_and_reconstruct,
search_and_return_codes, a direct map + reconstruct): oracle/_ref/libfaiss_ref_recons.so (oracle/ref_recons_shim.cpp,
built by oracle/recons.mk) over the UNMODIFIED reference CPU library of oracle/ref.py.  The functions take the IVF
handles of oracle.ref / oracle.ref_sq.

Only tests/, tests/golden/ and bench_reconstruct.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref_recons.so")

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)
_u8 = ctypes.POINTER(ctypes.c_uint8)


def build(verbose=False):
    """Compile oracle/_ref/libfaiss_ref_recons.so (only where the reference sources are mounted)."""
    if not os.path.isdir("/root/reference/faiss") or not ref.available():
        return available()
    r = subprocess.run(["make", "-C", _HERE, "-f", "recons.mk"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref retrieval shim build failed:\n" + (r.stdout or "")[-3000:] + (r.stderr or "")[-3000:])
    return True


def available():
    return ref.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        ref.lib()
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref_recons.so missing: run `make -C oracle -f recons.mk`")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_recons_last_error.restype = ctypes.c_char_p
        L.ref_ivf_coarse_code_size.restype = ctypes.c_int64
        L.ref_ivf_coarse_code_size.argtypes = [ctypes.c_void_p]
        _lib = L
    return _lib


def _ck(rc):
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_recons_last_error().decode(errors="replace"))


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
