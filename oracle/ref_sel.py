"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's IDSelectors and of a search with
SearchParameters::sel: oracle/_ref/libfaiss_ref_sel.so (oracle/ref_sel_shim.cpp, built by oracle/sel.mk) over the
UNMODIFIED reference CPU library of oracle/ref.py.  Selectors are given as the tuples of oracle/oracle_sel_np.py.

Only tests/, tests/golden/ and bench_filter.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref_sel.so")

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)
_u8 = ctypes.POINTER(ctypes.c_uint8)


def build(verbose=False):
    """Compile oracle/_ref/libfaiss_ref_sel.so (only where the reference sources are mounted)."""
    if not os.path.isdir("/root/reference/faiss") or not ref.available():
        return available()
    r = subprocess.run(["make", "-C", _HERE, "-f", "sel.mk"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref selector shim build failed:\n" + (r.stdout or "")[-3000:] + (r.stderr or "")[-3000:])
    return True


def available():
    return ref.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        ref.lib()
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref_sel.so missing: run `make -C oracle -f sel.mk`")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_sel_last_error.restype = ctypes.c_char_p
        for name in ("ref_sel_range", "ref_sel_array", "ref_sel_batch", "ref_sel_bitmap", "ref_sel_not", "ref_sel_binary"):
            getattr(L, name).restype = ctypes.c_void_p
        L.ref_sel_range.argtypes = [ctypes.c_int64, ctypes.c_int64]
        L.ref_sel_array.argtypes = [ctypes.c_int64, _i64]
        L.ref_sel_batch.argtypes = [ctypes.c_int64, _i64]
        L.ref_sel_bitmap.argtypes = [ctypes.c_int64, _u8]
        L.ref_sel_not.argtypes = [ctypes.c_void_p]
        L.ref_sel_binary.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.ref_sel_free.argtypes = [ctypes.c_void_p]
        L.ref_sel_free.restype = None
        L.ref_sel_is_member.argtypes = [ctypes.c_void_p, ctypes.c_int64]
        L.ref_search_sel.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, _f, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, _f, _i64]
        _lib = L
    return _lib


class Selector:
    """a reference faiss::IDSelector tree built from an oracle_sel_np tuple (keeps its arrays and children alive)"""

    def __init__(self, spec):
        L = lib()
        self._keep = []
        kind = spec[0]
        if kind == "range":
            self.h = L.ref_sel_range(int(spec[1]), int(spec[2]))
        elif kind in ("array", "batch"):
            ids = np.ascontiguousarray(np.asarray(spec[1], dtype=np.int64).reshape(-1))
            self._keep.append(ids)
            fn = L.ref_sel_array if kind == "array" else L.ref_sel_batch
            self.h = fn(ids.size, ids.ctypes.data_as(_i64))
        elif kind == "bitmap":
            bm = np.ascontiguousarray(np.asarray(spec[1], dtype=np.uint8).reshape(-1))
            self._keep.append(bm)
            self.h = L.ref_sel_bitmap(bm.size, bm.ctypes.data_as(_u8))
        elif kind == "not":
            c = Selector(spec[1])
            self._keep.append(c)
            self.h = L.ref_sel_not(c.h)
        else:
            a, b = Selector(spec[1]), Selector(spec[2])
            self._keep += [a, b]
            self.h = L.ref_sel_binary({"and": 0, "or": 1, "xor": 2}[kind], a.h, b.h)

    def is_member(self, ids):
        return np.array([bool(lib().ref_sel_is_member(self.h, int(i))) for i in np.asarray(ids).reshape(-1)])

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.ref_sel_free(self.h)
            self.h = None


def search(index, xq, k, spec, nprobe=0):
    """index.search(xq, k, params) with params->sel = the reference selector of spec; nprobe > 0 passes a
    SearchParametersIVF.  index: a RefIndex of oracle.ref / ref_pq / ref_sq."""
    xq = np.ascontiguousarray(xq, dtype=np.float32)
    sel = Selector(spec)
    D = np.empty((xq.shape[0], k), dtype=np.float32)
    I = np.empty((xq.shape[0], k), dtype=np.int64)
    rc = lib().ref_search_sel(
        index.h if isinstance(index.h, ctypes.c_void_p) else ctypes.c_void_p(index.h), xq.shape[0], xq.ctypes.data_as(_f), k, ctypes.c_void_p(sel.h), int(nprobe),
        D.ctypes.data_as(_f), I.ctypes.data_as(_i64))
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_sel_last_error().decode(errors="replace"))
    return D, I
