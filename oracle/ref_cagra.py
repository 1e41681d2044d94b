"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's IndexHNSWCagra: oracle/_ref/libfaiss_ref_cagra.so
(oracle/ref_cagra_shim.cpp, built by oracle/cagra.mk) over the UNMODIFIED reference CPU library of oracle/ref.py.

Only tests/ and bench_cagra.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref_cagra.so")

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)


def build(verbose=False):
    """Compile oracle/_ref/libfaiss_ref_cagra.so (only where the reference sources are mounted)."""
    if not os.path.isdir("/root/reference/faiss") or not ref.available():
        return available()
    r = subprocess.run(["make", "-C", _HERE, "-f", "cagra.mk"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref CAGRA shim build failed:\n" + (r.stdout or "")[-3000:] + (r.stderr or "")[-3000:])
    return True


def available():
    return ref.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        ref.lib()
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref_cagra.so missing: run `make -C oracle -f cagra.mk`")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_cagra_last_error.restype = ctypes.c_char_p
        _lib = L
    return _lib


def _ck(rc):
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_cagra_last_error().decode(errors="replace"))


def search_graph(xb, graph, metric, xq, k, ef_search=16, base_level_only=False):
    """IndexHNSWCagra made from (xb, graph) as GpuIndexCagra::copyTo does, searched with efSearch -> D, I"""
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    xq = np.ascontiguousarray(xq, dtype=np.float32)
    graph = np.ascontiguousarray(graph, dtype=np.int64)
    n, d = xb.shape
    nq = xq.shape[0]
    D = np.empty((nq, k), np.float32)
    I = np.empty((nq, k), np.int64)
    _ck(lib().ref_cagra_search_graph(
        int(d), int(metric), ctypes.c_int64(n), xb.ctypes.data_as(_f), graph.ctypes.data_as(_i64), int(graph.shape[1]),
        int(bool(base_level_only)), ctypes.c_int64(nq), xq.ctypes.data_as(_f), ctypes.c_int64(k), int(ef_search),
        D.ctypes.data_as(_f), I.ctypes.data_as(_i64)))
    return D, I


def build_cpu_graph(xb, metric, M=32):
    """IndexHNSWCagra(d, M).add(xb) on the CPU -> its level-0 table [n, 2M] int64 (-1 padded)"""
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    n, d = xb.shape
    graph = np.empty((n, 2 * M), np.int64)
    _ck(lib().ref_cagra_build_cpu(int(d), int(metric), int(M), ctypes.c_int64(n), xb.ctypes.data_as(_f),
                                  graph.ctypes.data_as(_i64)))
    return graph
