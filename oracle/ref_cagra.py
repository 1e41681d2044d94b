"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's IndexHNSWCagra: oracle/_ref/libfaiss_ref_cagra.so
(oracle/ref_cagra_shim.cpp, built by oracle/Makefile) over the UNMODIFIED reference CPU library of oracle/ref.py.

Only tests/ and bench_cagra.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes

import numpy as np

from oracle import ref

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)


_shim = ref.Shim("cagra")
LIB_PATH, build, available, lib, _ck = _shim.path, _shim.build, _shim.available, _shim.lib, _shim.ck


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
