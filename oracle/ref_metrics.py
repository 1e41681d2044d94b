"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's extra metrics: oracle/_ref/libfaiss_ref_metrics.so
(oracle/ref_metrics_shim.cpp, built by oracle/Makefile) over the UNMODIFIED reference CPU library of
oracle/ref.py.  IndexFlat handles are reference faiss::IndexFlat objects, so every generic Index call of
oracle.ref applies to them.

Only tests/, tests/golden/ and bench_metrics.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes

import numpy as np

from oracle import ref

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)


def _declare(L):
    L.ref_flat_new_ex.restype = ctypes.c_void_p
    L.ref_flat_new_ex.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float]


_shim = ref.Shim("metrics", _declare)
LIB_PATH, build, available, lib, _ck = _shim.path, _shim.build, _shim.available, _shim.lib, _shim.ck


class IndexFlat(ref.RefIndex):
    """faiss::IndexFlat(d, metric) with metric_arg (the exponent of METRIC_Lp)."""

    def __init__(self, d, metric=1, metric_arg=0.0):
        h = lib().ref_flat_new_ex(int(d), int(metric), float(metric_arg))
        if not h:
            _ck(-1)
        super().__init__(h)
        self.d = d


def knn_extra_metrics(xq, xb, k, metric, metric_arg=0.0):
    """faiss::knn_extra_metrics (faiss/utils/extra_distances.cpp:93-137): (D [nq, k], I [nq, k])"""
    xq = np.ascontiguousarray(xq, dtype=np.float32)
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    nq, d = xq.shape
    D = np.empty((nq, k), dtype=np.float32)
    I = np.empty((nq, k), dtype=np.int64)
    _ck(lib().ref_knn_extra_metrics(
        xq.ctypes.data_as(_f), xb.ctypes.data_as(_f), ctypes.c_int64(d), ctypes.c_int64(nq), ctypes.c_int64(xb.shape[0]),
        int(metric), ctypes.c_float(metric_arg), ctypes.c_int64(k), D.ctypes.data_as(_f), I.ctypes.data_as(_i64),
    ))
    return D, I
