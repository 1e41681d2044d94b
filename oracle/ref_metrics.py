"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's extra metrics: oracle/_ref/libfaiss_ref_metrics.so
(oracle/ref_metrics_shim.cpp, built by oracle/metrics.mk) over the UNMODIFIED reference CPU library of
oracle/ref.py.  IndexFlat handles are reference faiss::IndexFlat objects, so every generic Index call of
oracle.ref applies to them.

Only tests/, tests/golden/ and bench_metrics.py import this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref_metrics.so")

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)


def build(verbose=False):
    """Compile oracle/_ref/libfaiss_ref_metrics.so (only where the reference sources are mounted)."""
    if not os.path.isdir("/root/reference/faiss") or not ref.available():
        return available()
    r = subprocess.run(["make", "-C", _HERE, "-f", "metrics.mk"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref metrics shim build failed:\n" + (r.stdout or "")[-3000:] + (r.stderr or "")[-3000:])
    return True


def available():
    return ref.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        ref.lib()  # the reference library itself, with the generic entry points
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref_metrics.so missing: run `make -C oracle -f metrics.mk`")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_metrics_last_error.restype = ctypes.c_char_p
        L.ref_flat_new_ex.restype = ctypes.c_void_p
        L.ref_flat_new_ex.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float]
        _lib = L
    return _lib


class IndexFlat(ref.RefIndex):
    """faiss::IndexFlat(d, metric) with metric_arg (the exponent of METRIC_Lp)."""

    def __init__(self, d, metric=1, metric_arg=0.0):
        h = lib().ref_flat_new_ex(int(d), int(metric), float(metric_arg))
        if not h:
            raise RuntimeError("reference error: " + lib().ref_metrics_last_error().decode(errors="replace"))
        super().__init__(h)
        self.d = d


def knn_extra_metrics(xq, xb, k, metric, metric_arg=0.0):
    """faiss::knn_extra_metrics (faiss/utils/extra_distances.cpp:93-137): (D [nq, k], I [nq, k])"""
    xq = np.ascontiguousarray(xq, dtype=np.float32)
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    nq, d = xq.shape
    D = np.empty((nq, k), dtype=np.float32)
    I = np.empty((nq, k), dtype=np.int64)
    rc = lib().ref_knn_extra_metrics(
        xq.ctypes.data_as(_f), xb.ctypes.data_as(_f), ctypes.c_int64(d), ctypes.c_int64(nq), ctypes.c_int64(xb.shape[0]),
        int(metric), ctypes.c_float(metric_arg), ctypes.c_int64(k), D.ctypes.data_as(_f), I.ctypes.data_as(_i64),
    )
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_metrics_last_error().decode(errors="replace"))
    return D, I
