"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's CPU all-pairs distances:
oracle/_ref/libfaiss_ref_pairwise.so (oracle/ref_pairwise_shim.cpp, built by oracle/pairwise.mk) over the UNMODIFIED
reference CPU library of oracle/ref.py.

Only tests/ and tests/golden/ import this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref_pairwise.so")

_f = ctypes.POINTER(ctypes.c_float)
METRIC_L2 = 1


def build(verbose=False):
    """Compile oracle/_ref/libfaiss_ref_pairwise.so (only where the reference sources are mounted)."""
    if not os.path.isdir("/root/reference/faiss") or not ref.available():
        return available()
    r = subprocess.run(["make", "-C", _HERE, "-f", "pairwise.mk"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref pairwise shim build failed:\n" + (r.stdout or "")[-3000:] + (r.stderr or "")[-3000:])
    return True


def available():
    return ref.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        ref.lib()  # the reference library itself
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref_pairwise.so missing: run `make -C oracle -f pairwise.mk`")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_pairwise_last_error.restype = ctypes.c_char_p
        _lib = L
    return _lib


def pairwise(xq, xb, metric, metric_arg=0.0):
    """[nq, nb] float32: faiss::pairwise_L2sqr for L2 (faiss/utils/distances.h:116-125), else
    faiss::pairwise_extra_distances (faiss/utils/extra_distances.h:25-37), inner product included"""
    xq = np.ascontiguousarray(xq, dtype=np.float32)
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    nq, d = xq.shape
    nb = xb.shape[0]
    dis = np.empty((nq, nb), dtype=np.float32)
    args = (ctypes.c_int64(d), ctypes.c_int64(nq), xq.ctypes.data_as(_f), ctypes.c_int64(nb), xb.ctypes.data_as(_f))
    if metric == METRIC_L2:
        rc = lib().ref_pairwise_L2sqr(*args, dis.ctypes.data_as(_f))
    else:
        rc = lib().ref_pairwise_extra_distances(*args, int(metric), ctypes.c_float(metric_arg), dis.ctypes.data_as(_f))
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_pairwise_last_error().decode(errors="replace"))
    return dis
