"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper of the reference's CPU all-pairs distances:
oracle/_ref/libfaiss_ref_pairwise.so (oracle/ref_pairwise_shim.cpp, built by oracle/Makefile) over the UNMODIFIED
reference CPU library of oracle/ref.py.

Only tests/ and tests/golden/ import this module.  Nothing under faiss_b200/ does.
"""
import ctypes

import numpy as np

from oracle import ref

_f = ctypes.POINTER(ctypes.c_float)
METRIC_L2 = 1


_shim = ref.Shim("pairwise")
LIB_PATH, build, available, lib, _ck = _shim.path, _shim.build, _shim.available, _shim.lib, _shim.ck


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
        _ck(lib().ref_pairwise_L2sqr(*args, dis.ctypes.data_as(_f)))
    else:
        _ck(lib().ref_pairwise_extra_distances(*args, int(metric), ctypes.c_float(metric_arg), dis.ctypes.data_as(_f)))
    return dis
