"""faiss_b200_bfKnn_params / faiss_b200_bfKnn_tiling argument validation (no GPU): every invalid argument is refused
with -2 and a message before any CUDA call, and the Python FaissGpuDistanceParams has the C struct's layout."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import faiss_b200 as fb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def res():
    return fb.StandardGpuResources()


X = np.zeros((64, 8), dtype=np.float32)
X16 = np.zeros((64, 8), dtype=np.float16)
DOUT = np.zeros((64, 64 * 64), dtype=np.float32)
IOUT = np.zeros((64, 4096), dtype=np.int64)


def params(**kw):
    p = fb.GpuDistanceParams(
        fb.METRIC_L2, 0.0, 4, 8, X.ctypes.data, fb.DistanceDataType_F32, 1, 64, X.ctypes.data, fb.DistanceDataType_F32, 1,
        64, DOUT.ctypes.data, fb.IndicesDataType_I64, IOUT.ctypes.data, 0,
    )
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def refused(code, match):
    assert code == -2, code
    msg = fb.lib.faiss_get_last_error().decode()
    assert match in msg, msg


@pytest.mark.parametrize(
    "kw,match",
    [
        (dict(k=0), "k must be -1"),
        (dict(k=-2), "k must be -1"),
        (dict(k=2049), "k must be -1"),
        (dict(vectors=X16.ctypes.data, vectorType=fb.DistanceDataType_F16), "vectorType and queryType must be the same"),
        (dict(queryType=fb.DistanceDataType_BF16), "vectorType and queryType must be the same"),
        (dict(vectorType=7, queryType=7), "unknown vectorType"),
        (dict(outIndicesType=3), "unknown outIndicesType"),
        (dict(outIndicesType=fb.IndicesDataType_I32, numVectors=2**31), "INT32_MAX"),
        (dict(dims=0), "dims must be > 0"),
        (dict(vectors=None), "vectors must be provided"),
        (dict(outIndices=None), "outIndices must be provided"),
        (dict(metric=fb.METRIC_NaNEuclidean), "unimplemented metric type 24"),
        (dict(device=-1), "device ordinal"),
    ],
)
def test_params_refused(res, kw, match):
    refused(fb.lib.faiss_b200_bfKnn_params(res._h, ctypes.byref(params(**kw))), match)
    refused(fb.lib.faiss_b200_bfKnn_tiling(res._h, ctypes.byref(params(**kw)), ctypes.c_size_t(0), ctypes.c_size_t(0)), match)


@pytest.mark.parametrize(
    "kw,vlim,qlim,match",
    [
        (dict(vectorsRowMajor=0), 1024, 0, "only supported in row major mode"),
        (dict(queriesRowMajor=0), 0, 4096, "only supported in row major mode"),
        (dict(k=-1), 1024, 0, "only supported for k > 0"),
        (dict(k=-1), 0, 4096, "only supported for k > 0"),
        (dict(), 31, 0, "vectorsMemoryLimit is too low"),
        (dict(), 0, 4 * 12 + 8 * 4 - 1, "queriesMemoryLimit is too low"),
        (dict(numVectors=0), 1024, 0, "numVectors must be > 0"),
        (dict(numQueries=0), 0, 4096, "numQueries must be > 0"),
    ],
)
def test_tiling_refused(res, kw, vlim, qlim, match):
    refused(fb.lib.faiss_b200_bfKnn_tiling(res._h, ctypes.byref(params(**kw)), ctypes.c_size_t(vlim), ctypes.c_size_t(qlim)), match)


def test_null_params_and_resources(res):
    assert fb.lib.faiss_b200_bfKnn_params(res._h, None) == -2
    assert fb.lib.faiss_b200_bfKnn_params(None, ctypes.byref(params())) == -2
    refused(fb.lib.b200_pairwise_paged(res._h, ctypes.byref(params(k=0)), ctypes.c_size_t(4096)), "k must be -1")


PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "faiss_b200_c.h"
#define F(name) printf("%s %zu\n", #name, offsetof(FaissGpuDistanceParams, name));
int main(void) {
    printf("sizeof %zu\n", sizeof(FaissGpuDistanceParams));
    F(metric) F(metricArg) F(k) F(dims) F(vectors) F(vectorType) F(vectorsRowMajor) F(numVectors) F(queries)
    F(queryType) F(queriesRowMajor) F(numQueries) F(outDistances) F(outIndicesType) F(outIndices) F(device)
    return 0;
}
"""


def test_struct_layout_matches_header(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text(PROBE)
    exe = tmp_path / "probe"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = dict(line.split() for line in out if line.strip())
    assert int(got.pop("sizeof")) == ctypes.sizeof(fb.GpuDistanceParams)
    assert list(got) == [name for name, _ in fb.GpuDistanceParams._fields_]
    for name, off in got.items():
        assert int(off) == getattr(fb.GpuDistanceParams, name).offset, name


def test_wrong_output_shapes_refused(res):
    """a given D / I is written through its raw pointer: one of the wrong shape is refused before the library call"""
    xq = np.zeros((5, 8), dtype=np.float32)
    xb = np.zeros((20, 8), dtype=np.float32)
    for D in (np.empty((5, 3), np.float32), np.empty((4, 4), np.float32), np.empty(20, np.float32)):
        with pytest.raises(ValueError, match="D must have shape"):
            fb.knn_gpu(res, xq, xb, 4, D=D)
    for I in (np.empty((5, 3), np.int64), np.empty((5, 5), np.int32), np.empty(20, np.int64)):
        with pytest.raises(ValueError, match="I must have shape"):
            fb.knn_gpu(res, xq, xb, 4, I=I)
    for D in (np.empty((5, 19), np.float32), np.empty((5, 4), np.float32), np.empty((6, 20), np.float32)):
        with pytest.raises(ValueError, match="D must have shape"):
            fb.pairwise_distance_gpu(res, xq, xb, D=D)
