"""TEST INFRASTRUCTURE ONLY -- ctypes wrapper over oracle/_ref/libfaiss_ref.so, the UNMODIFIED
reference CPU library compiled from the reference tree (REF) by oracle/Makefile (+ oracle/ref_shim.cpp),
and the loader (Shim) of the shim libraries oracle/_ref/libfaiss_ref_<name>.so that the ref_<name>.py
modules wrap.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  Nothing under faiss_b200/ does.
"""
import ctypes
import os
import re
import subprocess

import numpy as np

REF = "/root/reference"  # the reference source tree; oracle/_ref is (re)built only where it is present
_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libfaiss_ref.so")

_f = ctypes.POINTER(ctypes.c_float)
_i64 = ctypes.POINTER(ctypes.c_int64)
_u8 = ctypes.POINTER(ctypes.c_uint8)
_i32 = ctypes.POINTER(ctypes.c_int)


def _make(target, verbose):
    """make -k one oracle/Makefile target; on failure, raise naming every file that did not build"""
    if not os.path.isdir(os.path.join(REF, "faiss")):
        return False
    r = subprocess.run(["make", "-k", "-C", _HERE, "-j", str(os.cpu_count() or 4), target], capture_output=True, text=True)
    if verbose:
        print(r.stdout + r.stderr, end="")
    if r.returncode != 0:
        failed = sorted(set(re.findall(r"\*\*\* \[(?:\S+: )?(\S+)\] Error", r.stderr)))
        raise RuntimeError("oracle/_ref: %s failed to build:\n%s" % (", ".join(failed) or target, r.stderr[-3000:]))
    return True


def build(verbose=False):
    """Compile the reference library and every shim library of oracle/Makefile (only where REF is present);
    returns whether the reference library is there."""
    return _make("all", verbose) or available()


def available():
    return os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError("oracle/_ref/libfaiss_ref.so missing: run `make -k -C oracle` where the reference tree is present")
        L = ctypes.CDLL(LIB_PATH)
        L.ref_last_error.restype = ctypes.c_char_p
        L.ref_compile_options.restype = ctypes.c_char_p
        for n in ("ref_flat_new", "ref_ivfflat_new", "ref_ivfpq_new", "ref_shards_new"):
            getattr(L, n).restype = ctypes.c_void_p
        L.ref_index_ntotal.restype = ctypes.c_int64
        L.ref_ivf_nlist.restype = ctypes.c_int64
        L.ref_ivf_list_size.restype = ctypes.c_int64
        L.ref_ivf_code_size.restype = ctypes.c_int64
        _lib = L
    return _lib


def _ck(rc):
    """raise the reference's own message when a call of this library or of any shim library returned non-zero
    (the shims report through libfaiss_ref.so's one error slot, oracle/ref_shim.h)"""
    if rc != 0:
        raise RuntimeError("reference error: " + lib().ref_last_error().decode(errors="replace"))


class Shim:
    """the shim library oracle/_ref/libfaiss_ref_<name>.so (oracle/ref_<name>_shim.cpp) over this library;
    declare(L) sets the restype / argtypes of its entry points once it is loaded"""

    def __init__(self, name, declare=None):
        self.name = name
        self._target = "_ref/libfaiss_ref_%s.so" % name  # relative to oracle/, as oracle/Makefile names it
        self.path = os.path.join(_HERE, self._target)
        self._declare = declare
        self._lib = None
        self._own_error = None

    def build(self, verbose=False):
        """Compile this shim library (and the reference library under it) where REF is present; returns
        whether it is there."""
        return _make(self._target, verbose) or self.available()

    def available(self):
        return available() and os.path.exists(self.path)

    def lib(self):
        if self._lib is None:
            lib()  # the reference library itself, with the generic entry points and the error slot
            if not self.available():
                raise RuntimeError("oracle/%s missing: run `make -k -C oracle` where the reference tree is present" % self._target)
            L = ctypes.CDLL(self.path)
            if self._declare:
                self._declare(L)
            # A shim library built before the shims shared libfaiss_ref.so's error slot keeps its message in its own
            # ref_<name>_last_error.  Such a prebuilt copy is not rebuilt where the reference tree is absent, nor by
            # make when it is newer than the sources, and it computes the same results, so it is read, not refused.
            self._own_error = getattr(L, "ref_%s_last_error" % self.name, None)
            if self._own_error:
                self._own_error.restype = ctypes.c_char_p
            self._lib = L
        return self._lib

    def ck(self, rc):
        """_ck for a call into this library"""
        if rc != 0 and self._own_error:
            raise RuntimeError("reference error: " + self._own_error().decode(errors="replace"))
        _ck(rc)


def _p(a, t):
    return a.ctypes.data_as(t)


def omp_threads():
    return lib().ref_omp_max_threads()


def set_omp_threads(n):
    lib().ref_omp_set_threads(int(n))


def set_blas_threads(n):
    """OpenBLAS (pthreads build) sizes its pool from the visible CPUs; inside a CPU-quota cgroup that
    oversubscribes badly.  Best effort: openblas_set_num_threads through the already-loaded library."""
    lib()
    try:
        for line in open("/proc/self/maps"):
            if "libopenblas" in line:
                path = line.split()[-1]
                L = ctypes.CDLL(path)
                L.openblas_set_num_threads(int(n))
                return True
    except Exception:
        pass
    return False


def compile_options():
    return lib().ref_compile_options().decode()


def float_rand(n, seed):
    x = np.empty(n, dtype=np.float32)
    lib().ref_float_rand(_p(x, _f), ctypes.c_size_t(n), ctypes.c_int64(seed))
    return x


def rand_perm(n, seed):
    x = np.empty(n, dtype=np.int32)
    lib().ref_rand_perm(_p(x, _i32), ctypes.c_size_t(n), ctypes.c_int64(seed))
    return x


class RefIndex:
    def __init__(self, handle):
        self.h = ctypes.c_void_p(handle)
        self._keep = []

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.ref_index_free(self.h)
            self.h = None

    @property
    def ntotal(self):
        return lib().ref_index_ntotal(self.h)

    @property
    def is_trained(self):
        return bool(lib().ref_index_is_trained(self.h))

    def train(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        _ck(lib().ref_index_train(self.h, ctypes.c_int64(x.shape[0]), _p(x, _f)))

    def add(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        _ck(lib().ref_index_add(self.h, ctypes.c_int64(x.shape[0]), _p(x, _f)))

    def add_with_ids(self, x, ids):
        x = np.ascontiguousarray(x, dtype=np.float32)
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        _ck(lib().ref_index_add_with_ids(self.h, ctypes.c_int64(x.shape[0]), _p(x, _f), _p(ids, _i64)))

    def search(self, x, k):
        x = np.ascontiguousarray(x, dtype=np.float32)
        D = np.empty((x.shape[0], k), dtype=np.float32)
        I = np.empty((x.shape[0], k), dtype=np.int64)
        _ck(lib().ref_index_search(self.h, ctypes.c_int64(x.shape[0]), _p(x, _f), ctypes.c_int64(k), _p(D, _f), _p(I, _i64)))
        return D, I

    def assign(self, x, k=1):
        x = np.ascontiguousarray(x, dtype=np.float32)
        I = np.empty((x.shape[0], k), dtype=np.int64)
        _ck(lib().ref_index_assign(self.h, ctypes.c_int64(x.shape[0]), _p(x, _f), _p(I, _i64), ctypes.c_int64(k)))
        return I

    def reset(self):
        _ck(lib().ref_index_reset(self.h))

    def reconstruct_n(self, i0, ni, d):
        out = np.empty((ni, d), dtype=np.float32)
        _ck(lib().ref_index_reconstruct_n(self.h, ctypes.c_int64(i0), ctypes.c_int64(ni), _p(out, _f)))
        return out

    def compute_residual_n(self, x, keys):
        x = np.ascontiguousarray(x, dtype=np.float32)
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        out = np.empty_like(x)
        _ck(lib().ref_index_compute_residual_n(self.h, ctypes.c_int64(x.shape[0]), _p(x, _f), _p(out, _f), _p(keys, _i64)))
        return out


class IndexFlat(RefIndex):
    def __init__(self, d, metric=1):
        super().__init__(lib().ref_flat_new(int(d), int(metric)))
        self.d = d


class _IVF(RefIndex):
    @property
    def nlist(self):
        return lib().ref_ivf_nlist(self.h)

    def set_nprobe(self, v):
        lib().ref_ivf_set_nprobe(self.h, ctypes.c_int64(v))

    def set_cp(self, niter=-1, seed=-1, max_points_per_centroid=-1):
        lib().ref_ivf_set_cp(self.h, int(niter), int(seed), int(max_points_per_centroid))

    def centroids(self):
        out = np.empty((self.nlist, self.d), dtype=np.float32)
        _ck(lib().ref_ivf_get_centroids(self.h, _p(out, _f)))
        return out

    def set_centroids(self, c):
        c = np.ascontiguousarray(c, dtype=np.float32)
        _ck(lib().ref_ivf_set_centroids(self.h, _p(c, _f)))

    def list_size(self, l):
        return lib().ref_ivf_list_size(self.h, ctypes.c_int64(l))

    def code_size(self):
        return lib().ref_ivf_code_size(self.h)

    def get_list(self, l):
        n = self.list_size(l)
        codes = np.empty(n * self.code_size(), dtype=np.uint8)
        ids = np.empty(n, dtype=np.int64)
        _ck(lib().ref_ivf_get_list(self.h, ctypes.c_int64(l), _p(codes, _u8), _p(ids, _i64)))
        return codes, ids

    def add_entries(self, l, ids, codes):
        """InvertedLists::add_entries: append pre-encoded vectors to list l (clone GPU -> CPU)."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        codes = np.ascontiguousarray(codes, dtype=np.uint8).reshape(-1)
        assert codes.size == ids.size * self.code_size()
        _ck(lib().ref_ivf_add_entries(self.h, ctypes.c_int64(l), ctypes.c_int64(ids.size), _p(ids, _i64), _p(codes, _u8)))

    def set_is_trained(self, v=True):
        lib().ref_ivf_set_is_trained(self.h, int(bool(v)))

    def quantizer_search(self, x, k):
        x = np.ascontiguousarray(x, dtype=np.float32)
        D = np.empty((x.shape[0], k), dtype=np.float32)
        I = np.empty((x.shape[0], k), dtype=np.int64)
        _ck(lib().ref_ivf_quantizer_search(self.h, ctypes.c_int64(x.shape[0]), _p(x, _f), ctypes.c_int64(k), _p(D, _f), _p(I, _i64)))
        return D, I

    def search_preassigned(self, x, k, assign, cdis):
        x = np.ascontiguousarray(x, dtype=np.float32)
        assign = np.ascontiguousarray(assign, dtype=np.int64)
        cdis = np.ascontiguousarray(cdis, dtype=np.float32)
        D = np.empty((x.shape[0], k), dtype=np.float32)
        I = np.empty((x.shape[0], k), dtype=np.int64)
        _ck(
            lib().ref_ivf_search_preassigned(
                self.h, ctypes.c_int64(x.shape[0]), _p(x, _f), ctypes.c_int64(k), _p(assign, _i64), _p(cdis, _f), _p(D, _f), _p(I, _i64)
            )
        )
        return D, I


class IndexIVFFlat(_IVF):
    def __init__(self, d, nlist, metric=1):
        super().__init__(lib().ref_ivfflat_new(int(d), ctypes.c_int64(nlist), int(metric)))
        self.d = d


class IndexIVFPQ(_IVF):
    def __init__(self, d, nlist, M, nbits=8, metric=1):
        super().__init__(lib().ref_ivfpq_new(int(d), ctypes.c_int64(nlist), int(M), int(nbits), int(metric)))
        self.d, self.M = d, M

    @property
    def use_precomputed_table(self):
        return lib().ref_ivfpq_use_precomputed_table(self.h)

    def set_precomputed_table(self, v):
        _ck(lib().ref_ivfpq_set_precomputed_table(self.h, int(v)))

    def pq_centroids(self):
        out = np.empty((self.M, 256, self.d // self.M), dtype=np.float32)
        _ck(lib().ref_ivfpq_get_pq_centroids(self.h, _p(out, _f)))
        return out

    def set_pq_centroids(self, c):
        c = np.ascontiguousarray(c, dtype=np.float32)
        _ck(lib().ref_ivfpq_set_pq_centroids(self.h, _p(c, _f)))

    def set_pq_cp(self, niter=-1, seed=-1):
        lib().ref_ivfpq_set_pq_niter(self.h, int(niter), int(seed))

    def pq_compute_codes(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        codes = np.empty((x.shape[0], self.M), dtype=np.uint8)
        _ck(lib().ref_pq_compute_codes(self.h, _p(x, _f), _p(codes, _u8), ctypes.c_int64(x.shape[0])))
        return codes


class IndexShards(RefIndex):
    def __init__(self, d, threaded=False, successive_ids=True):
        super().__init__(lib().ref_shards_new(int(d), int(threaded), int(successive_ids)))
        self.d = d

    def add_shard(self, idx):
        self._keep.append(idx)
        _ck(lib().ref_shards_add_shard(self.h, idx.h))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.ref_index_free(self.h)
            self.h = None
        self._keep = []


def kmeans(x, k, niter=25, seed=1234, max_points_per_centroid=256, min_points_per_centroid=39):
    x = np.ascontiguousarray(x, dtype=np.float32)
    n, d = x.shape
    cent = np.empty((k, d), dtype=np.float32)
    obj = np.zeros(niter, dtype=np.float32)
    nsplit = np.zeros(niter, dtype=np.int64)
    _ck(
        lib().ref_kmeans(
            int(d), ctypes.c_int64(n), ctypes.c_int64(k), _p(x, _f), int(niter), int(seed), int(max_points_per_centroid),
            int(min_points_per_centroid), _p(cent, _f), _p(obj, _f), _p(nsplit, _i64),
        )
    )
    return cent, obj, nsplit


def pq_train(x, M, nbits=8, niter=25, seed=1234):
    """faiss::ProductQuantizer::train on x [n, d]; returns centroids [M, 2^nbits, d/M]."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    n, d = x.shape
    out = np.empty((M, 1 << nbits, d // M), dtype=np.float32)
    _ck(lib().ref_pq_train(int(d), int(M), int(nbits), ctypes.c_int64(n), _p(x, _f), int(niter), int(seed), _p(out, _f)))
    return out


def kmeans_spherical_ip(x, k, niter=10, seed=1234):
    """faiss::Clustering with spherical=True over an IndexFlatIP (what GpuIndexIVF uses for METRIC_INNER_PRODUCT)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    n, d = x.shape
    cent = np.empty((k, d), dtype=np.float32)
    obj = np.zeros(niter, dtype=np.float32)
    _ck(lib().ref_kmeans_spherical_ip(int(d), ctypes.c_int64(n), ctypes.c_int64(k), _p(x, _f), int(niter), int(seed), _p(cent, _f), _p(obj, _f)))
    return cent, obj


def merge_knn_results(all_D, all_I, metric=1):
    """all_D/all_I: [nshard, n, k] -> [n, k]"""
    all_D = np.ascontiguousarray(all_D, dtype=np.float32)
    all_I = np.ascontiguousarray(all_I, dtype=np.int64)
    ns, n, k = all_D.shape
    D = np.empty((n, k), dtype=np.float32)
    I = np.empty((n, k), dtype=np.int64)
    _ck(lib().ref_merge_knn_results(ctypes.c_int64(n), ctypes.c_int64(k), int(ns), int(metric), _p(all_D, _f), _p(all_I, _i64), _p(D, _f), _p(I, _i64)))
    return D, I


def knn(xq, xb, k, metric=1):
    xq = np.ascontiguousarray(xq, dtype=np.float32)
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    D = np.empty((xq.shape[0], k), dtype=np.float32)
    I = np.empty((xq.shape[0], k), dtype=np.int64)
    _ck(
        lib().ref_knn(
            int(metric), _p(xq, _f), _p(xb, _f), ctypes.c_int64(xq.shape[1]), ctypes.c_int64(xq.shape[0]),
            ctypes.c_int64(xb.shape[0]), ctypes.c_int64(k), _p(D, _f), _p(I, _i64),
        )
    )
    return D, I
