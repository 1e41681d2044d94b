"""faiss_b200 -- H100-native (sm_90a) similarity search behind the Faiss GPU plugin surface.

Python mirror of the reference's index classes over the C ABI of ``libfaiss_b200.so``
(``include/faiss_b200_c.h``).  Same class / method names and argument meaning as
``faiss.GpuIndexFlat{,L2,IP}``, ``faiss.GpuIndexIVFFlat``, ``faiss.GpuIndexIVFPQ``,
``faiss.StandardGpuResources``, ``faiss.IndexShards`` (faiss/python/gpu_wrappers.py:21-60,
faiss/gpu/GpuIndex*.h).  Inputs may be numpy arrays (host) or torch CUDA tensors (device);
outputs follow the input's residency.

There is no CPU fallback: importing this package without the compiled CUDA library fails.
"""
import ctypes
import json
import os

import numpy as np

from ._lib import lib, check, FaissError  # noqa: F401  (loading fails loudly)

# faiss::MetricType (faiss/MetricType.h:29-49).  Every index takes L2 and inner product; GpuIndexFlat and
# bfKnn / knn_gpu also take the others (METRIC_Lp's exponent is Index.metric_arg / bfKnn's metric_arg).
# METRIC_NaNEuclidean is not implemented.
METRIC_INNER_PRODUCT = 0
METRIC_L2 = 1
METRIC_L1 = 2
METRIC_Linf = 3
METRIC_Lp = 4
METRIC_Canberra = 20
METRIC_BrayCurtis = 21
METRIC_JensenShannon = 22
METRIC_Jaccard = 23
METRIC_NaNEuclidean = 24
METRIC_GOWER = 25

# faiss::ScalarQuantizer::QuantizerType (faiss/impl/ScalarQuantizer.h:27-40); GpuIndexIVFScalarQuantizer
# accepts QT_8bit ... QT_6bit, as the reference GPU index does
QT_8bit = 0
QT_4bit = 1
QT_8bit_uniform = 2
QT_4bit_uniform = 3
QT_fp16 = 4
QT_8bit_direct = 5
QT_6bit = 6
QT_bf16 = 7
# faiss::ScalarQuantizer::RangeStat (faiss/impl/ScalarQuantizer.h:66-71)
RS_minmax = 0
RS_meanstd = 1
RS_quantiles = 2
RS_optim = 3

_c_f = ctypes.POINTER(ctypes.c_float)
_c_i64 = ctypes.POINTER(ctypes.c_int64)
_c_u8 = ctypes.POINTER(ctypes.c_uint8)


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _ptr(x, ctype):
    """Raw pointer of a numpy array or torch tensor (host or device)."""
    if x is None:
        return ctypes.cast(None, ctype)
    if _is_torch(x):
        assert x.is_contiguous(), "tensor must be contiguous"
        return ctypes.cast(x.data_ptr(), ctype)
    assert x.flags["C_CONTIGUOUS"], "array must be C-contiguous"
    return x.ctypes.data_as(ctype)


def _as_f32(x):
    if _is_torch(x):
        import torch

        assert x.dtype == torch.float32
        return x.contiguous()
    return np.ascontiguousarray(x, dtype=np.float32)


def _as_i64(x):
    if x is None:
        return None
    if _is_torch(x):
        import torch

        assert x.dtype == torch.int64
        return x.contiguous()
    return np.ascontiguousarray(x, dtype=np.int64)


def _empty_like_residency(x, shape, dtype):
    if _is_torch(x) and x.is_cuda:
        import torch

        tdt = {np.float32: torch.float32, np.int64: torch.int64, np.uint8: torch.uint8, np.int32: torch.int32}[dtype]
        return torch.empty(shape, dtype=tdt, device=x.device)
    return np.empty(shape, dtype=dtype)


class StandardGpuResources:
    """faiss::gpu::StandardGpuResources (faiss/gpu/StandardGpuResources.h:199-266)."""

    def __init__(self):
        self._h = ctypes.c_void_p()
        check(lib.faiss_StandardGpuResources_new(ctypes.byref(self._h)))

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_StandardGpuResources_free(self._h)
            self._h = None

    def noTempMemory(self):
        check(lib.faiss_StandardGpuResources_noTempMemory(self._h))

    def setTempMemory(self, size):
        check(lib.faiss_StandardGpuResources_setTempMemory(self._h, ctypes.c_size_t(size)))

    def setPinnedMemory(self, size):
        check(lib.faiss_StandardGpuResources_setPinnedMemory(self._h, ctypes.c_size_t(size)))

    def setDefaultStream(self, device, stream):
        check(lib.faiss_StandardGpuResources_setDefaultStream(self._h, int(device), ctypes.c_void_p(int(stream))))

    def setDefaultNullStreamAllDevices(self):
        check(lib.faiss_StandardGpuResources_setDefaultNullStreamAllDevices(self._h))

    def getDefaultStream(self, device):
        out = ctypes.c_void_p()
        check(lib.faiss_StandardGpuResources_getDefaultStream(self._h, int(device), ctypes.byref(out)))
        return out.value or 0

    def syncDefaultStream(self, device):
        check(lib.faiss_StandardGpuResources_syncDefaultStream(self._h, int(device)))

    def getMemoryInfo(self):
        buf = ctypes.create_string_buffer(1 << 16)
        check(lib.faiss_StandardGpuResources_getMemoryInfo(self._h, buf, ctypes.c_size_t(len(buf))))
        raw = json.loads(buf.value.decode())
        return {int(d): {k: tuple(v) for k, v in m.items()} for d, m in raw.items()}

    # -- NCCL communicator ownership (SURVEY 7 step 1)
    def ncclInitAll(self, devices):
        """all listed devices of this process in one clique (rank i = devices[i])"""
        arr = (ctypes.c_int * len(devices))(*[int(d) for d in devices])
        check(lib.faiss_StandardGpuResources_ncclInitAll(self._h, len(devices), arr))

    def ncclInitRank(self, device, nranks, rank, unique_id):
        """this process = rank `rank` of `nranks`; unique_id: the 128 bytes of nccl_unique_id() from one rank"""
        unique_id = bytes(unique_id)
        assert len(unique_id) == 128
        check(lib.faiss_StandardGpuResources_ncclInitRank(self._h, int(device), int(nranks), int(rank), unique_id))

    def ncclRank(self, device):
        r, n = ctypes.c_int(), ctypes.c_int()
        check(lib.faiss_StandardGpuResources_ncclRank(self._h, int(device), ctypes.byref(r), ctypes.byref(n)))
        return r.value, n.value

    def getTempMemoryAvailable(self, device):
        out = ctypes.c_size_t()
        check(lib.faiss_StandardGpuResources_getTempMemoryAvailable(self._h, int(device), ctypes.byref(out)))
        return out.value


class Index:
    """faiss::Index surface (faiss/Index.h:101-435) over an opaque C handle."""

    def __init__(self):
        self._h = ctypes.c_void_p()
        self._keep = []

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_Index_free(self._h)
            self._h = None

    def _use_torch_stream(self, *tensors):
        """PyTorch interop as in faiss.contrib.torch_utils: when an argument is a CUDA tensor, order
        the library's work on torch's current stream (StandardGpuResources::setDefaultStream,
        faiss/gpu/StandardGpuResources.h:75,232) so that torch ops before/after the call are
        correctly ordered with it."""
        for t in tensors:
            if t is not None and _is_torch(t) and t.is_cuda:
                import torch

                dev = t.device.index if t.device.index is not None else torch.cuda.current_device()
                for r in self._resources():
                    r.setDefaultStream(dev, torch.cuda.current_stream(dev).cuda_stream)
                return

    def _resources(self):
        return [r for r in self._keep if isinstance(r, StandardGpuResources)]

    # -- fields
    @property
    def d(self):
        return lib.faiss_Index_d(self._h)

    @property
    def ntotal(self):
        return lib.faiss_Index_ntotal(self._h)

    @property
    def is_trained(self):
        return bool(lib.faiss_Index_is_trained(self._h))

    @property
    def metric_type(self):
        return lib.faiss_Index_metric_type(self._h)

    @property
    def metric_arg(self):
        """faiss::Index::metric_arg (the exponent of METRIC_Lp); read at search time"""
        return lib.faiss_Index_metric_arg(self._h)

    @metric_arg.setter
    def metric_arg(self, v):
        lib.faiss_Index_set_metric_arg(self._h, float(v))

    @property
    def verbose(self):
        return bool(lib.faiss_Index_verbose(self._h))

    @verbose.setter
    def verbose(self, v):
        lib.faiss_Index_set_verbose(self._h, int(bool(v)))

    # -- methods
    def _check_x(self, x):
        x = _as_f32(x)
        assert x.ndim == 2 and x.shape[1] == self.d, "x must be [n, d=%d], got %s" % (self.d, tuple(x.shape))
        return x

    def train(self, x):
        x = self._check_x(x)
        self._use_torch_stream(x)
        check(lib.faiss_Index_train(self._h, ctypes.c_int64(x.shape[0]), _ptr(x, _c_f)))

    def add(self, x):
        x = self._check_x(x)
        self._use_torch_stream(x)
        check(lib.faiss_Index_add(self._h, ctypes.c_int64(x.shape[0]), _ptr(x, _c_f)))

    def add_with_ids(self, x, ids):
        x = self._check_x(x)
        ids = _as_i64(ids)
        assert ids.shape == (x.shape[0],)
        self._use_torch_stream(x, ids)
        check(lib.faiss_Index_add_with_ids(self._h, ctypes.c_int64(x.shape[0]), _ptr(x, _c_f), _ptr(ids, _c_i64)))

    def setMinPagingSize(self, size):
        """GpuIndex::setMinPagingSize (faiss/gpu/GpuIndex.h:66-69)"""
        check(lib.faiss_GpuIndex_setMinPagingSize(self._h, ctypes.c_size_t(size)))

    def getMinPagingSize(self):
        out = ctypes.c_size_t()
        check(lib.faiss_GpuIndex_getMinPagingSize(self._h, ctypes.byref(out)))
        return int(out.value)

    def search(self, x, k, D=None, I=None, params=None):
        """params: SearchParameters(sel=) / SearchParametersIVF (per-call nprobe, sel) or None --
        faiss::Index::search(..., params)"""
        x = self._check_x(x)
        n = x.shape[0]
        if D is None:
            D = _empty_like_residency(x, (n, k), np.float32)
        if I is None:
            I = _empty_like_residency(x, (n, k), np.int64)
        self._use_torch_stream(x, D, I)
        if params is not None:
            rc = lib.faiss_Index_search_with_params(
                self._h, ctypes.c_int64(n), _ptr(x, _c_f), ctypes.c_int64(k), params._h, _ptr(D, _c_f), _ptr(I, _c_i64)
            )
            if getattr(params, "sel", None) is not None:
                params.sel._raise_pending()
            check(rc)
            return D, I
        check(
            lib.faiss_Index_search(
                self._h, ctypes.c_int64(n), _ptr(x, _c_f), ctypes.c_int64(k), _ptr(D, _c_f), _ptr(I, _c_i64)
            )
        )
        return D, I

    def search_and_reconstruct(self, x, k, params=None):
        """faiss::Index::search_and_reconstruct -> (D, I, R), R [n, k, d] the stored vector of each result (all 0xFF
        bytes where I is -1); outputs follow x's residency.  GpuIndexFlat and the IVF indexes."""
        x = self._check_x(x)
        n = x.shape[0]
        D = _empty_like_residency(x, (n, k), np.float32)
        I = _empty_like_residency(x, (n, k), np.int64)
        R = _empty_like_residency(x, (n, k, self.d), np.float32)
        self._use_torch_stream(x, D, I, R)
        rc = lib.faiss_Index_search_and_reconstruct(
            self._h, ctypes.c_int64(n), _ptr(x, _c_f), ctypes.c_int64(k), params._h if params is not None else None,
            _ptr(D, _c_f), _ptr(I, _c_i64), _ptr(R, _c_f)
        )
        if params is not None and getattr(params, "sel", None) is not None:
            params.sel._raise_pending()
        check(rc)
        return D, I, R

    def assign(self, x, k=1):
        x = self._check_x(x)
        n = x.shape[0]
        I = _empty_like_residency(x, (n, k), np.int64)
        self._use_torch_stream(x)
        check(lib.faiss_Index_assign(self._h, ctypes.c_int64(n), _ptr(x, _c_f), _ptr(I, _c_i64), ctypes.c_int64(k)))
        return I

    def reset(self):
        check(lib.faiss_Index_reset(self._h))

    def reconstruct(self, key):
        out = np.empty(self.d, dtype=np.float32)
        check(lib.faiss_Index_reconstruct(self._h, ctypes.c_int64(key), _ptr(out, _c_f)))
        return out

    def reconstruct_n(self, i0=0, ni=-1):
        if ni < 0:
            ni = self.ntotal - i0
        out = np.empty((ni, self.d), dtype=np.float32)
        check(lib.faiss_Index_reconstruct_n(self._h, ctypes.c_int64(i0), ctypes.c_int64(ni), _ptr(out, _c_f)))
        return out

    def reconstruct_batch(self, keys):
        keys = _as_i64(np.asarray(keys))
        out = np.empty((keys.shape[0], self.d), dtype=np.float32)
        check(lib.faiss_Index_reconstruct_batch(self._h, ctypes.c_int64(keys.shape[0]), _ptr(keys, _c_i64), _ptr(out, _c_f)))
        return out

    def compute_residual(self, x, key):
        x = _as_f32(x).reshape(1, -1)
        return self.compute_residual_n(x, np.array([key], dtype=np.int64))[0]

    def compute_residual_n(self, x, keys):
        x = self._check_x(x)
        keys = _as_i64(keys)
        out = _empty_like_residency(x, tuple(x.shape), np.float32)
        self._use_torch_stream(x, keys)
        check(
            lib.faiss_Index_compute_residual_n(
                self._h, ctypes.c_int64(x.shape[0]), _ptr(x, _c_f), _ptr(out, _c_f), _ptr(keys, _c_i64)
            )
        )
        return out


class IDSelector:
    """faiss::IDSelector (faiss/impl/IDSelector.h): restricts a search to the stored ids it accepts -- the row
    number for GpuIndexFlat, the id stored in the list for the IVF indexes (whose coarse search is not
    filtered).  Leaves copy their inputs; combinators keep their operands alive."""

    def __init__(self, make, *children):
        self._children = children
        self._h = ctypes.c_void_p()
        check(make(ctypes.byref(self._h)))

    def _raise_pending(self):
        """re-raise what a callback leaf raised during the last search (the C ABI only sees "not selected")"""
        for c in self._children:
            c._raise_pending()

    def is_member(self, i):
        r = lib.faiss_IDSelector_is_member(self._h, ctypes.c_int64(int(i)))
        if r < 0:
            raise FaissError(-1, "null IDSelector handle")
        return bool(r)

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_IDSelector_free(self._h)
            self._h = None


class IDSelectorRange(IDSelector):
    """imin <= id < imax (an empty range selects nothing)"""

    def __init__(self, imin, imax):
        self.imin, self.imax = int(imin), int(imax)
        super().__init__(lambda p: lib.faiss_IDSelectorRange_new(p, ctypes.c_int64(self.imin), ctypes.c_int64(self.imax)))


def _id_array(ids):
    ids = np.ascontiguousarray(np.asarray(ids, dtype=np.int64).reshape(-1))
    return ids, ids.ctypes.data_as(_c_i64)


class IDSelectorArray(IDSelector):
    """id is one of ids (membership: duplicates and ids past ntotal are harmless)"""

    def __init__(self, ids):
        ids, p_ids = _id_array(ids)
        super().__init__(lambda p: lib.faiss_IDSelectorArray_new(p, ctypes.c_size_t(ids.shape[0]), p_ids))


class IDSelectorBatch(IDSelector):
    """id is one of indices"""

    def __init__(self, indices):
        ids, p_ids = _id_array(indices)
        super().__init__(lambda p: lib.faiss_IDSelectorBatch_new(p, ctypes.c_size_t(ids.shape[0]), p_ids))


class IDSelectorBitmap(IDSelector):
    """bit (id & 7) of byte id >> 3 of a uint8 bitmap (ids past the bitmap are not selected)"""

    def __init__(self, bitmap):
        bm = np.ascontiguousarray(np.asarray(bitmap, dtype=np.uint8).reshape(-1))
        super().__init__(lambda p: lib.faiss_IDSelectorBitmap_new(p, ctypes.c_size_t(bm.shape[0]), bm.ctypes.data_as(_c_u8)))


class IDSelectorNot(IDSelector):
    def __init__(self, sel):
        super().__init__(lambda p: lib.faiss_IDSelectorNot_new(p, sel._h), sel)


class IDSelectorAnd(IDSelector):
    def __init__(self, lhs, rhs):
        super().__init__(lambda p: lib.faiss_IDSelectorAnd_new(p, lhs._h, rhs._h), lhs, rhs)


class IDSelectorOr(IDSelector):
    def __init__(self, lhs, rhs):
        super().__init__(lambda p: lib.faiss_IDSelectorOr_new(p, lhs._h, rhs._h), lhs, rhs)


class IDSelectorXOr(IDSelector):
    def __init__(self, lhs, rhs):
        super().__init__(lambda p: lib.faiss_IDSelectorXOr_new(p, lhs._h, rhs._h), lhs, rhs)


_SEL_CB = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_int64)


class IDSelectorCallback(IDSelector):
    """fn(id) -> bool, called on the host once per stored entry and search call"""

    def __init__(self, fn):
        self._error = None

        def call(ctx, i):
            if self._error is not None:
                return 0
            try:
                return 1 if fn(int(i)) else 0
            except BaseException as e:  # kept, and raised again when the search returns
                self._error = e
                return 0

        self._cb = _SEL_CB(call)
        super().__init__(lambda p: lib.faiss_b200_IDSelectorCallback_new(p, self._cb, None))

    def _raise_pending(self):
        e, self._error = self._error, None
        if e is not None:
            raise e


class SearchParameters:
    """faiss::SearchParameters (faiss/Index.h:88-93): sel restricts the search to the ids it accepts."""

    def __init__(self, sel=None):
        self.sel = sel
        self._h = ctypes.c_void_p()
        check(lib.faiss_SearchParameters_new(ctypes.byref(self._h), sel._h if sel is not None else None))

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_SearchParameters_free(self._h)
            self._h = None


class SearchParametersIVF(SearchParameters):
    """faiss::SearchParametersIVF (faiss/IndexIVF.h:68-90): per-call nprobe and IDSelector; max_codes must stay 0
    on the GPU."""

    def __init__(self, nprobe=1, max_codes=0, sel=None):
        self.sel = sel
        self._h = ctypes.c_void_p()
        check(
            lib.faiss_SearchParametersIVF_new_with_sel(
                ctypes.byref(self._h),
                sel._h if sel is not None else None,
                ctypes.c_size_t(int(nprobe)),
                ctypes.c_size_t(int(max_codes)),
            )
        )


_INTERRUPT_CB = None


def set_interrupt_callback(fn):
    """faiss::InterruptCallback: fn() -> truthy to make the running call fail with 'computation interrupted'; None clears."""
    global _INTERRUPT_CB
    proto = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p)
    if fn is None:
        lib.faiss_b200_set_interrupt_callback(ctypes.cast(None, proto), None)
        _INTERRUPT_CB = None
        return
    _INTERRUPT_CB = proto(lambda _ctx: 1 if fn() else 0)  # keep the thunk alive
    lib.faiss_b200_set_interrupt_callback(_INTERRUPT_CB, None)


class GpuIndexFlat(Index):
    """faiss::gpu::GpuIndexFlat (faiss/gpu/GpuIndexFlat.h:43-141)."""

    def __init__(self, res, d, metric=METRIC_L2, device=0, use_tensor_cores=True, use_float16=False):
        super().__init__()
        self._keep.append(res)
        check(
            lib.faiss_GpuIndexFlat_new_with_config(
                ctypes.byref(self._h), res._h, int(d), int(metric), int(device), int(bool(use_tensor_cores)),
                int(bool(use_float16)),
            )
        )

    def copyFrom(self, xb):
        xb = _as_f32(xb)
        check(lib.faiss_GpuIndexFlat_copyFrom(self._h, ctypes.c_int64(xb.shape[0]), _ptr(xb, _c_f)))

    def copyTo(self):
        out = np.empty((self.ntotal, self.d), dtype=np.float32)
        check(lib.faiss_GpuIndexFlat_copyTo(self._h, _ptr(out, _c_f)))
        return out

    def setUseTensorCores(self, enable):
        check(lib.faiss_GpuIndexFlat_setUseTensorCores(self._h, int(bool(enable))))

    def lastSearchInfo(self):
        out = (ctypes.c_int * 2)()
        check(lib.faiss_GpuIndexFlat_lastSearchInfo(self._h, out))
        return {"tensor_cores": int(out[0]), "fallback_queries": int(out[1])}

    def lastSearchOperandBits(self):
        """Operand width of the last search's tensor-core scoring: 8 (int8), 16 (fp16), or 0 (exact kernel)."""
        out = ctypes.c_int(0)
        check(lib.faiss_GpuIndexFlat_lastSearchOperandBits(self._h, ctypes.byref(out)))
        return int(out.value)

    def lastSearchRepairedQueries(self):
        """Queries of the last search searched again with provable thresholds because their estimated thresholds
        overshot; they are not among lastSearchInfo()'s fallback (exact-kernel) queries."""
        out = ctypes.c_int(0)
        check(lib.faiss_GpuIndexFlat_lastSearchRepairedQueries(self._h, ctypes.byref(out)))
        return int(out.value)


class GpuIndexFlatL2(GpuIndexFlat):
    def __init__(self, res, d, device=0, use_tensor_cores=True, use_float16=False):
        super().__init__(res, d, METRIC_L2, device, use_tensor_cores, use_float16)


class GpuIndexFlatIP(GpuIndexFlat):
    def __init__(self, res, d, device=0, use_tensor_cores=True, use_float16=False):
        super().__init__(res, d, METRIC_INNER_PRODUCT, device, use_tensor_cores, use_float16)


class GpuIndexIVF(Index):
    """faiss::gpu::GpuIndexIVF (faiss/gpu/GpuIndexIVF.h:40-167)."""

    @property
    def nprobe(self):
        return lib.faiss_GpuIndexIVF_nprobe(self._h)

    @nprobe.setter
    def nprobe(self, v):
        check(lib.faiss_GpuIndexIVF_set_nprobe(self._h, ctypes.c_size_t(int(v))))

    @property
    def nlist(self):
        return lib.faiss_GpuIndexIVF_nlist(self._h)

    def setClustering(self, niter=-1, seed=-1, max_points_per_centroid=-1):
        check(lib.faiss_GpuIndexIVF_set_clustering(self._h, int(niter), int(seed), int(max_points_per_centroid)))

    def reserveMemory(self, n):
        check(lib.faiss_GpuIndexIVF_reserveMemory(self._h, ctypes.c_size_t(int(n))))

    def reclaimMemory(self):
        out = ctypes.c_size_t()
        check(lib.faiss_GpuIndexIVF_reclaimMemory(self._h, ctypes.byref(out)))
        return out.value

    def getListLength(self, l):
        return lib.faiss_GpuIndexIVF_get_list_size(self._h, ctypes.c_size_t(int(l)))

    def _code_size(self):
        raise NotImplementedError

    def getListVectorData(self, l):
        n = self.getListLength(l)
        out = np.empty(n * self._code_size(), dtype=np.uint8)
        check(lib.faiss_GpuIndexIVF_getListVectorData(self._h, ctypes.c_size_t(int(l)), _ptr(out, _c_u8)))
        return out

    def getListIndices(self, l):
        n = self.getListLength(l)
        out = np.empty(n, dtype=np.int64)
        check(lib.faiss_GpuIndexIVF_getListIndices(self._h, ctypes.c_size_t(int(l)), _ptr(out, _c_i64)))
        return out

    def setCoarseCentroids(self, c):
        c = _as_f32(c)
        assert tuple(c.shape) == (self.nlist, self.d)
        check(lib.faiss_GpuIndexIVF_setCoarseCentroids(self._h, _ptr(c, _c_f)))

    def getCoarseCentroids(self):
        out = np.empty((self.nlist, self.d), dtype=np.float32)
        check(lib.faiss_GpuIndexIVF_getCoarseCentroids(self._h, _ptr(out, _c_f)))
        return out

    def setList(self, l, codes, ids):
        codes = np.ascontiguousarray(codes, dtype=np.uint8).reshape(-1)
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        assert codes.size == ids.size * self._code_size()
        check(
            lib.faiss_GpuIndexIVF_setList(
                self._h, ctypes.c_size_t(int(l)), ctypes.c_int64(ids.size), _ptr(codes, _c_u8), _ptr(ids, _c_i64)
            )
        )

    def setListSizes(self, lens):
        """exact capacity for every list in one relayout (call before the per-list setList of a bulk clone)"""
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        assert lens.shape == (self.nlist,)
        check(lib.faiss_GpuIndexIVF_setListSizes(self._h, _ptr(lens, _c_i64)))

    def setIsTrained(self, v=True):
        check(lib.faiss_GpuIndexIVF_set_is_trained(self._h, int(bool(v))))

    def code_sizes(self):
        """(coarse_code_size, code_size): IndexIVF's list-number and code byte widths"""
        c, s = ctypes.c_int(), ctypes.c_int()
        check(lib.faiss_GpuIndexIVF_code_sizes(self._h, ctypes.byref(c), ctypes.byref(s)))
        return c.value, s.value

    def search_and_return_codes(self, x, k, include_listnos=False, params=None):
        """faiss::IndexIVF::search_and_return_codes -> (D, I, codes), codes [n, k, (coarse_code_size if include_listnos)
        + code_size] uint8: the CPU inverted-list bytes of each result, prefixed by its list number (little-endian);
        all 0xFF where I is -1.  Outputs follow x's residency."""
        x = self._check_x(x)
        n = x.shape[0]
        ccs, cs = self.code_sizes()
        D = _empty_like_residency(x, (n, k), np.float32)
        I = _empty_like_residency(x, (n, k), np.int64)
        C = _empty_like_residency(x, (n, k, (ccs if include_listnos else 0) + cs), np.uint8)
        self._use_torch_stream(x, D, I, C)
        rc = lib.faiss_GpuIndexIVF_search_and_return_codes(
            self._h, ctypes.c_int64(n), _ptr(x, _c_f), ctypes.c_int64(k), params._h if params is not None else None,
            _ptr(D, _c_f), _ptr(I, _c_i64), _ptr(C, _c_u8), int(bool(include_listnos))
        )
        if params is not None and getattr(params, "sel", None) is not None:
            params.sel._raise_pending()
        check(rc)
        return D, I, C

    def search_preassigned(self, x, k, assign, centroid_dis=None):
        x = self._check_x(x)
        n = x.shape[0]
        assign = _as_i64(assign)
        if centroid_dis is None:
            centroid_dis = np.zeros(assign.shape, dtype=np.float32)
            if _is_torch(x) and x.is_cuda:
                import torch

                centroid_dis = torch.zeros(tuple(assign.shape), dtype=torch.float32, device=x.device)
        centroid_dis = _as_f32(centroid_dis)
        D = _empty_like_residency(x, (n, k), np.float32)
        I = _empty_like_residency(x, (n, k), np.int64)
        self._use_torch_stream(x, assign)
        check(
            lib.faiss_GpuIndexIVF_search_preassigned(
                self._h,
                ctypes.c_int64(n),
                _ptr(x, _c_f),
                ctypes.c_int64(k),
                _ptr(assign, _c_i64),
                _ptr(centroid_dis, _c_f),
                _ptr(D, _c_f),
                _ptr(I, _c_i64),
            )
        )
        return D, I


class GpuIndexIVFFlat(GpuIndexIVF):
    """faiss::gpu::GpuIndexIVFFlat (faiss/gpu/GpuIndexIVFFlat.h:24-119)."""

    def __init__(self, res, d, nlist, metric=METRIC_L2, device=0, quantizer=None):
        """quantizer: a GpuIndexFlat to share as the coarse quantiser (faiss/gpu/GpuIndexIVFFlat.h:48-59), or None"""
        super().__init__()
        self._keep.append(res)
        if quantizer is not None:
            self._keep.append(quantizer)
            check(
                lib.faiss_GpuIndexIVFFlat_new_with_quantizer(
                    ctypes.byref(self._h), res._h, quantizer._h, int(d), ctypes.c_int64(nlist), int(metric), int(device)
                )
            )
            return
        check(
            lib.faiss_GpuIndexIVFFlat_new(
                ctypes.byref(self._h), res._h, int(d), ctypes.c_int64(nlist), int(metric), int(device)
            )
        )

    def _code_size(self):
        return 4 * self.d


class GpuIndexIVFPQ(GpuIndexIVF):
    """faiss::gpu::GpuIndexIVFPQ (faiss/gpu/GpuIndexIVFPQ.h:56-181)."""

    def __init__(self, res, d, nlist, M, nbits=8, metric=METRIC_L2, device=0, quantizer=None, interleaved_layout=False):
        """quantizer: a GpuIndexFlat to share as the coarse quantiser (faiss/gpu/GpuIndexIVFPQ.h:69-82), or None.
        interleaved_layout: GpuIndexIVFPQConfig::interleavedLayout; with it nbits may be 4, 5, 6 or 8."""
        super().__init__()
        self._keep.append(res)
        self.M = int(M)
        self.nbits = int(nbits)
        if interleaved_layout:
            if quantizer is not None:
                self._keep.append(quantizer)
            check(
                lib.faiss_GpuIndexIVFPQ_new_with_config(
                    ctypes.byref(self._h), res._h, quantizer._h if quantizer is not None else None, int(d),
                    ctypes.c_int64(nlist), ctypes.c_int64(M), ctypes.c_int64(nbits), int(metric), int(device), 1,
                )
            )
            return
        if quantizer is not None:
            self._keep.append(quantizer)
            check(
                lib.faiss_GpuIndexIVFPQ_new_with_quantizer(
                    ctypes.byref(self._h), res._h, quantizer._h, int(d), ctypes.c_int64(nlist), ctypes.c_int64(M), ctypes.c_int64(nbits),
                    int(metric), int(device),
                )
            )
            return
        check(
            lib.faiss_GpuIndexIVFPQ_new(
                ctypes.byref(self._h),
                res._h,
                int(d),
                ctypes.c_int64(nlist),
                ctypes.c_int64(M),
                ctypes.c_int64(nbits),
                int(metric),
                int(device),
            )
        )

    def _code_size(self):
        return (self.M * self.nbits + 7) // 8  # ProductQuantizer::code_size

    def setPQCentroids(self, c):
        """c: [M, 2^nbits, d/M] (ProductQuantizer::centroids)"""
        c = _as_f32(c)
        assert c.size == (1 << self.nbits) * self.d
        check(lib.faiss_GpuIndexIVFPQ_setPQCentroids(self._h, _ptr(c, _c_f)))

    def getPQCentroids(self):
        out = np.empty((self.M, 1 << self.nbits, self.d // self.M), dtype=np.float32)
        check(lib.faiss_GpuIndexIVFPQ_getPQCentroids(self._h, _ptr(out, _c_f)))
        return out

    def setPQClustering(self, niter=-1, seed=-1, max_points_per_centroid=-1):
        check(lib.faiss_GpuIndexIVFPQ_set_pq_clustering(self._h, int(niter), int(seed), int(max_points_per_centroid)))

    def setPrecomputedCodes(self, enable):
        check(lib.faiss_GpuIndexIVFPQ_setPrecomputedCodes(self._h, int(bool(enable))))


class GpuIndexIVFScalarQuantizer(GpuIndexIVF):
    """faiss::gpu::GpuIndexIVFScalarQuantizer (faiss/gpu/GpuIndexIVFScalarQuantizer.h:30-139).

    qtype is a ScalarQuantizer::QuantizerType (QT_8bit ... QT_6bit); trained parameters use the CPU's
    ScalarQuantizer::trained layout, lists the CPU's ArrayInvertedLists bytes."""

    def __init__(self, res, d, nlist, qtype=None, metric=METRIC_L2, encodeResidual=True, device=0, quantizer=None):
        """quantizer: a GpuIndexFlat to share as the coarse quantiser, or None"""
        super().__init__()
        self._keep.append(res)
        qtype = QT_8bit if qtype is None else int(qtype)
        if quantizer is not None:
            self._keep.append(quantizer)
            check(
                lib.faiss_GpuIndexIVFScalarQuantizer_new_with_quantizer(
                    ctypes.byref(self._h), res._h, quantizer._h, int(d), ctypes.c_int64(nlist), qtype, int(metric),
                    int(bool(encodeResidual)), int(device),
                )
            )
            return
        check(
            lib.faiss_GpuIndexIVFScalarQuantizer_new(
                ctypes.byref(self._h), res._h, int(d), ctypes.c_int64(nlist), qtype, int(metric),
                int(bool(encodeResidual)), int(device),
            )
        )

    def _code_size(self):
        out = ctypes.c_size_t()
        check(lib.faiss_GpuIndexIVFScalarQuantizer_code_size(self._h, ctypes.byref(out)))
        return out.value

    @property
    def code_size(self):
        return self._code_size()

    @property
    def qtype(self):
        out = ctypes.c_int()
        check(lib.faiss_GpuIndexIVFScalarQuantizer_qtype(self._h, ctypes.byref(out)))
        return out.value

    @property
    def by_residual(self):
        out = ctypes.c_int()
        check(lib.faiss_GpuIndexIVFScalarQuantizer_by_residual(self._h, ctypes.byref(out)))
        return bool(out.value)

    def getTrained(self):
        n = ctypes.c_size_t()
        check(lib.faiss_GpuIndexIVFScalarQuantizer_get_trained(self._h, ctypes.cast(None, _c_f), ctypes.byref(n)))
        out = np.empty(n.value, dtype=np.float32)
        check(lib.faiss_GpuIndexIVFScalarQuantizer_get_trained(self._h, _ptr(out, _c_f), ctypes.byref(n)))
        return out

    def setTrained(self, t):
        t = np.ascontiguousarray(t, dtype=np.float32).reshape(-1)
        check(lib.faiss_GpuIndexIVFScalarQuantizer_set_trained(self._h, _ptr(t, _c_f), ctypes.c_size_t(t.size)))

    def setRangeStat(self, rangestat, rangestat_arg=0.0):
        """ScalarQuantizer::rangestat / rangestat_arg for train(); only RS_minmax trains on the GPU"""
        check(lib.faiss_GpuIndexIVFScalarQuantizer_set_rangestat(self._h, int(rangestat), ctypes.c_float(rangestat_arg)))


# faiss::gpu::graph_build_algo, codebook_gen, search_algo, hash_mode (faiss/gpu/GpuIndexCagra.h:44-204)
graph_build_algo_IVF_PQ = 0
graph_build_algo_NN_DESCENT = 1
graph_build_algo_ITERATIVE_SEARCH = 2
codebook_gen_PER_SUBSPACE = 0
codebook_gen_PER_CLUSTER = 1
search_algo_SINGLE_CTA = 0
search_algo_MULTI_CTA = 1
search_algo_MULTI_KERNEL = 2
search_algo_AUTO = 100
hash_mode_HASH = 0
hash_mode_SMALL = 1
hash_mode_AUTO = 100


class _CagraConfigC(ctypes.Structure):
    """FaissGpuIndexCagraConfig (include/faiss_b200_c.h)"""

    _fields_ = [
        ("device", ctypes.c_int),
        ("intermediate_graph_degree", ctypes.c_size_t),
        ("graph_degree", ctypes.c_size_t),
        ("build_algo", ctypes.c_int),
        ("nn_descent_niter", ctypes.c_size_t),
        ("refine_rate", ctypes.c_float),
        ("store_dataset", ctypes.c_int),
        ("guarantee_connectivity", ctypes.c_int),
        ("n_lists", ctypes.c_uint32),
        ("kmeans_n_iters", ctypes.c_uint32),
        ("kmeans_trainset_fraction", ctypes.c_double),
        ("pq_bits", ctypes.c_uint32),
        ("pq_dim", ctypes.c_uint32),
        ("codebook_kind", ctypes.c_int),
        ("force_random_rotation", ctypes.c_int),
        ("conservative_memory_allocation", ctypes.c_int),
        ("n_probes", ctypes.c_uint32),
        ("max_internal_batch_size", ctypes.c_uint32),
    ]


class _CagraSearchC(ctypes.Structure):
    """FaissSearchParametersCagraConfig (include/faiss_b200_c.h)"""

    _fields_ = [
        ("max_queries", ctypes.c_size_t),
        ("itopk_size", ctypes.c_size_t),
        ("max_iterations", ctypes.c_size_t),
        ("algo", ctypes.c_int),
        ("team_size", ctypes.c_size_t),
        ("search_width", ctypes.c_size_t),
        ("min_iterations", ctypes.c_size_t),
        ("thread_block_size", ctypes.c_size_t),
        ("hashmap_mode", ctypes.c_int),
        ("hashmap_min_bitlen", ctypes.c_size_t),
        ("hashmap_max_fill_rate", ctypes.c_float),
        ("num_random_samplings", ctypes.c_uint32),
        ("seed", ctypes.c_uint64),
    ]


def _defaults(struct, init):
    c = struct()
    init(ctypes.byref(c))
    return c


class IVFPQBuildCagraConfig:
    """faiss::gpu::IVFPQBuildCagraConfig (faiss/gpu/GpuIndexCagra.h:59-127)"""

    _names = ("n_lists", "kmeans_n_iters", "kmeans_trainset_fraction", "pq_bits", "pq_dim", "codebook_kind",
              "force_random_rotation", "conservative_memory_allocation")

    def __init__(self):
        c = _defaults(_CagraConfigC, lib.faiss_GpuIndexCagraConfig_init)
        for n in self._names:
            setattr(self, n, getattr(c, n))


class IVFPQSearchCagraConfig:
    """faiss::gpu::IVFPQSearchCagraConfig (faiss/gpu/GpuIndexCagra.h:129-174); lut_dtype, internal_distance_dtype and
    preferred_shmem_carveout are accepted and have no effect"""

    def __init__(self):
        c = _defaults(_CagraConfigC, lib.faiss_GpuIndexCagraConfig_init)
        self.n_probes = c.n_probes
        self.max_internal_batch_size = c.max_internal_batch_size
        self.lut_dtype = None
        self.internal_distance_dtype = None
        self.preferred_shmem_carveout = 1.0


class GpuIndexCagraConfig:
    """faiss::gpu::GpuIndexCagraConfig (faiss/gpu/GpuIndexCagra.h:176-193)"""

    _names = ("device", "intermediate_graph_degree", "graph_degree", "build_algo", "nn_descent_niter", "refine_rate",
              "store_dataset", "guarantee_connectivity")

    def __init__(self):
        c = _defaults(_CagraConfigC, lib.faiss_GpuIndexCagraConfig_init)
        for n in self._names:
            setattr(self, n, getattr(c, n))
        self.store_dataset = bool(self.store_dataset)
        self.guarantee_connectivity = bool(self.guarantee_connectivity)
        self.ivf_pq_params = None  # None: IVFPQBuildCagraConfig()
        self.ivf_pq_search_params = None  # None: IVFPQSearchCagraConfig()

    def _c(self):
        c = _defaults(_CagraConfigC, lib.faiss_GpuIndexCagraConfig_init)
        for n in self._names:
            setattr(c, n, type(getattr(c, n))(getattr(self, n)))
        bp = self.ivf_pq_params or IVFPQBuildCagraConfig()
        for n in IVFPQBuildCagraConfig._names:
            setattr(c, n, type(getattr(c, n))(getattr(bp, n)))
        sp = self.ivf_pq_search_params or IVFPQSearchCagraConfig()
        c.n_probes = int(sp.n_probes)
        c.max_internal_batch_size = int(sp.max_internal_batch_size)
        return c


class SearchParametersCagra(SearchParameters):
    """faiss::gpu::SearchParametersCagra (faiss/gpu/GpuIndexCagra.h:206-251).  Fields may be set after construction;
    a search reads them when it starts."""

    _names = tuple(f[0] for f in _CagraSearchC._fields_)

    def __init__(self, sel=None, **kw):
        self.sel = sel
        self._handle = None
        c = _defaults(_CagraSearchC, lib.faiss_SearchParametersCagraConfig_init)
        for n in self._names:
            setattr(self, n, getattr(c, n))
        for n, v in kw.items():
            assert n in self._names, "unknown SearchParametersCagra field %s" % n
            setattr(self, n, v)

    @property
    def _h(self):
        c = _defaults(_CagraSearchC, lib.faiss_SearchParametersCagraConfig_init)
        for n in self._names:
            setattr(c, n, type(getattr(c, n))(getattr(self, n)))
        self._free()
        self._handle = ctypes.c_void_p()
        check(lib.faiss_SearchParametersCagra_new(
            ctypes.byref(self._handle), self.sel._h if self.sel is not None else None, ctypes.byref(c)))
        return self._handle

    def _free(self):
        if getattr(self, "_handle", None) and lib is not None:
            lib.faiss_SearchParameters_free(self._handle)
            self._handle = None

    def __del__(self):
        self._free()


class GpuIndexCagra(Index):
    """faiss::gpu::GpuIndexCagra (faiss/gpu/GpuIndexCagra.h:253-379): fp32, METRIC_L2 / METRIC_INNER_PRODUCT.
    train (or add) builds the graph on the device: IVF-PQ candidates, exact refine, optimise (DESIGN "GpuIndexCagra").
    Search takes SearchParametersCagra through params=."""

    def __init__(self, res, d, metric=METRIC_L2, config=None):
        super().__init__()
        self._keep.append(res)
        c = (config or GpuIndexCagraConfig())._c()
        check(lib.faiss_GpuIndexCagra_new(ctypes.byref(self._h), res._h, int(d), int(metric), ctypes.byref(c)))

    @property
    def graph_degree(self):
        out = ctypes.c_int()
        check(lib.faiss_GpuIndexCagra_graph_degree(self._h, ctypes.byref(out)))
        return out.value

    def get_knngraph(self):
        """[ntotal, graph_degree] int64 (-1: no edge)"""
        out = np.empty((self.ntotal, self.graph_degree), dtype=np.int64)
        check(lib.faiss_GpuIndexCagra_get_knngraph(self._h, _ptr(out, _c_i64)))
        return out

    def copyFrom(self, xb, graph):
        """the IndexHNSWCagra payload: xb [n, d], graph [n, degree] int64 (its level-0 table; -1 entries are skipped)"""
        xb = _as_f32(xb)
        graph = np.ascontiguousarray(graph, dtype=np.int64)
        assert graph.ndim == 2 and graph.shape[0] == xb.shape[0] and xb.shape[1] == self.d
        check(lib.faiss_GpuIndexCagra_copyFrom(
            self._h, ctypes.c_int64(xb.shape[0]), _ptr(xb, _c_f), _ptr(graph, _c_i64), int(graph.shape[1])))

    def copyTo(self):
        """-> (xb [ntotal, d] float32, graph [ntotal, graph_degree] int64)"""
        xb = np.empty((self.ntotal, self.d), dtype=np.float32)
        graph = np.empty((self.ntotal, self.graph_degree), dtype=np.int64)
        check(lib.faiss_GpuIndexCagra_copyTo(self._h, _ptr(xb, _c_f), _ptr(graph, _c_i64)))
        return xb, graph

    def lastSearchDistanceCount(self):
        """distance evaluations of the last search, summed over its queries"""
        out = ctypes.c_int64()
        check(lib.faiss_GpuIndexCagra_lastSearchDistanceCount(self._h, ctypes.byref(out)))
        return out.value

    def lastBuildSeconds(self):
        """{"ivf_pq", "refine", "optimize"}: seconds of the last build's three stages"""
        out = (ctypes.c_double * 3)()
        check(lib.faiss_GpuIndexCagra_lastBuildSeconds(self._h, out))
        return {"ivf_pq": out[0], "refine": out[1], "optimize": out[2]}


def cagra_optimize(res, G0, K, device=0):
    """The build's graph optimisation on its own (b200_cagra_optimize): G0 [n, K0] -> G [n, K], uint32 ids.  G0 may be a
    numpy array or a CUDA tensor (int32 / int64 / uint32 values); the result follows its residency as int64."""
    import torch

    t = G0 if _is_torch(G0) else torch.from_numpy(np.ascontiguousarray(G0).astype(np.int64))
    g0 = t.to(device="cuda:%d" % device, dtype=torch.int64).to(torch.int32).contiguous()
    n, K0 = g0.shape
    G = torch.empty((n, int(K)), dtype=torch.int32, device=g0.device)
    torch.cuda.synchronize(g0.device)
    check(lib.b200_cagra_optimize(res._h, int(device), ctypes.c_void_p(g0.data_ptr()), ctypes.c_int64(n), int(K0), int(K),
                                  ctypes.c_void_p(G.data_ptr())))
    res.syncDefaultStream(device)
    out = G.to(torch.int64) & 0xFFFFFFFF
    return out if _is_torch(G0) else out.cpu().numpy()


class IndexShards(Index):
    """faiss::IndexShards (faiss/IndexShards.h:21-106)."""

    def __init__(self, d, threaded=False, successive_ids=True):
        super().__init__()
        check(
            lib.faiss_IndexShards_new_with_options(
                ctypes.byref(self._h), ctypes.c_int64(d), int(bool(threaded)), int(bool(successive_ids))
            )
        )
        self._shards = []

    def add_shard(self, index):
        check(lib.faiss_IndexShards_add_shard(self._h, index._h))
        self._shards.append(index)

    def _resources(self):
        out = []
        for s in self._shards:
            out.extend(s._resources())
        return out

    def remove_shard(self, index):
        check(lib.faiss_IndexShards_remove_shard(self._h, index._h))
        self._shards.remove(index)

    def at(self, i):
        return self._shards[i]

    def count(self):
        return len(self._shards)

    def lastSearchPath(self):
        """'nccl' if the last search ran per-device threads + ncclAllGather + device merge, 'host' for the
        reference's thread-per-shard + host merge"""
        return {0: "host", 1: "nccl"}.get(lib.faiss_IndexShards_lastSearchPath(self._h), "?")

    def __del__(self):
        # free the meta index before the shards it points to
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_Index_free(self._h)
            self._h = None
        self._shards = []


class IndexShardsIVF(IndexShards):
    """faiss::IndexShardsIVF (faiss/IndexShardsIVF.cpp:100-251): IVF shards over one shared coarse quantiser (a
    GpuIndexFlat): one coarse search, search_preassigned on every shard, merge."""

    def __init__(self, quantizer, nlist, threaded=False, successive_ids=True):
        Index.__init__(self)
        self._keep.append(quantizer)
        check(lib.faiss_IndexShardsIVF_new(ctypes.byref(self._h), quantizer._h, ctypes.c_int64(nlist), int(bool(threaded)), int(bool(successive_ids))))
        self._shards = []

    def add_shard(self, index):
        check(lib.faiss_IndexShardsIVF_add_shard(self._h, index._h))
        self._shards.append(index)


def nccl_unique_id():
    """128 bytes to hand to every rank's StandardGpuResources.ncclInitRank (ncclGetUniqueId)."""
    buf = ctypes.create_string_buffer(128)
    check(lib.faiss_b200_nccl_unique_id(buf))
    return buf.raw


class DistributedIndexShards(Index):
    """IndexShards with one shard per NCCL rank (faiss/IndexShards.cpp:197-264 semantics; one grouped
    all-gather + device merge; Flat shards pool their thresholds).  `search` is a collective call."""

    def __init__(self, res, local, successive_ids=True):
        super().__init__()
        self._keep.append(res)
        self._local = local
        check(lib.faiss_DistributedIndexShards_new(ctypes.byref(self._h), res._h, local._h, int(bool(successive_ids))))

    def _resources(self):
        return [r for r in self._keep if isinstance(r, StandardGpuResources)]

    def sync(self):
        check(lib.faiss_DistributedIndexShards_sync(self._h))

    def info(self):
        r, n, o = ctypes.c_int(), ctypes.c_int(), ctypes.c_int64()
        check(lib.faiss_DistributedIndexShards_info(self._h, ctypes.byref(r), ctypes.byref(n), ctypes.byref(o)))
        return {"rank": r.value, "world": n.value, "id_offset": o.value}

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_Index_free(self._h)
            self._h = None
        self._local = None


def kmeans(res, x, k, niter=25, seed=1234, max_points_per_centroid=256, device=0):
    """Lloyd k-means on the device (role of faiss.Kmeans / faiss::Clustering); returns (centroids, obj)."""
    x = _as_f32(x)
    n, d = x.shape
    cent = np.empty((k, d), dtype=np.float32)
    obj = np.zeros(niter, dtype=np.float32)
    check(
        lib.faiss_b200_kmeans(
            res._h,
            int(device),
            ctypes.c_size_t(d),
            ctypes.c_size_t(n),
            ctypes.c_size_t(k),
            _ptr(x, _c_f),
            int(niter),
            int(seed),
            int(max_points_per_centroid),
            _ptr(cent, _c_f),
            _ptr(obj, _c_f),
        )
    )
    return cent, obj


def kmeans_ex(res, x, k, niter=25, seed=1234, max_points_per_centroid=256, metric=METRIC_L2, spherical=False, device=0):
    """k-means with an assignment index of `metric` and ClusteringParameters::spherical."""
    x = _as_f32(x)
    n, d = x.shape
    cent = np.empty((k, d), dtype=np.float32)
    obj = np.zeros(niter, dtype=np.float32)
    check(
        lib.faiss_b200_kmeans_ex(
            res._h, int(device), ctypes.c_size_t(d), ctypes.c_size_t(n), ctypes.c_size_t(k), _ptr(x, _c_f), int(niter), int(seed),
            int(max_points_per_centroid), int(metric), int(bool(spherical)), _ptr(cent, _c_f), _ptr(obj, _c_f),
        )
    )
    return cent, obj


# faiss::gpu::DistanceDataType / IndicesDataType (faiss/gpu/GpuDistance.h:18-29)
DistanceDataType_F32 = 1
DistanceDataType_F16 = 2
DistanceDataType_BF16 = 3
IndicesDataType_I64 = 1
IndicesDataType_I32 = 2


class GpuDistanceParams(ctypes.Structure):
    """FaissGpuDistanceParams of include/faiss_b200_c.h (faiss::gpu::GpuDistanceParams, faiss/gpu/GpuDistance.h:32-152)."""

    _fields_ = [
        ("metric", ctypes.c_int),
        ("metricArg", ctypes.c_float),
        ("k", ctypes.c_int),
        ("dims", ctypes.c_int),
        ("vectors", ctypes.c_void_p),
        ("vectorType", ctypes.c_int),
        ("vectorsRowMajor", ctypes.c_int),
        ("numVectors", ctypes.c_int64),
        ("queries", ctypes.c_void_p),
        ("queryType", ctypes.c_int),
        ("queriesRowMajor", ctypes.c_int),
        ("numQueries", ctypes.c_int64),
        ("outDistances", ctypes.c_void_p),
        ("outIndicesType", ctypes.c_int),
        ("outIndices", ctypes.c_void_p),
        ("device", ctypes.c_int),
    ]


def _distance_input(x):
    """(x as passed to the library, pointer, DistanceDataType, row-major?) of an [n, d] input.  numpy fp32 / fp16 and
    torch fp32 / fp16 / bf16 go as they are, in C order or (as column-major) F order; other numpy dtypes are converted
    to fp32, other strides made contiguous."""
    if _is_torch(x):
        import torch

        types = {torch.float32: DistanceDataType_F32, torch.float16: DistanceDataType_F16, torch.bfloat16: DistanceDataType_BF16}
        if x.dtype not in types:
            raise TypeError("knn_gpu: tensors must be float32, float16 or bfloat16 (got %s)" % x.dtype)
        assert x.dim() == 2, "inputs must be 2-D"
        if x.is_contiguous():
            return x, x.data_ptr(), types[x.dtype], True
        if x.t().is_contiguous():
            return x, x.data_ptr(), types[x.dtype], False
        x = x.contiguous()
        return x, x.data_ptr(), types[x.dtype], True
    x = np.asarray(x)
    if x.dtype not in (np.float32, np.float16):
        x = x.astype(np.float32)
    assert x.ndim == 2, "inputs must be 2-D"
    t = DistanceDataType_F32 if x.dtype == np.float32 else DistanceDataType_F16
    if x.flags["C_CONTIGUOUS"]:
        return x, x.ctypes.data, t, True
    if x.flags["F_CONTIGUOUS"]:
        return x, x.ctypes.data, t, False
    x = np.ascontiguousarray(x)
    return x, x.ctypes.data, t, True


def _addr(x):
    if x is None:
        return None
    return x.data_ptr() if _is_torch(x) else x.ctypes.data


def _is_cuda(x):
    return x is not None and _is_torch(x) and x.is_cuda


def _is_c_contiguous(x, dtypes):
    if _is_torch(x):
        return x.is_contiguous() and str(x.dtype).split(".")[-1] in dtypes
    return isinstance(x, np.ndarray) and x.flags["C_CONTIGUOUS"] and x.dtype.name in dtypes


def _distance_call(res, xq, xb, k, D, I, metric, device, metric_arg, vectorsMemoryLimit=0, queriesMemoryLimit=0, page_bytes=None):
    xq, qp, qt, qrm = _distance_input(xq)
    xb, bp, bt, brm = _distance_input(xb)
    nq, d = xq.shape
    assert xb.shape[1] == d, "xq and xb must have the same dimension"
    ncol = xb.shape[0] if k == -1 else k
    # the library writes nq * ncol entries through the raw pointer: a given output must have exactly that shape
    # (faiss/python/gpu_wrappers.py:160-169, 285)
    if D is not None and tuple(D.shape) != (nq, ncol):
        raise ValueError("D must have shape %s (got %s)" % ((nq, ncol), tuple(D.shape)))
    if k != -1 and I is not None and tuple(I.shape) != (nq, k):
        raise ValueError("I must have shape %s (got %s)" % ((nq, k), tuple(I.shape)))
    # outputs follow xq's residency unless given; a given output of another layout or dtype receives a copy
    outD = D if D is not None and _is_c_contiguous(D, ("float32",)) else _empty_like_residency(xq, (nq, ncol), np.float32)
    outI = None
    if k != -1:
        outI = I if I is not None and _is_c_contiguous(I, ("int64", "int32")) else _empty_like_residency(xq, (nq, k), np.int64)
        it = IndicesDataType_I32 if str(outI.dtype).split(".")[-1] == "int32" else IndicesDataType_I64
    else:
        it = IndicesDataType_I64
    p = GpuDistanceParams(
        int(metric), float(metric_arg), int(k), int(d), bp, bt, int(brm), int(xb.shape[0]), qp, qt, int(qrm), int(nq),
        _addr(outD), it, _addr(outI), int(device),
    )
    # CUDA tensors: order the work on torch's current stream, as the index classes do
    if any(_is_cuda(t) for t in (xq, xb, outD, outI)):
        import torch

        res.setDefaultStream(device, torch.cuda.current_stream(device).cuda_stream)
    if page_bytes is not None:
        check(lib.b200_pairwise_paged(res._h, ctypes.byref(p), ctypes.c_size_t(page_bytes)))
    elif vectorsMemoryLimit or queriesMemoryLimit:
        check(lib.faiss_b200_bfKnn_tiling(res._h, ctypes.byref(p), ctypes.c_size_t(vectorsMemoryLimit), ctypes.c_size_t(queriesMemoryLimit)))
    else:
        check(lib.faiss_b200_bfKnn_params(res._h, ctypes.byref(p)))
    if D is not None and outD is not D:
        D[...] = outD
        outD = D
    if k != -1 and I is not None and outI is not I:
        I[...] = outI
        outI = I
    return outD, outI


def knn_gpu(res, xq, xb, k, D=None, I=None, metric=METRIC_L2, device=0, metric_arg=0.0, vectorsMemoryLimit=0, queriesMemoryLimit=0):
    """faiss.knn_gpu (faiss/python/gpu_wrappers.py:60-200, GpuDistance.h:33-181): brute-force k-NN of xq [nq, d] in
    xb [nb, d]; returns (D [nq, k] float32, I [nq, k]).

    Inputs: numpy float32 / float16 in C or F order, torch float32 / float16 / bfloat16 (a tensor whose transpose is
    contiguous goes as column-major; other strides are made contiguous); xq and xb of the same dtype.  Host or CUDA.
    Outputs follow xq's residency unless D / I are given; I may be int64 or int32.  CUDA tensors run on torch's current
    stream.  vectorsMemoryLimit / queriesMemoryLimit: bfKnn_tiling (host-resident row-major inputs, byte budgets).
    Distances are GpuIndexFlat's, bit for bit."""
    assert k > 0, "k must be > 0 (pairwise_distance_gpu gives all distances)"
    return _distance_call(res, xq, xb, k, D, I, metric, device, metric_arg, vectorsMemoryLimit, queriesMemoryLimit)


def pairwise_distance_gpu(res, xq, xb, D=None, metric=METRIC_L2, device=0, metric_arg=0.0):
    """faiss.pairwise_distance_gpu (faiss/python/gpu_wrappers.py:203-310; bfKnn with k = -1): D [nq, nb] float32 with
    D[i, j] the distance of xq[i] to xb[j], the value knn_gpu returns for that pair, bit for bit (direct form, no
    ||x||^2 + ||y||^2 - 2<x, y> expansion; the raw inner product / Jaccard similarity; NaN as computed).  Inputs as for
    knn_gpu.  A host-resident D is computed in blocks of at most 256 MiB."""
    return _distance_call(res, xq, xb, -1, D, None, metric, device, metric_arg)[0]


def bfKnn(res, xq, xb, k, metric=METRIC_L2, device=0, metric_arg=0.0):
    """knn_gpu without preallocated outputs (faiss/gpu/GpuDistance.h:33-181)."""
    return knn_gpu(res, xq, xb, k, metric=metric, device=device, metric_arg=metric_arg)


def kmeans_sharded(res, x_local, k, niter=25, seed=1234, device=0):
    """Collective: k-means over the rows of ALL ranks of the device's NCCL communicator (this rank passes its own
    rows; rank order = row order).  Returns (centroids [k, d] identical on every rank, objective per iteration,
    stats dict)."""
    x_local = _as_f32(x_local)
    n, d = x_local.shape
    cent = np.empty((k, d), dtype=np.float32)
    obj = np.zeros(niter, dtype=np.float32)
    st = (ctypes.c_double * 4)()
    check(
        lib.faiss_b200_kmeans_sharded(
            res._h, int(device), ctypes.c_size_t(d), ctypes.c_size_t(n), ctypes.c_size_t(k), _ptr(x_local, _c_f), int(niter), int(seed),
            _ptr(cent, _c_f), _ptr(obj, _c_f), st,
        )
    )
    return cent, obj, {"total_s": st[0], "search_update_allreduce_s": st[1], "split_clusters_s": st[2], "nsplit": int(st[3])}


def pq_train(res, x, M, niter=25, seed=1234, device=0):
    """faiss::ProductQuantizer::train (M independent 256-centroid k-means); returns [M, 256, d/M]."""
    x = _as_f32(x)
    n, d = x.shape
    out = np.empty((M, 256, d // M), dtype=np.float32)
    check(
        lib.faiss_b200_pq_train(
            res._h, int(device), ctypes.c_size_t(d), ctypes.c_size_t(M), ctypes.c_size_t(n), _ptr(x, _c_f), int(niter), int(seed),
            _ptr(out, _c_f),
        )
    )
    return out


# ------------------------------------------------------------------ tier-2 seams (torch CUDA tensors)
def flat_search_exact(res, Y, Q, k, metric=METRIC_L2, device=0):
    import torch

    assert Y.is_cuda and Q.is_cuda
    res.setDefaultStream(device, torch.cuda.current_stream(device).cuda_stream)
    nq = Q.shape[0]
    D = torch.empty((nq, k), dtype=torch.float32, device=Q.device)
    I = torch.empty((nq, k), dtype=torch.int64, device=Q.device)
    check(
        lib.b200_flat_search_exact(
            res._h, int(device), _ptr(Y, _c_f), ctypes.c_int64(Y.shape[0]), int(Y.shape[1]), _ptr(Q, _c_f),
            ctypes.c_int64(nq), int(k), int(metric), _ptr(D, _c_f), _ptr(I, _c_i64),
        )
    )
    return D, I


def kmeans_accumulate(res, x, assign, k, device=0):
    """Per-centroid partial sums [k, d] and counts [k] of the CUDA rows `x` under `assign` (int64 [n]) --
    the device half of compute_centroids (faiss/impl/ClusteringHelpers.cpp:101-172); the caller
    all-reduces them across shards and divides."""
    import torch

    assert x.is_cuda and assign.is_cuda
    res.setDefaultStream(device, torch.cuda.current_stream(device).cuda_stream)
    n, d = x.shape
    sums = torch.zeros((k, d), dtype=torch.float32, device=x.device)
    counts = torch.zeros((k,), dtype=torch.float32, device=x.device)
    check(
        lib.b200_kmeans_update(
            res._h, int(device), _ptr(x, _c_f), _ptr(assign, _c_i64), ctypes.c_int64(n), int(d), ctypes.c_int64(k),
            _ptr(sums, _c_f), _ptr(counts, _c_f), None,
        )
    )
    return sums, counts


def rand_perm(n, seed):
    """faiss::rand_perm (faiss/utils/random.cpp:130-142), host."""
    perm = np.empty(int(n), dtype=np.int32)
    check(lib.faiss_b200_rand_perm(perm.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), ctypes.c_size_t(int(n)), ctypes.c_int64(int(seed))))
    return perm


def split_clusters(hassign, centroids, n):
    """faiss split_clusters (faiss/impl/ClusteringHelpers.cpp:177-240) in place on host arrays; returns nsplit."""
    k, d = centroids.shape
    assert hassign.dtype == np.float32 and centroids.dtype == np.float32
    ns = ctypes.c_int(0)
    fp = ctypes.POINTER(ctypes.c_float)
    check(
        lib.faiss_b200_split_clusters(
            ctypes.c_size_t(d), ctypes.c_size_t(k), ctypes.c_size_t(int(n)), hassign.ctypes.data_as(fp), centroids.ctypes.data_as(fp),
            ctypes.byref(ns),
        )
    )
    return ns.value


def topk_merge(res, D_in, I_in, k, metric=METRIC_L2, id_offsets=None, device=0):
    """D_in/I_in: CUDA tensors [nq, nshard, k_in] -> merged [nq, k] (role of merge_knn_results)."""
    import torch

    nq, nshard, kin = D_in.shape
    res.setDefaultStream(device, torch.cuda.current_stream(device).cuda_stream)
    D = torch.empty((nq, k), dtype=torch.float32, device=D_in.device)
    I = torch.empty((nq, k), dtype=torch.int64, device=D_in.device)
    check(
        lib.b200_topk_merge(
            res._h, int(device), _ptr(D_in, _c_f), _ptr(I_in, _c_i64), ctypes.c_int64(nq), int(nshard), int(kin),
            _ptr(id_offsets, _c_i64), int(k), int(metric), _ptr(D, _c_f), _ptr(I, _c_i64),
        )
    )
    return D, I


def flat_tc_scores_debug(res, Q16, Y16, device=0):
    """Raw tensor-core score matrix [nq, roundup(N,256)] (unit-test seam): fp16 rows, or int8 rows of 128 whose
    scores are the exact integer dot products."""
    import torch

    nq, dpad = Q16.shape
    N = Y16.shape[0]
    res.setDefaultStream(device, torch.cuda.current_stream(device).cuda_stream)
    npad = (N + 255) // 256 * 256
    S = torch.zeros((nq, npad), dtype=torch.float32, device=Q16.device)
    if Q16.dtype == torch.int8:
        check(
            lib.b200_flat_tc_scores_debug_s8(
                res._h, int(device), ctypes.c_void_p(Q16.data_ptr()), ctypes.c_int64(nq), ctypes.c_void_p(Y16.data_ptr()),
                ctypes.c_int64(N), _ptr(S, _c_f),
            )
        )
        return S
    check(
        lib.b200_flat_tc_scores_debug(
            res._h, int(device), ctypes.c_void_p(Q16.data_ptr()), ctypes.c_int64(nq), ctypes.c_void_p(Y16.data_ptr()),
            ctypes.c_int64(N), int(dpad), _ptr(S, _c_f),
        )
    )
    return S


_c_i32 = ctypes.POINTER(ctypes.c_int32)


def _as_i32(x):
    if _is_torch(x):
        import torch

        assert x.dtype == torch.int32
        return x.contiguous()
    return np.ascontiguousarray(x, dtype=np.int32)


class GpuIcmEncoder:
    """faiss::gpu::GpuIcmEncoder (faiss/gpu/GpuIcmEncoder.h): LocalSearchQuantizer's ICM encoding
    (lsq::IcmEncoder::encode, faiss/impl/LocalSearchQuantizer.cpp:539-795) on one or more devices.

    ``res`` is one StandardGpuResources per entry of ``devices``.  The perturbation draws are the caller's, an int32
    array [ils_iters, n, nperts, 2] of (m, k) in the order of LocalSearchQuantizer::perturb_codes; given the CPU's
    draws, the codes equal the CPU encoder's where fp32 is exact.  Limits: 1 <= K <= 1024, nperts <= M."""

    def __init__(self, M, K, d, res, devices=(0,)):
        if isinstance(res, StandardGpuResources):
            res = [res]
        devices = [int(v) for v in devices]
        assert len(res) == len(devices), "one StandardGpuResources per device"
        self.M, self.K, self.d = int(M), int(K), int(d)
        self._res = list(res)  # the handle keeps its own references; this keeps the Python objects alive too
        hs = (ctypes.c_void_p * len(res))(*[r._h.value for r in res])
        devs = (ctypes.c_int * len(devices))(*devices)
        self._h = ctypes.c_void_p()
        check(lib.faiss_GpuIcmEncoder_new(ctypes.byref(self._h), self.M, self.K, self.d, len(devices), hs, devs))

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_GpuIcmEncoder_free(self._h)
            self._h = None

    def setBinaryTerm(self, codebooks):
        """codebooks [M, K, d] (or [M * K, d]), numpy or torch"""
        cb = _as_f32(codebooks)
        size = cb.numel() if _is_torch(cb) else cb.size
        assert size == self.M * self.K * self.d, "codebooks must hold M * K * d floats"
        check(lib.faiss_GpuIcmEncoder_set_binary_term(self._h, _ptr(cb, _c_f)))

    def encode(self, codes, x, perturbations, icm_iters=4, page_bytes=None):
        """codes [n, M] int32 (start codes), x [n, d], perturbations [ils_iters, n, nperts, 2] int32 -> the best codes
        [n, M] int32, with the residency of ``codes``.  page_bytes: the page budget (default 256 MiB)."""
        x = _as_f32(x)
        codes = _as_i32(codes)
        pert = _as_i32(perturbations)
        n = int(x.shape[0])
        assert tuple(codes.shape) == (n, self.M) and tuple(x.shape) == (n, self.d)
        assert len(pert.shape) == 4 and int(pert.shape[1]) == n and int(pert.shape[3]) == 2, "perturbations [ils, n, nperts, 2]"
        ils, nperts = int(pert.shape[0]), int(pert.shape[2])
        out = codes.clone() if _is_torch(codes) else codes.copy()
        if _is_torch(out) and out.is_cuda:
            import torch

            torch.cuda.current_stream(out.device).synchronize()  # the clone is read on the resources' stream
        args = (self._h, _ptr(out, _c_i32), _ptr(x, _c_f), ctypes.c_int64(n), ctypes.c_size_t(ils), ctypes.c_size_t(nperts),
                ctypes.c_size_t(int(icm_iters)), _ptr(pert, _c_i32))
        if page_bytes is None:
            check(lib.faiss_GpuIcmEncoder_encode(*args))
        else:
            check(lib.b200_icm_encode_paged(*args, ctypes.c_size_t(int(page_bytes))))
        return out


# AdditiveQuantizer::Search_type_t (faiss/impl/AdditiveQuantizer.h:71-86)
ST_decompress, ST_LUT_nonorm, ST_norm_from_LUT, ST_norm_float, ST_norm_qint8, ST_norm_qint4 = range(6)
ST_norm_cqint8, ST_norm_cqint4, ST_norm_lsq2x4, ST_norm_rq2x4 = range(6, 10)


class GpuRqEncoder:
    """ResidualQuantizer's beam-search encoding (faiss/impl/ResidualQuantizer.cpp:432-520) on one device.

    ``nbits`` is one entry per codebook (1 <= nbits[m] <= 12); every beam is in [1, 256].  Inputs may be numpy arrays or
    torch tensors, host or device; outputs have the residency of the first array argument.  On integer-valued data and
    codebooks the results equal the CPU's bit for bit.  ``page_bytes`` overrides the 256 MiB page budget."""

    def __init__(self, d, nbits, res, device=0):
        self.d, self.nbits = int(d), [int(b) for b in nbits]
        self.M = len(self.nbits)
        self._res = res
        nb = (ctypes.c_int * self.M)(*self.nbits)
        self._h = ctypes.c_void_p()
        check(lib.faiss_b200_RqEncoder_new(ctypes.byref(self._h), res._h, int(device), self.d, self.M, nb))

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.faiss_b200_RqEncoder_free(self._h)
            self._h = None

    def setCodebooks(self, codebooks):
        """codebooks [total_K, d], numpy or torch, host or device"""
        cb = _as_f32(codebooks)
        size = cb.numel() if _is_torch(cb) else cb.size
        assert size == sum(1 << b for b in self.nbits) * self.d, "codebooks must hold total_K * d floats"
        check(lib.faiss_b200_RqEncoder_set_codebooks(self._h, _ptr(cb, _c_f)))

    def finalBeam(self, beam_in, out_beam):
        b = ctypes.c_int()
        check(lib.faiss_b200_RqEncoder_final_beam(self._h, int(beam_in), int(out_beam), ctypes.byref(b)))
        return b.value

    def refineBeam(self, residuals, out_beam, page_bytes=None):
        """ResidualQuantizer::refine_beam: residuals [n, beam_in, d] -> (codes [n, B, M] int32, residuals [n, B, d],
        distances [n, B])"""
        r = _as_f32(residuals)
        n, beam_in = int(r.shape[0]), int(r.shape[1])
        assert len(r.shape) == 3 and int(r.shape[2]) == self.d, "residuals [n, beam_in, d]"
        B = self.finalBeam(beam_in, out_beam)
        codes = _empty_like_residency(r, (n, B, self.M), np.int32)
        ro = _empty_like_residency(r, (n, B, self.d), np.float32)
        dis = _empty_like_residency(r, (n, B), np.float32)
        args = (self._h, ctypes.c_int64(n), int(beam_in), _ptr(r, _c_f), int(out_beam), _ptr(codes, _c_i32), _ptr(ro, _c_f),
                _ptr(dis, _c_f))
        if page_bytes is None:
            check(lib.faiss_b200_RqEncoder_refine_beam(*args))
        else:
            check(lib.b200_rq_refine_beam_paged(*args, ctypes.c_size_t(int(page_bytes))))
        return codes, ro, dis

    def refineBeamLUT(self, x, out_beam, page_bytes=None):
        """ResidualQuantizer::refine_beam_LUT from x [n, d] (the device makes ‖x‖² and x·Cᵀ) -> (codes [n, B, M] int32,
        distances [n, B])"""
        x = _as_f32(x)
        n = int(x.shape[0])
        assert tuple(x.shape) == (n, self.d)
        B = self.finalBeam(1, out_beam)
        codes = _empty_like_residency(x, (n, B, self.M), np.int32)
        dis = _empty_like_residency(x, (n, B), np.float32)
        args = (self._h, ctypes.c_int64(n), _ptr(x, _c_f), int(out_beam), _ptr(codes, _c_i32), _ptr(dis, _c_f))
        if page_bytes is None:
            check(lib.faiss_b200_RqEncoder_refine_beam_lut(*args))
        else:
            check(lib.b200_rq_refine_beam_lut_paged(*args, ctypes.c_size_t(int(page_bytes))))
        return codes, dis

    def codeSize(self, search_type=ST_decompress):
        norm_bits = {ST_norm_float: 32, ST_norm_qint8: 8, ST_norm_qint4: 4, ST_norm_cqint8: 8, ST_norm_cqint4: 4,
                     ST_norm_lsq2x4: 8, ST_norm_rq2x4: 8}.get(search_type, 0)
        return (sum(self.nbits) + norm_bits + 7) // 8

    def computeCodes(self, x, use_beam_LUT=0, max_beam_size=5, search_type=ST_decompress, norm_min=0.0, norm_max=0.0,
                     centroids=None, page_bytes=None):
        """ResidualQuantizer::compute_codes_add_centroids -> packed codes [n, code_size] uint8"""
        x = _as_f32(x)
        n = int(x.shape[0])
        assert tuple(x.shape) == (n, self.d)
        cen = None if centroids is None else _as_f32(centroids)
        out = _empty_like_residency(x, (n, self.codeSize(search_type)), np.uint8)
        args = (self._h, _ptr(x, _c_f), ctypes.c_int64(n), int(bool(use_beam_LUT)), int(max_beam_size), int(search_type),
                ctypes.c_float(norm_min), ctypes.c_float(norm_max), _ptr(cen, _c_f), _ptr(out, _c_u8))
        if page_bytes is None:
            check(lib.faiss_b200_RqEncoder_compute_codes(*args))
        else:
            check(lib.b200_rq_compute_codes_paged(*args, ctypes.c_size_t(int(page_bytes))))
        return out

    def encodeUnpacked(self, x, use_beam_LUT=0, max_beam_size=5):
        """the compute_codes search, unpacked -> codes [n, M] int32 (entry 0 of the beam)"""
        x = _as_f32(x)
        n = int(x.shape[0])
        codes = _empty_like_residency(x, (n, self.M), np.int32)
        check(lib.faiss_b200_RqEncoder_encode_unpacked(self._h, _ptr(x, _c_f), ctypes.c_int64(n), int(bool(use_beam_LUT)),
                                                       int(max_beam_size), _ptr(codes, _c_i32)))
        return codes
