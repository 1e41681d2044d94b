// faiss_b200 -- host driver of bfKnn / bfKnn_tiling / all-pairs distances (distance.h), and the two small kernels it
// needs: input widening / transposition to fp32 row-major, and int64 -> int32 ids.
#include "distance.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <climits>
#include <vector>

#include "index.h"
#include "kernels.h"

namespace fb200 {

namespace {

__device__ __forceinline__ float widen(float v) {
    return v;
}
__device__ __forceinline__ float widen(__half v) {
    return __half2float(v);
}
__device__ __forceinline__ float widen(__nv_bfloat16 v) {
    return __bfloat162float(v);
}

// [n, d] of T, row-major (row r at src + r * ld) or column-major (column c at src + c * ld) -> fp32 row-major [n][d],
// through a 32 x 32 shared-memory tile so that both the reads (along the source's inner dimension) and the writes
// (along d) are coalesced.  Widening fp16 / bf16 to fp32 is exact.
constexpr int kTile = 32;
template <typename T, bool COL>
__global__ void __launch_bounds__(256) to_f32_rows_kernel(const T* __restrict__ src, int64_t n, int d, int64_t ld, float* __restrict__ out) {
    __shared__ float tile[kTile][kTile + 1]; // [row][col]
    const int64_t r0 = (int64_t)blockIdx.x * kTile;
    const int c0 = blockIdx.y * kTile;
    const int tx = threadIdx.x, ty = threadIdx.y; // 32 x 8
#pragma unroll
    for (int j = ty; j < kTile; j += 8) {
        if (COL) {
            const int64_t r = r0 + tx;
            const int c = c0 + j;
            if (r < n && c < d)
                tile[tx][j] = widen(src[(int64_t)c * ld + r]);
        } else {
            const int64_t r = r0 + j;
            const int c = c0 + tx;
            if (r < n && c < d)
                tile[j][tx] = widen(src[r * ld + c]);
        }
    }
    __syncthreads();
#pragma unroll
    for (int j = ty; j < kTile; j += 8) {
        const int64_t r = r0 + j;
        const int c = c0 + tx;
        if (r < n && c < d)
            out[r * d + c] = tile[j][tx];
    }
}

size_t elemSize(DistanceDataType t) {
    return t == DistanceDataType::F32 ? 4 : 2;
}

// src: device pointer on the current device; ld as for to_f32_rows_kernel
void runToF32Rows(const void* src, DistanceDataType t, bool rowMajor, int64_t n, int d, int64_t ld, float* out, cudaStream_t stream) {
    if (n == 0)
        return;
    FB_THROW_IF_NOT(ceil_div(d, kTile) <= 65535);
    const dim3 grid((unsigned)ceil_div(n, kTile), (unsigned)ceil_div(d, kTile)), block(kTile, 8);
    auto launch = [&](auto tag) {
        using T = decltype(tag);
        const T* s = reinterpret_cast<const T*>(src);
        if (rowMajor)
            to_f32_rows_kernel<T, false><<<grid, block, 0, stream>>>(s, n, d, ld, out);
        else
            to_f32_rows_kernel<T, true><<<grid, block, 0, stream>>>(s, n, d, ld, out);
    };
    switch (t) {
        case DistanceDataType::F32:
            launch(float{});
            break;
        case DistanceDataType::F16:
            launch(__half{});
            break;
        case DistanceDataType::BF16:
            launch(__nv_bfloat16{});
            break;
    }
    CUDA_CHECK_LAST();
}

__global__ void ids_to_i32_kernel(const idx_t* __restrict__ in, int64_t n, int32_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (int32_t)in[i]; // ids < numVectors <= INT32_MAX, or -1
}

void runIdsToI32(const idx_t* in, int64_t n, int32_t* out, cudaStream_t stream) {
    if (n == 0)
        return;
    ids_to_i32_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n, 256), 65535 * 16), 256, 0, stream>>>(in, n, out);
    CUDA_CHECK_LAST();
}

bool isPlainF32(DistanceDataType t, bool rowMajor) {
    return t == DistanceDataType::F32 && rowMajor;
}

// Inputs that are not resident on the device are converted in pages of at most this many fp32 bytes, so that the raw
// copy in temporary memory stays one page (and k-NN holds one page of converted queries at a time).
constexpr size_t kConvertPageBytes = size_t(256) << 20;

idx_t convertPageRows(int d) {
    return std::max<idx_t>(1, (idx_t)(kConvertPageBytes / (sizeof(float) * d)));
}

// rows [i0, i0 + nb) of the [n, d] input p (layout t / rowMajor) -> fp32 row-major out [nb][d] on `device`
void convertRows(
        GpuResources* res,
        int device,
        const void* p,
        DistanceDataType t,
        bool rowMajor,
        idx_t n,
        idx_t i0,
        idx_t nb,
        int d,
        float* out,
        cudaStream_t stream) {
    if (nb == 0)
        return;
    const size_t es = elemSize(t);
    const char* base = reinterpret_cast<const char*>(p);
    if (getDeviceForAddress(p) == device) {
        runToF32Rows(base + (rowMajor ? i0 * d : i0) * es, t, rowMajor, nb, d, rowMajor ? d : n, out, stream);
        return;
    }
    // the raw rows first, in their own layout: one copy (row-major) or a 2-D copy of a column range (column-major)
    auto raw = res->temp(device, (size_t)nb * d * es);
    if (rowMajor)
        CUDA_VERIFY(cudaMemcpyAsync(raw.data, base + (size_t)i0 * d * es, (size_t)nb * d * es, cudaMemcpyDefault, stream));
    else
        CUDA_VERIFY(cudaMemcpy2DAsync(raw.data, nb * es, base + i0 * es, n * es, nb * es, d, cudaMemcpyDefault, stream));
    runToF32Rows(raw.data, t, rowMajor, nb, d, rowMajor ? d : nb, out, stream);
}

// all of rows [i0, i0 + nb) of p (an [n, d] input) into `out`, page by page when p is not on the device
void convertRowsPaged(
        GpuResources* res,
        int device,
        const void* p,
        DistanceDataType t,
        bool rowMajor,
        idx_t n,
        idx_t i0,
        idx_t nb,
        int d,
        float* out,
        cudaStream_t stream) {
    const idx_t page = getDeviceForAddress(p) == device ? std::max<idx_t>(nb, 1) : convertPageRows(d);
    for (idx_t r = 0; r < nb; r += page) {
        InterruptCallback::check(); // between pages
        convertRows(res, device, p, t, rowMajor, n, i0 + r, std::min(page, nb - r), d, out + (size_t)r * d, stream);
    }
}

// rows [i0, i0 + nb) of the [n, d] input p as fp32 row-major on `device`: the input itself when it already is that and
// is resident there, else a copy or conversion into `hold`
const float* deviceRows(
        GpuResources* res,
        int device,
        const void* p,
        DistanceDataType t,
        bool rowMajor,
        idx_t n,
        idx_t i0,
        idx_t nb,
        int d,
        GpuMemoryReservation& hold,
        cudaStream_t stream) {
    const size_t count = (size_t)nb * d;
    if (count == 0)
        return nullptr;
    if (isPlainF32(t, rowMajor)) {
        DeviceView<float> v(res, device, reinterpret_cast<const float*>(p) + (size_t)i0 * d, count, stream);
        hold = std::move(v.hold);
        return v.ptr;
    }
    hold = res->temp(device, sizeof(float) * count);
    convertRowsPaged(res, device, p, t, rowMajor, n, i0, nb, d, hold.as<float>(), stream);
    return hold.as<float>();
}

// the k-NN results of a search with int64 ids, written to `out` as the requested id type
struct IdsOut {
    IdsOut(GpuResources* res, int device, IndicesDataType t, void* out, size_t count) : res_(res), device_(device), out_(out), n_(count) {
        if (t == IndicesDataType::I64) {
            ids = reinterpret_cast<idx_t*>(out);
        } else {
            wide_ = res->temp(device, sizeof(idx_t) * count);
            ids = wide_.as<idx_t>();
        }
    }
    // after the search: narrow to int32 on the device, then copy out if `out` is not on the device
    void finish(cudaStream_t stream) {
        if (!wide_.data)
            return;
        DeviceOut<int32_t> o(res_, device_, reinterpret_cast<int32_t*>(out_), n_);
        runIdsToI32(ids, (int64_t)n_, o.ptr, stream);
        o.finish(stream);
        if (o.staged)
            CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
    idx_t* ids;

   private:
    GpuResources* res_;
    int device_;
    void* out_;
    size_t n_;
    GpuMemoryReservation wide_;
};

void knnImpl(const std::shared_ptr<GpuResources>& res, const GpuDistanceParams& a) {
    const int device = a.device;
    auto stream = res->getDefaultStream(device);
    GpuIndexFlatConfig cfg;
    cfg.device = device;
    GpuIndexFlat index(res, a.dims, a.metric, cfg);
    index.metric_arg = a.metricArg;
    if (isPlainF32(a.vectorType, a.vectorsRowMajor)) {
        index.add(a.numVectors, reinterpret_cast<const float*>(a.vectors));
    } else if (a.numVectors > 0) {
        // converted straight into the index's storage: no second copy of the vectors
        float* rows = index.resizeVectorsDevice(a.numVectors);
        convertRowsPaged(res.get(), device, a.vectors, a.vectorType, a.vectorsRowMajor, a.numVectors, 0, a.numVectors, a.dims, rows, stream);
    }
    if (a.numQueries == 0)
        return;
    // fp32 row-major queries keep GpuIndex::search's own residency handling (host query paging); other queries are
    // converted on the device, one page at a time when they are not resident there
    const bool plain = isPlainF32(a.queryType, a.queriesRowMajor);
    const idx_t page =
            plain || getDeviceForAddress(a.queries) == device ? a.numQueries : convertPageRows(a.dims);
    const size_t idBytes = a.outIndicesType == IndicesDataType::I64 ? sizeof(idx_t) : sizeof(int32_t);
    for (idx_t i0 = 0; i0 < a.numQueries; i0 += page) {
        const idx_t nb = std::min(page, a.numQueries - i0);
        GpuMemoryReservation qHold;
        const float* q = plain ? reinterpret_cast<const float*>(a.queries) + (size_t)i0 * a.dims
                               : deviceRows(res.get(), device, a.queries, a.queryType, a.queriesRowMajor, a.numQueries, i0, nb, a.dims, qHold, stream);
        IdsOut ids(res.get(), device, a.outIndicesType, reinterpret_cast<char*>(a.outIndices) + idBytes * a.k * i0, (size_t)nb * a.k);
        index.search(nb, q, a.k, a.outDistances + (size_t)a.k * i0, ids.ids);
        ids.finish(stream);
    }
}

// the all-pairs matrix into a host (or other device's) D: blocks of whole rows when 32 of them fit the budget, else
// 32 rows x a column range; two device buffers alternate so that a block's copy-out overlaps the next block's kernel
void pairwisePaged(
        GpuResources* res,
        int device,
        const float* Q,
        idx_t nq,
        const float* Y,
        idx_t n,
        int d,
        MetricType metric,
        float metricArg,
        float* D,
        size_t pageBytes,
        cudaStream_t stream) {
    const int64_t rowBytes = (int64_t)n * sizeof(float);
    int64_t rb, cb;
    if ((int64_t)pageBytes / rowBytes >= std::min<int64_t>(nq, 32)) {
        rb = std::min<int64_t>(nq, (int64_t)pageBytes / rowBytes);
        cb = n;
    } else {
        rb = std::min<int64_t>(nq, 32);
        cb = std::max<int64_t>(64, (int64_t)pageBytes / (rb * (int64_t)sizeof(float)) / 64 * 64);
        cb = std::min<int64_t>(cb, n);
    }
    auto copyStream = res->getAsyncCopyStream(device);
    GpuMemoryReservation buf[2] = {res->temp(device, sizeof(float) * rb * cb), res->temp(device, sizeof(float) * rb * cb)};
    struct Events {
        cudaEvent_t computed[2] = {nullptr, nullptr}, copied[2] = {nullptr, nullptr};
        cudaStream_t stream, copyStream;
        ~Events() { // also on an interrupt: no copy may still read a buffer that is released
            cudaStreamSynchronize(copyStream);
            for (auto* es : {computed, copied})
                for (int b = 0; b < 2; b++)
                    if (es[b])
                        cudaEventDestroy(es[b]);
        }
    } ev;
    ev.stream = stream;
    ev.copyStream = copyStream;
    for (int b = 0; b < 2; b++) {
        CUDA_VERIFY(cudaEventCreateWithFlags(&ev.computed[b], cudaEventDisableTiming));
        CUDA_VERIFY(cudaEventCreateWithFlags(&ev.copied[b], cudaEventDisableTiming));
    }
    struct Block {
        int64_t i0, j0, nr, nc;
    };
    // the copy of block p is issued after block p + 1's kernel has been queued: a copy to pageable memory returns
    // only when it is done, and the kernel then runs meanwhile
    auto copyOut = [&](const Block& blk, int b) {
        CUDA_VERIFY(cudaStreamWaitEvent(copyStream, ev.computed[b], 0));
        CUDA_VERIFY(cudaMemcpy2DAsync(
                D + blk.i0 * n + blk.j0, sizeof(float) * n, buf[b].data, sizeof(float) * blk.nc, sizeof(float) * blk.nc,
                blk.nr, cudaMemcpyDefault, copyStream));
        CUDA_VERIFY(cudaEventRecord(ev.copied[b], copyStream));
    };
    Block prev{};
    int64_t p = 0;
    for (int64_t i0 = 0; i0 < nq; i0 += rb) {
        for (int64_t j0 = 0; j0 < n; j0 += cb, p++) {
            InterruptCallback::check(); // between blocks
            const int b = (int)(p & 1);
            const Block blk{i0, j0, std::min(rb, nq - i0), std::min(cb, n - j0)};
            if (p >= 2)
                CUDA_VERIFY(cudaStreamWaitEvent(stream, ev.copied[b], 0));
            runFlatPairwise(res, device, Q + i0 * d, blk.nr, Y + j0 * d, blk.nc, d, metric, metricArg, buf[b].as<float>(), blk.nc, stream);
            CUDA_VERIFY(cudaEventRecord(ev.computed[b], stream));
            if (p >= 1)
                copyOut(prev, 1 - b);
            prev = blk;
        }
    }
    if (p >= 1)
        copyOut(prev, (int)((p - 1) & 1));
    // the buffers go back to the default stream's temp memory: order their release after the copies
    for (int b = 0; b < 2 && b < p; b++)
        CUDA_VERIFY(cudaStreamWaitEvent(stream, ev.copied[b], 0));
    CUDA_VERIFY(cudaStreamSynchronize(copyStream));
}

void pairwiseImpl(const std::shared_ptr<GpuResources>& res, const GpuDistanceParams& a, size_t pageBytes) {
    const int device = a.device;
    auto stream = res->getDefaultStream(device);
    if (a.numQueries == 0 || a.numVectors == 0)
        return;
    const MetricType metric = flatKernelMetric(a.metric, a.metricArg);
    GpuMemoryReservation qHold, yHold; // released in reverse order: temp memory is a stack
    const float* Q = deviceRows(res.get(), device, a.queries, a.queryType, a.queriesRowMajor, a.numQueries, 0, a.numQueries, a.dims, qHold, stream);
    const float* Y = deviceRows(res.get(), device, a.vectors, a.vectorType, a.vectorsRowMajor, a.numVectors, 0, a.numVectors, a.dims, yHold, stream);
    if (getDeviceForAddress(a.outDistances) == device) {
        runFlatPairwise(res.get(), device, Q, a.numQueries, Y, a.numVectors, a.dims, metric, a.metricArg, a.outDistances, a.numVectors, stream);
        return;
    }
    pairwisePaged(res.get(), device, Q, a.numQueries, Y, a.numVectors, a.dims, metric, a.metricArg, a.outDistances, pageBytes, stream);
}

bool validType(DistanceDataType t) {
    return t == DistanceDataType::F32 || t == DistanceDataType::F16 || t == DistanceDataType::BF16;
}

} // namespace

void validateDistanceParams(const GpuDistanceParams& a) {
    FB_THROW_IF_NOT_FMT(is_implemented_metric(a.metric), "bfKnn: unimplemented metric type %d", (int)a.metric);
    FB_THROW_IF_NOT_FMT(
            a.k == -1 || (a.k > 0 && a.k <= kMaxK),
            "bfKnn: k must be -1 (all pairwise distances) or in [1, %d] (requested %d)", kMaxK, a.k);
    FB_THROW_IF_NOT_MSG(a.dims > 0, "bfKnn: dims must be > 0");
    FB_THROW_IF_NOT_MSG(a.numVectors >= 0 && a.numQueries >= 0, "bfKnn: negative numVectors / numQueries");
    FB_THROW_IF_NOT_MSG(validType(a.vectorType) && validType(a.queryType), "bfKnn: unknown vectorType / queryType");
    // faiss/gpu/GpuDistance.cu:246-248
    FB_THROW_IF_NOT_MSG(a.vectorType == a.queryType, "bfKnn: vectorType and queryType must be the same");
    FB_THROW_IF_NOT_MSG(a.numVectors == 0 || a.vectors, "bfKnn: vectors must be provided (passed null)");
    FB_THROW_IF_NOT_MSG(a.numQueries == 0 || a.queries, "bfKnn: queries must be provided (passed null)");
    FB_THROW_IF_NOT_MSG(a.numQueries == 0 || a.outDistances, "bfKnn: outDistances must be provided (passed null)");
    FB_THROW_IF_NOT_MSG(a.device >= 0, "bfKnn: device must be a device ordinal");
    if (a.k > 0) {
        FB_THROW_IF_NOT_MSG(
                a.outIndicesType == IndicesDataType::I64 || a.outIndicesType == IndicesDataType::I32,
                "bfKnn: unknown outIndicesType");
        FB_THROW_IF_NOT_MSG(a.numQueries == 0 || a.outIndices, "bfKnn: outIndices must be provided (passed null)");
        // the reference narrows silently; an id that does not fit is an error here
        FB_THROW_IF_NOT_MSG(
                a.outIndicesType != IndicesDataType::I32 || a.numVectors <= INT32_MAX,
                "bfKnn: int32 indices cannot address more than INT32_MAX vectors");
    } else {
        FB_THROW_IF_NOT_MSG(a.numQueries < (idx_t(1) << 31), "bfKnn: too many queries for all pairwise distances");
    }
}

void bfKnn(const std::shared_ptr<GpuResources>& res, const GpuDistanceParams& a, size_t pairwisePageBytes) {
    validateDistanceParams(a);
    FB_THROW_IF_NOT_MSG(pairwisePageBytes > 0, "bfKnn: the pairwise block budget must be > 0");
    DeviceScope scope(a.device);
    if (a.k == -1)
        pairwiseImpl(res, a, pairwisePageBytes);
    else
        knnImpl(res, a);
}

namespace {

// faiss/gpu/GpuDistance.cu:457-511 (bfKnn_single_query_shard), with the shards merged on the device
void bfKnnVectorShards(const std::shared_ptr<GpuResources>& res, const GpuDistanceParams& a, size_t vectorsMemoryLimit) {
    if (vectorsMemoryLimit == 0) {
        bfKnn(res, a);
        return;
    }
    FB_THROW_IF_NOT_MSG(a.numVectors > 0, "bfKnn_tiling: numVectors must be > 0");
    FB_THROW_IF_NOT_MSG(a.vectors, "bfKnn_tiling: vectors must be provided (passed null)");
    FB_THROW_IF_NOT_MSG(
            getDeviceForAddress(a.vectors) == -1,
            "bfKnn_tiling: vectors should be in CPU memory when vectorsMemoryLimit > 0");
    FB_THROW_IF_NOT_MSG(a.vectorsRowMajor, "bfKnn_tiling: tiling vectors is only supported in row major mode");
    FB_THROW_IF_NOT_MSG(a.k > 0, "bfKnn_tiling: tiling vectors is only supported for k > 0");
    const size_t es = elemSize(a.vectorType);
    const idx_t shard = (idx_t)(vectorsMemoryLimit / ((size_t)a.dims * es));
    FB_THROW_IF_NOT_MSG(shard > 0, "bfKnn_tiling: vectorsMemoryLimit is too low");
    if (a.numVectors <= shard) {
        bfKnn(res, a);
        return;
    }
    const int device = a.device;
    DeviceScope scope(device);
    auto stream = res->getDefaultStream(device);
    const idx_t nq = a.numQueries, nsh = ceil_div(a.numVectors, shard);
    const size_t per = (size_t)nq * a.k;
    // [2][nq][k]: the running top-k (global ids) and the shard just searched (ids local to the shard).  Merging after
    // every shard keeps device memory at three [nq][k] slabs whatever the number of shards.
    auto partD = res->temp(device, sizeof(float) * per * 2);
    auto partI = res->temp(device, sizeof(idx_t) * per * 2);
    auto mergedD = res->temp(device, sizeof(float) * per);
    auto mergedI = res->temp(device, sizeof(idx_t) * per);
    std::vector<idx_t> offsets(2 * nsh); // merge s: {0, first id of shard s}
    for (idx_t s = 0; s < nsh; s++) {
        offsets[2 * s] = 0;
        offsets[2 * s + 1] = s * shard;
    }
    DeviceView<idx_t> offs(res.get(), device, offsets.data(), offsets.size(), stream);
    DeviceOut<float> dOut(res.get(), device, a.outDistances, per);
    IdsOut ids(res.get(), device, a.outIndicesType, a.outIndices, per);
    DeviceOut<idx_t> iOut(res.get(), device, ids.ids, per);
    for (idx_t s = 0; s < nsh; s++) {
        const int slab = s == 0 ? 0 : 1;
        GpuDistanceParams b = a;
        b.vectors = reinterpret_cast<const char*>(a.vectors) + es * a.dims * (s * shard);
        b.numVectors = std::min(shard, a.numVectors - s * shard);
        b.outDistances = partD.as<float>() + per * slab;
        b.outIndices = partI.as<idx_t>() + per * slab;
        b.outIndicesType = IndicesDataType::I64;
        bfKnn(res, b);
        if (s == 0)
            continue;
        // shards in id order, (distance, id) order within the merge: the untiled result, bit for bit
        const bool last = s == nsh - 1;
        float* mD = last ? dOut.ptr : mergedD.as<float>();
        idx_t* mI = last ? iOut.ptr : mergedI.as<idx_t>();
        runMergeTopKListMajor(partD.as<float>(), partI.as<idx_t>(), nq, 2, a.k, offs.ptr + 2 * s, a.k, a.metric, mD, mI, stream);
        if (!last) {
            CUDA_VERIFY(cudaMemcpyAsync(partD.data, mD, sizeof(float) * per, cudaMemcpyDeviceToDevice, stream));
            CUDA_VERIFY(cudaMemcpyAsync(partI.data, mI, sizeof(idx_t) * per, cudaMemcpyDeviceToDevice, stream));
        }
    }
    dOut.finish(stream);
    iOut.finish(stream);
    ids.finish(stream);
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

} // namespace

// faiss/gpu/GpuDistance.cu:513-570
void bfKnn_tiling(
        const std::shared_ptr<GpuResources>& res,
        const GpuDistanceParams& a,
        size_t vectorsMemoryLimit,
        size_t queriesMemoryLimit) {
    validateDistanceParams(a);
    if (queriesMemoryLimit == 0) {
        bfKnnVectorShards(res, a, vectorsMemoryLimit);
        return;
    }
    FB_THROW_IF_NOT_MSG(a.numQueries > 0, "bfKnn_tiling: numQueries must be > 0");
    FB_THROW_IF_NOT_MSG(a.queries, "bfKnn_tiling: queries must be provided (passed null)");
    FB_THROW_IF_NOT_MSG(
            getDeviceForAddress(a.queries) == -1,
            "bfKnn_tiling: queries should be in CPU memory when queriesMemoryLimit > 0");
    FB_THROW_IF_NOT_MSG(a.queriesRowMajor, "bfKnn_tiling: tiling queries is only supported in row major mode");
    FB_THROW_IF_NOT_MSG(a.k > 0, "bfKnn_tiling: tiling queries is only supported for k > 0");
    const size_t es = elemSize(a.queryType);
    const size_t ls = a.outIndicesType == IndicesDataType::I64 ? 8 : 4;
    const idx_t shard = (idx_t)(queriesMemoryLimit / ((size_t)a.k * (es + ls) + (size_t)a.dims * es));
    FB_THROW_IF_NOT_MSG(shard > 0, "bfKnn_tiling: queriesMemoryLimit is too low");
    for (idx_t i = 0; i < a.numQueries; i += shard) {
        GpuDistanceParams b = a;
        b.numQueries = std::min(shard, a.numQueries - i);
        b.queries = reinterpret_cast<const char*>(a.queries) + es * a.dims * i;
        b.outDistances = a.outDistances + (size_t)a.k * i;
        b.outIndices = reinterpret_cast<char*>(a.outIndices) + (size_t)a.k * ls * i;
        bfKnnVectorShards(res, b, vectorsMemoryLimit);
    }
}

} // namespace fb200
