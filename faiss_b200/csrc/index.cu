// faiss_b200 -- host-side index objects.  See index.h for the reference map.
#include "index.h"

#include "comm.h"
#include "ivf_layout.cuh"

#include <algorithm>
#include <cfloat>
#include <chrono>
#include <condition_variable>
#include <cmath>
#include <cstring>
#include <future>
#include <mutex>
#include <numeric>
#include <random>
#include <thread>

namespace fb200 {

// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------
namespace {

double now_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// faiss/gpu/impl/IndexUtils.cu:21-43
void validateKSelect(idx_t k) {
    FB_THROW_IF_NOT_FMT(
            k > 0 && k <= kMaxK,
            "GPU index only supports min/max-K selection up to %d (requested %d)",
            kMaxK,
            (int)k);
}
void validateNProbe(size_t nprobe) {
    FB_THROW_IF_NOT_FMT(
            nprobe > 0 && nprobe <= (size_t)kMaxNprobe,
            "GPU IVF index only supports nprobe selection up to %d (requested %zu)",
            kMaxNprobe,
            nprobe);
}

__global__ void iota_ids_kernel(idx_t* out, idx_t n, idx_t base) {
    idx_t i = (idx_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        out[i] = base + i;
}
// fp32 -> fp16 (round to nearest even), written as fp16 and / or widened back to fp32 (GpuIndexFlat useFloat16)
__global__ void float_to_half_kernel(const float* __restrict__ x, __half* __restrict__ out16, float* __restrict__ out32, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const __half h = __float2half_rn(x[i]);
        if (out16)
            out16[i] = h;
        if (out32)
            out32[i] = __half2float(h);
    }
}
__global__ void half_to_float_kernel(const __half* __restrict__ x, float* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = __half2float(x[i]);
}

__global__ void slice_cols_kernel(const float* x, int64_t n, int d, int c0, int dsub, float* out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * dsub) {
        int64_t r = i / dsub;
        int j = (int)(i - r * dsub);
        out[i] = x[r * d + c0 + j];
    }
}
__global__ void gather_rows_int_kernel(const float* src, const int* idx, int64_t n, int d, float* out) {
    int64_t i = blockIdx.x;
    int64_t a = idx[i];
    for (int j = threadIdx.x; j < d; j += blockDim.x)
        out[i * d + j] = src[a * d + j];
}
__global__ void sum_kernel(const float* x, int64_t n, double* out) {
    double acc = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        acc += x[i];
    for (int o = 16; o > 0; o >>= 1)
        acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0)
        atomicAdd(out, acc);
}
__global__ void copy_lists_kernel(
        const uint8_t* srcCodes,
        const idx_t* srcIds,
        const int64_t* srcStart,
        const int* len,
        const int64_t* dstStart,
        int codeSize,
        int group, // codes are copied in whole groups (32 for the interleaved PQ layout)
        uint8_t* dstCodes,
        idx_t* dstIds) {
    const int l = blockIdx.x;
    const int64_t n = len[l];
    const uint8_t* s = srcCodes + srcStart[l] * codeSize;
    uint8_t* t = dstCodes + dstStart[l] * codeSize;
    const int64_t bytes = ((n + group - 1) / group) * group * codeSize;
    if ((codeSize & 15) == 0) {
        for (int64_t i = threadIdx.x; i < (bytes >> 4); i += blockDim.x)
            reinterpret_cast<uint4*>(t)[i] = reinterpret_cast<const uint4*>(s)[i];
    } else {
        for (int64_t i = threadIdx.x; i < bytes; i += blockDim.x)
            t[i] = s[i];
    }
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x)
        dstIds[dstStart[l] + i] = srcIds[srcStart[l] + i];
}

// an output that may live on the host and whose rows are only partly written: the device staging starts as a copy
// of the caller's contents
template <typename T>
struct DeviceInOut : DeviceOut<T> {
    DeviceInOut(GpuResources* res, int device, T* p, size_t count, cudaStream_t stream) : DeviceOut<T>(res, device, p, count) {
        if (this->staged)
            CUDA_VERIFY(cudaMemcpyAsync(this->ptr, p, count * sizeof(T), cudaMemcpyDefault, stream));
    }
};

// outputs of a retrieval call are staged per page of at most this many bytes
constexpr size_t kRetrievalPageBytes = size_t(256) << 20;

} // namespace

// ------------------------------------------------------------------------------------------
// Index defaults
// ------------------------------------------------------------------------------------------
void Index::add_with_ids(idx_t, const float*, const idx_t*) {
    FB_THROW_MSG("add_with_ids not implemented for this type of index");
}
void Index::assign(idx_t n, const float* x, idx_t* labels, idx_t k) const {
    std::vector<float> dis((size_t)n * k);
    search(n, x, k, dis.data(), labels);
}
void Index::reconstruct(idx_t, float*) const {
    FB_THROW_MSG("reconstruct not implemented for this type of index");
}
void Index::reconstruct_batch(idx_t n, const idx_t* keys, float* recons) const {
    for (idx_t i = 0; i < n; i++)
        reconstruct(keys[i], recons + (size_t)i * d);
}
void Index::reconstruct_n(idx_t i0, idx_t ni, float* recons) const {
    for (idx_t i = 0; i < ni; i++)
        reconstruct(i0 + i, recons + (size_t)i * d);
}
void Index::search_and_reconstruct(idx_t, const float*, idx_t, float*, idx_t*, float*, const SearchParameters*) const {
    FB_THROW_MSG("search_and_reconstruct not implemented for this type of index");
}
void Index::compute_residual(const float* x, float* residual, idx_t key) const {
    reconstruct(key, residual);
    for (int i = 0; i < d; i++)
        residual[i] = x[i] - residual[i];
}
void Index::compute_residual_n(idx_t n, const float* xs, float* residuals, const idx_t* keys) const {
    for (idx_t i = 0; i < n; i++)
        compute_residual(xs + (size_t)i * d, residuals + (size_t)i * d, keys[i]);
}

// ------------------------------------------------------------------------------------------
// GpuIndex
// ------------------------------------------------------------------------------------------
GpuIndex::GpuIndex(
        std::shared_ptr<GpuResources> resources,
        int dims,
        MetricType metric,
        float metricArg,
        GpuIndexConfig config)
        : Index(dims, metric), resources_(std::move(resources)), config_(config) {
    metric_arg = metricArg;
    FB_THROW_IF_NOT_MSG(resources_ != nullptr, "null GpuResources");
    FB_THROW_IF_NOT_MSG(dims > 0, "Invalid number of dimensions");
    // every metric but METRIC_NaNEuclidean (faiss/gpu/impl/Distance.cuh:289); the IVF indexes and the clustering
    // entry points narrow this to L2 / inner product themselves
    if (!is_implemented_metric(metric))
        FB_THROW_FMT("unimplemented metric type %d", (int)metric);
    resources_->initializeForDevice(config_.device);
}

void GpuIndex::add(idx_t n, const float* x) {
    add_with_ids(n, x, nullptr);
}

void GpuIndex::add_with_ids(idx_t n, const float* x, const idx_t* ids) {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(this->is_trained, "Index not trained");
    if (n == 0)
        return;
    auto stream = stream_();
    // page large adds (faiss/gpu/GpuIndex.cu:36-44,181-230): <= 512 Ki vectors and <= 256 MiB
    const idx_t maxVecs = std::max<idx_t>(1, std::min<idx_t>(idx_t(512) * 1024, (idx_t(256) << 20) / (sizeof(float) * d)));
    for (idx_t i0 = 0; i0 < n; i0 += maxVecs) {
        InterruptCallback::check(); // between add pages
        const idx_t nb = std::min(maxVecs, n - i0);
        DeviceView<float> xv(resources_.get(), config_.device, x + (size_t)i0 * d, (size_t)nb * d, stream);
        GpuMemoryReservation genIds;
        const idx_t* idp = nullptr;
        DeviceView<idx_t> iv(resources_.get(), config_.device, ids ? ids + i0 : nullptr, nb, stream);
        if (ids) {
            idp = iv.ptr;
        } else if (addImplRequiresIDs_()) {
            genIds = resources_->temp(config_.device, sizeof(idx_t) * nb);
            iota_ids_kernel<<<(unsigned)ceil_div(nb, 256), 256, 0, stream>>>(genIds.as<idx_t>(), nb, this->ntotal);
            CUDA_CHECK_LAST();
            idp = genIds.as<idx_t>();
        }
        addImpl_(nb, xv.ptr, idp);
        CUDA_VERIFY(cudaStreamSynchronize(stream)); // staging buffers die here
    }
}

void GpuIndex::assign(idx_t n, const float* x, idx_t* labels, idx_t k) const {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(this->is_trained, "Index not trained");
    validateKSelect(k);
    if (n == 0)
        return;
    auto dis = resources_->temp(config_.device, sizeof(float) * n * k);
    search(n, x, k, dis.as<float>(), labels);
}

// ------------------------------------------------------------------------------------------
// InterruptCallback
// ------------------------------------------------------------------------------------------
namespace {
std::mutex g_intMu;
InterruptCallback::Fn g_intFn = nullptr;
void* g_intCtx = nullptr;
} // namespace
void InterruptCallback::set(Fn fn, void* ctx) {
    std::lock_guard<std::mutex> g(g_intMu);
    g_intFn = fn;
    g_intCtx = ctx;
}
void InterruptCallback::clear() {
    set(nullptr, nullptr);
}
bool InterruptCallback::is_interrupted() {
    std::lock_guard<std::mutex> g(g_intMu);
    return g_intFn != nullptr && g_intFn(g_intCtx) != 0;
}
void InterruptCallback::check() {
    if (is_interrupted())
        FB_THROW_MSG("computation interrupted");
}

void GpuIndex::search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const {
    search(n, x, k, distances, labels, nullptr);
}

void GpuIndex::search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, const SearchParameters* params) const {
    searchPaged_(n, x, k, distances, labels, params, 0, [&](idx_t nb, const float* xDev, float* dDev, idx_t* iDev, const SearchCall& call) {
        searchImpl_(nb, xDev, (int)k, dDev, iDev, call);
    });
}

void GpuIndex::searchPaged_(
        idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, const SearchParameters* params,
        size_t resultBytes, const SearchPage& page) const {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(this->is_trained, "Index not trained");
    validateKSelect(k);
    if (n == 0)
        return;
    FB_THROW_IF_NOT_MSG(x && distances && labels, "null pointer passed to search");
    SearchCall call;
    call.params = params;
    // the selector is evaluated once per call, before the query pages (temporary memory, released last)
    GpuMemoryReservation mask;
    if (params && params->sel && this->ntotal > 0) {
        mask = selMask_(*params->sel, call.selected);
        call.mask = mask.as<uint32_t>();
    }
    auto stream = stream_();
    // Query paging (role of searchFromCpuPaged_ / searchNonPaged_, faiss/gpu/GpuIndex.cu:554-788).
    // minPagedSize_ is only the THRESHOLD above which host-resident queries are paged (as upstream:
    // setMinPagingSize(0) means "always page", not "one query per page"); the page itself is a fixed
    // byte budget (kSearchPageBytes) and is further bounded by k so that a page's result staging
    // (k * 12 B per query, a few partial copies inside the kernels) stays within the temp arena.
    constexpr size_t kSearchPageBytes = size_t(256) << 20;
    const bool hostPaged = getDeviceForAddress(x) != config_.device && (size_t)n * d * sizeof(float) >= minPagedSize_;
    idx_t maxQ = idx_t(1) << 18;
    if (hostPaged)
        maxQ = std::min<idx_t>(maxQ, (idx_t)(kSearchPageBytes / (sizeof(float) * d)));
    maxQ = std::min<idx_t>(maxQ, (idx_t)((size_t(1) << 30) / ((size_t)k * 12 * 8)));
    if (resultBytes > 0)
        maxQ = std::min<idx_t>(maxQ, (idx_t)(kRetrievalPageBytes / ((size_t)k * resultBytes)));
    maxQ = std::max<idx_t>(maxQ, 1);
    if (hostPaged && searchFromCpuPaged_(n, x, k, distances, labels, maxQ, call, page))
        return;
    for (idx_t i0 = 0; i0 < n; i0 += maxQ) {
        InterruptCallback::check(); // between query pages
        const idx_t nb = std::min(maxQ, n - i0);
        DeviceView<float> xv(resources_.get(), config_.device, x + (size_t)i0 * d, (size_t)nb * d, stream);
        DeviceOut<float> dv(resources_.get(), config_.device, distances + (size_t)i0 * k, (size_t)nb * k);
        DeviceOut<idx_t> lv(resources_.get(), config_.device, labels + (size_t)i0 * k, (size_t)nb * k);
        call.row0 = i0;
        page(nb, xv.ptr, dv.ptr, lv.ptr, call);
        dv.finish(stream);
        lv.finish(stream);
        if (dv.staged || lv.staged || xv.hold.data)
            CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
}

// Host-resident queries above the paging threshold (role of searchFromCpuPaged_, faiss/gpu/GpuIndex.cu:620-788): the
// pinned staging buffer of the resources object is split in two halves; a stager thread copies page p+1 into its
// pinned half and queues the H2D copy on the async-copy stream while the calling thread searches page p on the
// default stream.  (searchImpl_ synchronises with the host -- certificate flags, list offsets -- so the overlap needs
// a second host thread rather than the reference's single-thread event chain.)  Returns false when there is no
// pinned memory to page through; the caller then takes the plain loop.
bool GpuIndex::searchFromCpuPaged_(
        idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, idx_t maxQ, SearchCall call,
        const SearchPage& page) const {
    auto pinned = resources_->getPinnedMemory();
    const size_t half = pinned.second / 2;
    const idx_t pageQ = std::min<idx_t>(maxQ, (idx_t)(half / (sizeof(float) * d)));
    if (!pinned.first || pageQ < 1 || n <= pageQ)
        return false;
    auto stream = stream_();
    auto copyStream = resources_->getAsyncCopyStream(config_.device);
    const idx_t numPages = ceil_div(n, pageQ);
    GpuMemoryReservation devBuf[2] = {
            resources_->temp(config_.device, sizeof(float) * (size_t)pageQ * d),
            resources_->temp(config_.device, sizeof(float) * (size_t)pageQ * d)};
    float* pin[2] = {reinterpret_cast<float*>(pinned.first), reinterpret_cast<float*>((char*)pinned.first + half)};
    cudaEvent_t ready[2];
    for (auto& e : ready)
        CUDA_VERIFY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));

    std::mutex mu;
    std::condition_variable cv;
    idx_t issued = 0;   // pages whose H2D has been queued
    idx_t consumed = 0; // pages whose search has finished (their buffers are free again)
    bool abort = false;
    std::string stagerError;
    const int device = config_.device;
    std::thread stager([&] {
        try {
            CUDA_VERIFY(cudaSetDevice(device));
            for (idx_t p = 0; p < numPages; p++) {
                {
                    std::unique_lock<std::mutex> lk(mu);
                    cv.wait(lk, [&] { return abort || p < consumed + 2; });
                    if (abort)
                        return;
                }
                const int b = (int)(p & 1);
                const idx_t i0 = p * pageQ, nb = std::min(pageQ, n - i0);
                const size_t bytes = sizeof(float) * (size_t)nb * d;
                std::memcpy(pin[b], x + (size_t)i0 * d, bytes);
                CUDA_VERIFY(cudaMemcpyAsync(devBuf[b].data, pin[b], bytes, cudaMemcpyHostToDevice, copyStream));
                CUDA_VERIFY(cudaEventRecord(ready[b], copyStream));
                {
                    std::lock_guard<std::mutex> lk(mu);
                    issued = p + 1;
                }
                cv.notify_all();
            }
        } catch (const std::exception& e) {
            std::lock_guard<std::mutex> lk(mu);
            stagerError = e.what();
            abort = true;
            cv.notify_all();
        }
    });
    auto finish = [&](bool failed) {
        {
            std::lock_guard<std::mutex> lk(mu);
            if (failed)
                abort = true;
        }
        cv.notify_all();
        stager.join();
        cudaStreamSynchronize(copyStream);
        for (auto& e : ready)
            cudaEventDestroy(e);
    };
    try {
        for (idx_t p = 0; p < numPages; p++) {
            InterruptCallback::check(); // between query pages
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return abort || issued > p; });
                if (abort)
                    FB_THROW_FMT("query staging failed: %s", stagerError.c_str());
            }
            const int b = (int)(p & 1);
            const idx_t i0 = p * pageQ, nb = std::min(pageQ, n - i0);
            CUDA_VERIFY(cudaStreamWaitEvent(stream, ready[b], 0));
            DeviceOut<float> dv(resources_.get(), config_.device, distances + (size_t)i0 * k, (size_t)nb * k);
            DeviceOut<idx_t> lv(resources_.get(), config_.device, labels + (size_t)i0 * k, (size_t)nb * k);
            call.row0 = i0;
            page(nb, devBuf[b].as<float>(), dv.ptr, lv.ptr, call);
            dv.finish(stream);
            lv.finish(stream);
            CUDA_VERIFY(cudaStreamSynchronize(stream));
            {
                std::lock_guard<std::mutex> lk(mu);
                consumed = p + 1;
            }
            cv.notify_all();
        }
    } catch (...) {
        finish(true);
        throw;
    }
    finish(false);
    return true;
}

void GpuIndex::compute_residual(const float* x, float* residual, idx_t key) const {
    compute_residual_n(1, x, residual, &key);
}
void GpuIndex::compute_residual_n(idx_t, const float*, float*, const idx_t*) const {
    FB_THROW_MSG("compute_residual not implemented for this type of index");
}

// ------------------------------------------------------------------------------------------
// GpuIndexFlat
// ------------------------------------------------------------------------------------------
GpuIndexFlat::GpuIndexFlat(
        std::shared_ptr<GpuResources> resources,
        int dims,
        MetricType metric,
        GpuIndexFlatConfig config)
        : GpuIndex(std::move(resources), dims, metric, 0, config),
          flatConfig_(config),
          vecs_(resources_.get(), config.device, AllocType::FlatData),
          vecs16_(resources_.get(), config.device, AllocType::FlatData),
          tc_(resources_.get(), config.device, dims) {
    this->is_trained = true;
}

GpuIndexFlat::~GpuIndexFlat() {}

void GpuIndexFlat::reset() {
    DeviceScope scope(config_.device);
    vecs_.clear();
    vecs16_.clear();
    tc_.clear();
    this->ntotal = 0;
}

void GpuIndexFlat::train(idx_t, const float*) {
    // nothing to do
}

void GpuIndexFlat::copyFrom(idx_t n, const float* xb) {
    reset();
    if (n > 0)
        add(n, xb);
}

void GpuIndexFlat::copyTo(float* out) const {
    reconstruct_n(0, ntotal, out);
}

void GpuIndexFlat::add(idx_t n, const float* x) {
    GpuIndex::add_with_ids(n, x, nullptr);
}

void GpuIndexFlat::add_with_ids(idx_t n, const float* x, const idx_t* ids) {
    FB_THROW_IF_NOT_MSG(ids == nullptr, "add_with_ids not supported"); // faiss/gpu/GpuIndexFlat.cu:210
    GpuIndex::add_with_ids(n, x, nullptr);
}

void GpuIndexFlat::addImpl_(idx_t n, const float* xDev, const idx_t* idsDev) {
    FB_THROW_IF_NOT_MSG(idsDev == nullptr, "add_with_ids not supported");
    auto stream = stream_();
    if (flatConfig_.useFloat16) {
        const size_t old = vecs16_.size(), cnt = (size_t)n * d;
        vecs16_.resize(old + cnt, stream);
        float_to_half_kernel<<<(unsigned)std::min<size_t>(ceil_div(cnt, (size_t)256), 65535 * 16), 256, 0, stream>>>(
                xDev, vecs16_.data() + old, nullptr, (int64_t)cnt);
        CUDA_CHECK_LAST();
    } else {
        vecs_.append(xDev, (size_t)n * d, stream);
    }
    this->ntotal += n;
    tc_.invalidate();
}

const float* GpuIndexFlat::roundedQueries_(idx_t n, const float* xDev, GpuMemoryReservation& hold) const {
    if (!flatConfig_.useFloat16 || n == 0)
        return xDev;
    auto stream = stream_();
    const size_t cnt = (size_t)n * d;
    hold = resources_->temp(config_.device, sizeof(float) * cnt);
    float_to_half_kernel<<<(unsigned)std::min<size_t>(ceil_div(cnt, (size_t)256), 65535 * 16), 256, 0, stream>>>(
            xDev, nullptr, hold.as<float>(), (int64_t)cnt);
    CUDA_CHECK_LAST();
    return hold.as<float>();
}

void GpuIndexFlat::replaceVectorsDevice(idx_t n, const float* xDev) {
    DeviceScope scope(config_.device);
    auto stream = stream_();
    if (flatConfig_.useFloat16) {
        vecs16_.resize(0, stream);
        this->ntotal = 0;
        if (n > 0)
            addImpl_(n, xDev, nullptr);
        return;
    }
    float* rows = resizeVectorsDevice(n);
    if (n > 0)
        CUDA_VERIFY(cudaMemcpyAsync(rows, xDev, sizeof(float) * n * d, cudaMemcpyDeviceToDevice, stream));
}

float* GpuIndexFlat::resizeVectorsDevice(idx_t n) {
    FB_THROW_IF_NOT_MSG(!flatConfig_.useFloat16, "fp32 row access on a float16 GpuIndexFlat");
    DeviceScope scope(config_.device);
    vecs_.resize((size_t)n * d, stream_()); // keeps the allocation when it is large enough
    this->ntotal = n;
    tc_.invalidate();
    return vecs_.data();
}

MetricType GpuIndexFlat::searchMetric_() const {
    return flatKernelMetric(metric_type, metric_arg);
}

// faiss/gpu/impl/Distance.cu:152-164: fill with "no result"
void GpuIndexFlat::fillEmpty_(idx_t n, int k, float* dDev, idx_t* iDev) const {
    auto stream = stream_();
    std::vector<float> hd((size_t)n * k, is_similarity_metric(metric_type) ? -FLT_MAX : FLT_MAX);
    std::vector<idx_t> hi((size_t)n * k, -1);
    CUDA_VERIFY(cudaMemcpyAsync(dDev, hd.data(), hd.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaMemcpyAsync(iDev, hi.data(), hi.size() * sizeof(idx_t), cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

GpuMemoryReservation GpuIndexFlat::selMask_(const IDSelector& sel, idx_t& selected) const {
    auto mask = resources_->temp(config_.device, sizeof(uint32_t) * slotMaskWords(this->ntotal));
    buildSlotMask(resources_.get(), config_.device, sel, this->ntotal, nullptr, nullptr, mask.as<uint32_t>(), stream_());
    selected = runCountMask(resources_.get(), config_.device, mask.as<uint32_t>(), this->ntotal, stream_());
    return mask;
}

// A selector that keeps at most 1 row in kCompactRatio searches the gathered selected rows with the exact kernel;
// a larger selection runs the full-size search with the excluded rows masked out.  Both give the same results.
// Measured at N = 10M, d = 128, nq = 10k, k = 100 (bench_filter.py, README): the masked tensor-core search costs
// 45-67 ms whatever the selection, the exact kernel about 0.22 ms per 1000 selected rows (24 ms at 1 %, 220 ms at
// 10 %); the two meet near 250k rows, 1 in 40.  Both costs scale with nq and d alike.
constexpr idx_t kCompactRatio = 40;

void GpuIndexFlat::searchCompacted_(
        idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, const uint32_t* mask, idx_t selected) const {
    auto stream = stream_();
    auto rows = resources_->temp(config_.device, sizeof(idx_t) * this->ntotal);
    runCompactMask(resources_.get(), config_.device, mask, this->ntotal, rows.as<idx_t>(), stream);
    auto sub = resources_->temp(config_.device, sizeof(float) * selected * d);
    runGatherRows(rows_(), rows.as<idx_t>(), selected, d, sub.as<float>(), stream, yHalf_()); // fp16 widens exactly
    runFlatExact(
            resources_.get(), config_.device, xDev, n, sub.as<float>(), selected, d, k, searchMetric_(), 0, dDev, iDev,
            stream, 0, metric_arg);
    runRemapLabels(iDev, n * k, rows.as<idx_t>(), stream);
}

void GpuIndexFlat::searchImpl_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, const SearchCall& call) const {
    auto stream = stream_();
    if (call.row0 == 0)
        lastSearchFallbackQueries = 0;
    lastSearchUsedTensorCores = 0;
    lastSearchOperandBits = 0;
    if (this->ntotal == 0) {
        fillEmpty_(n, k, dDev, iDev);
        return;
    }
    // metrics without a product form (L1, Linf, Lp, Canberra, ...) always run the exact kernel
    const bool tc = useTensorCores_(k, n);
    GpuMemoryReservation qHold;
    xDev = roundedQueries_(n, xDev, qHold);
    const uint32_t* mask = call.mask;
    if (mask) {
        if (call.selected == 0) {
            fillEmpty_(n, k, dDev, iDev);
            return;
        }
        if (call.selected * kCompactRatio <= this->ntotal) {
            searchCompacted_(n, xDev, k, dDev, iDev, mask, call.selected);
            return;
        }
    }
    if (tc) {
        tc_.prepare(rows_(), this->ntotal, searchMetric_(), yHalf_(), stream);
        lastSearchFallbackQueries += (int)tc_.search(xDev, n, k, dDev, iDev, stream, nullptr, mask);
        lastSearchUsedTensorCores = 1;
        lastSearchOperandBits = tc_.lastOperandBits();
    } else {
        runFlatExact(
                resources_.get(), config_.device, xDev, n, rows_(), this->ntotal, d, k, searchMetric_(), 0, dDev, iDev,
                stream, yHalf_(), metric_arg, mask);
    }
}

bool GpuIndexFlat::shardPoolingEligible(int k, idx_t n) const {
    // pooled thresholds are a tensor-core certificate: other metrics take the plain all-gather + merge path
    return useTensorCores_(k, n);
}

void GpuIndexFlat::searchShardDevice(
        idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, const FlatTcShard* flatShard, const SearchCall& call) const {
    if (!flatShard) {
        searchImpl_(n, xDev, k, dDev, iDev, call);
        return;
    }
    FB_THROW_IF_NOT_MSG(shardPoolingEligible(k, n), "pooled sharded search requested on a shard that cannot take the tensor-core path");
    auto stream = stream_();
    tc_.prepare(rows_(), this->ntotal, searchMetric_(), yHalf_(), stream);
    GpuMemoryReservation qHold;
    xDev = roundedQueries_(n, xDev, qHold);
    if (call.row0 == 0)
        lastSearchFallbackQueries = 0;
    lastSearchFallbackQueries += (int)tc_.search(xDev, n, k, dDev, iDev, stream, flatShard);
    lastSearchUsedTensorCores = 1;
    lastSearchOperandBits = tc_.lastOperandBits();
}

void GpuIndexFlat::search_and_reconstruct(
        idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, float* recons, const SearchParameters* params) const {
    search(n, x, k, distances, labels, params);
    if (n == 0)
        return;
    FB_THROW_IF_NOT_MSG(recons, "null pointer passed to search_and_reconstruct");
    DeviceScope scope(config_.device);
    auto stream = stream_();
    // labels are row numbers: gather the rows, a page of results at a time
    const idx_t total = n * k;
    const idx_t pageRows = std::max<idx_t>(1, (idx_t)(kRetrievalPageBytes / (sizeof(float) * d)));
    for (idx_t r0 = 0; r0 < total; r0 += pageRows) {
        const idx_t nr = std::min(pageRows, total - r0);
        DeviceView<idx_t> lv(resources_.get(), config_.device, labels + r0, nr, stream);
        DeviceOut<float> rv(resources_.get(), config_.device, recons + (size_t)r0 * d, (size_t)nr * d);
        runGatherRows(rows_(), lv.ptr, nr, d, rv.ptr, stream, yHalf_(), true);
        rv.finish(stream);
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
}

void GpuIndexFlat::reconstruct(idx_t key, float* out) const {
    reconstruct_n(key, 1, out);
}

void GpuIndexFlat::reconstruct_n(idx_t i0, idx_t num, float* out) const {
    DeviceScope scope(config_.device);
    if (num == 0)
        return;
    FB_THROW_IF_NOT_MSG(i0 >= 0 && i0 + num <= this->ntotal, "reconstruct: index out of bounds");
    auto stream = stream_();
    if (flatConfig_.useFloat16) { // widen through a device buffer, 64 MiB of fp32 at a time
        const idx_t step = std::max<idx_t>(1, (idx_t)((size_t(64) << 20) / (sizeof(float) * d)));
        for (idx_t r = 0; r < num; r += step) {
            const idx_t m = std::min(step, num - r);
            const size_t cnt = (size_t)m * d;
            DeviceOut<float> ov(resources_.get(), config_.device, out + (size_t)r * d, cnt);
            half_to_float_kernel<<<(unsigned)std::min<size_t>(ceil_div(cnt, (size_t)256), 65535 * 16), 256, 0, stream>>>(
                    vecs16_.data() + (size_t)(i0 + r) * d, ov.ptr, (int64_t)cnt);
            CUDA_CHECK_LAST();
            ov.finish(stream);
            CUDA_VERIFY(cudaStreamSynchronize(stream));
        }
        return;
    }
    CUDA_VERIFY(cudaMemcpyAsync(out, vecs_.data() + (size_t)i0 * d, sizeof(float) * num * d, cudaMemcpyDefault, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

void GpuIndexFlat::reconstruct_batch(idx_t n, const idx_t* keys, float* out) const {
    DeviceScope scope(config_.device);
    if (n == 0)
        return;
    auto stream = stream_();
    DeviceView<idx_t> kv(resources_.get(), config_.device, keys, n, stream);
    DeviceOut<float> ov(resources_.get(), config_.device, out, (size_t)n * d);
    runGatherRows(rows_(), kv.ptr, n, d, ov.ptr, stream, yHalf_());
    ov.finish(stream);
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

void GpuIndexFlat::compute_residual(const float* x, float* residual, idx_t key) const {
    compute_residual_n(1, x, residual, &key);
}

void GpuIndexFlat::compute_residual_n(idx_t n, const float* xs, float* residuals, const idx_t* keys) const {
    DeviceScope scope(config_.device);
    if (n == 0)
        return;
    auto stream = stream_();
    DeviceView<float> xv(resources_.get(), config_.device, xs, (size_t)n * d, stream);
    DeviceView<idx_t> kv(resources_.get(), config_.device, keys, n, stream);
    DeviceOut<float> ov(resources_.get(), config_.device, residuals, (size_t)n * d);
    runCalcResidual(xv.ptr, rows_(), kv.ptr, n, d, ov.ptr, stream, yHalf_());
    ov.finish(stream);
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

// ------------------------------------------------------------------------------------------
// Clustering
// ------------------------------------------------------------------------------------------
void rand_perm(int* perm, size_t n, int64_t seed) {
    std::iota(perm, perm + n, 0);
    std::mt19937 mt((unsigned int)seed);
    for (size_t i = 0; i + 1 < n; i++) {
        int i2 = (int)(i + mt() % (n - i));
        std::swap(perm[i], perm[i2]);
    }
}

int split_clusters(size_t d, size_t k, size_t n, float* hassign, float* centroids) {
    const float EPS = 1.f / 1024.f;
    FB_THROW_IF_NOT_MSG(n > k, "split_clusters: n must exceed k to find a non-empty donor centroid");
    std::mt19937 mt(1234u);
    size_t nsplit = 0;
    for (size_t ci = 0; ci < k; ci++) {
        if (hassign[ci] != 0)
            continue;
        size_t cj = 0, tries = 0;
        const size_t maxTries = 10 * k;
        bool found = false;
        for (cj = 0; tries < maxTries; cj = (cj + 1) % k) {
            float p = (hassign[cj] - 1.0) / (float)(n - k);
            float r = mt() / float(mt.max());
            if (r < p) {
                found = true;
                break;
            }
            tries++;
        }
        if (!found) {
            cj = 0;
            for (size_t j = 1; j < k; j++)
                if (hassign[j] > hassign[cj])
                    cj = j;
        }
        memcpy(centroids + ci * d, centroids + cj * d, sizeof(float) * d);
        for (size_t j = 0; j < d; j++) {
            if (j % 2 == 0) {
                centroids[ci * d + j] *= 1 + EPS;
                centroids[cj * d + j] *= 1 - EPS;
            } else {
                centroids[ci * d + j] *= 1 - EPS;
                centroids[cj * d + j] *= 1 + EPS;
            }
        }
        hassign[ci] = hassign[cj] / 2;
        hassign[cj] -= hassign[ci];
        nsplit++;
    }
    return (int)nsplit;
}

namespace {
__global__ void scatter_rows_kernel(const float* src, const int* srcRow, const int* dstRow, int64_t n, int d, float* dst) {
    const int64_t i = blockIdx.x;
    if (i >= n)
        return;
    for (int j = threadIdx.x; j < d; j += blockDim.x)
        dst[(int64_t)dstRow[i] * d + j] = src[(int64_t)srcRow[i] * d + j];
}
__global__ void store_obj_kernel(const double* acc, float* out) {
    *out = (float)*acc;
}
} // namespace

float Clustering::lloyd_(
        idx_t nLocal,
        const float* x,
        idx_t nTotal,
        idx_t off,
        GpuIndexFlat& index,
        int redo,
        const Communicator* comm,
        double t0,
        double& tSearch) {
    GpuResources* res = index.getResources().get();
    const int device = index.getDevice();
    cudaStream_t stream = res->getDefaultStream(device);

    centroids.resize(d * k);
    const size_t packedLen = k * d + k + 1; // sums | counts | objective
    auto cDev = res->device_alloc(device, sizeof(float) * k * d, AllocType::Other);
    auto packed = res->device_alloc(device, sizeof(float) * packedLen, AllocType::Other);
    auto assign = res->device_alloc(device, sizeof(idx_t) * std::max<idx_t>(nLocal, 1), AllocType::Other);
    auto dis = res->device_alloc(device, sizeof(float) * std::max<idx_t>(nLocal, 1), AllocType::Other);
    auto objBuf = res->device_alloc(device, sizeof(double), AllocType::Other);

    // initial centroids = rows rand_perm(nTotal, seed + 1 + redo*15486557)[:k] of the concatenated set: every row is
    // owned by exactly one rank, which writes it into a zeroed table; the all-reduce assembles the table everywhere
    {
        std::vector<int> perm(nTotal);
        rand_perm(perm.data(), nTotal, (int64_t)seed + 1 + redo * 15486557L);
        std::vector<int> srcRow, dstRow;
        for (size_t i = 0; i < k; i++) {
            const idx_t g = perm[i];
            if (g >= off && g < off + nLocal) {
                srcRow.push_back((int)(g - off));
                dstRow.push_back((int)i);
            }
        }
        CUDA_VERIFY(cudaMemsetAsync(cDev.data, 0, sizeof(float) * k * d, stream));
        if (!srcRow.empty()) {
            auto sd = res->temp(device, sizeof(int) * srcRow.size() * 2);
            CUDA_VERIFY(cudaMemcpyAsync(sd.data, srcRow.data(), sizeof(int) * srcRow.size(), cudaMemcpyHostToDevice, stream));
            CUDA_VERIFY(cudaMemcpyAsync(sd.as<int>() + srcRow.size(), dstRow.data(), sizeof(int) * srcRow.size(), cudaMemcpyHostToDevice, stream));
            scatter_rows_kernel<<<(unsigned)srcRow.size(), std::min<int>(256, (int)d), 0, stream>>>(
                    x, sd.as<int>(), sd.as<int>() + srcRow.size(), (int64_t)srcRow.size(), (int)d, cDev.as<float>());
            CUDA_CHECK_LAST();
            CUDA_VERIFY(cudaStreamSynchronize(stream));
        }
        if (comm)
            comm->allReduceSum(cDev.as<float>(), k * d, stream);
        runKmeansPostProcess(cDev.as<float>(), (int64_t)k, (int)d, spherical, int_centroids, stream);
    }
    if (index.ntotal != 0)
        index.reset();
    if (!index.is_trained)
        index.train(k, cDev.as<float>());
    index.add(k, cDev.as<float>());

    float obj = 0;
    std::vector<float> hcounts(k + 1); // k counts | objective
    for (int it = 0; it < niter; it++) {
        const double t0s = now_ms();
        if (nLocal > 0)
            index.searchDevice(nLocal, x, 1, dis.as<float>(), assign.as<idx_t>());
        CUDA_VERIFY(cudaMemsetAsync(objBuf.data, 0, sizeof(double), stream));
        CUDA_VERIFY(cudaMemsetAsync(packed.data, 0, sizeof(float) * packedLen, stream));
        if (nLocal > 0) {
            sum_kernel<<<296, 256, 0, stream>>>(dis.as<float>(), nLocal, objBuf.as<double>());
            CUDA_CHECK_LAST();
            runKmeansAccumulate(x, assign.as<idx_t>(), nLocal, (int)d, (int64_t)k, packed.as<float>(), packed.as<float>() + k * d, stream);
        }
        store_obj_kernel<<<1, 1, 0, stream>>>(objBuf.as<double>(), packed.as<float>() + k * d + k);
        CUDA_CHECK_LAST();
        if (comm) // ONE packed reduction per iteration
            comm->allReduceSum(packed.as<float>(), packedLen, stream);
        runKmeansFinalize(packed.as<float>(), packed.as<float>() + k * d, (int64_t)k, (int)d, cDev.as<float>(), stream);
        CUDA_VERIFY(cudaMemcpyAsync(hcounts.data(), packed.as<float>() + k * d, sizeof(float) * (k + 1), cudaMemcpyDeviceToHost, stream));
        CUDA_VERIFY(cudaStreamSynchronize(stream));
        tSearch += now_ms() - t0s;
        obj = hcounts[k];

        // empty clusters -> split on the host exactly as the reference does
        int nsplit = 0;
        double tot = 0, uf = 0;
        bool anyEmpty = false;
        for (size_t c = 0; c < k; c++) {
            tot += hcounts[c];
            uf += (double)hcounts[c] * hcounts[c];
            anyEmpty |= hcounts[c] == 0;
        }
        const double imb = tot > 0 ? uf * k / (tot * tot) : 0;
        if (anyEmpty) {
            // identical inputs and a fixed-seed generator: every rank computes the same split
            const double ts = now_ms();
            CUDA_VERIFY(cudaMemcpyAsync(centroids.data(), cDev.data, sizeof(float) * k * d, cudaMemcpyDeviceToHost, stream));
            CUDA_VERIFY(cudaStreamSynchronize(stream));
            nsplit = split_clusters(d, k, nTotal, hcounts.data(), centroids.data());
            CUDA_VERIFY(cudaMemcpyAsync(cDev.data, centroids.data(), sizeof(float) * k * d, cudaMemcpyHostToDevice, stream));
            splitSeconds += (now_ms() - ts) / 1000.0;
        }
        iteration_stats.push_back({obj, (now_ms() - t0) / 1000.0, tSearch / 1000.0, imb, nsplit});
        if (verbose) {
            printf("  Iteration %d (%.2f s, search %.2f s): objective=%g imbalance=%.3f nsplit=%d       \r",
                   it, (now_ms() - t0) / 1000.0, tSearch / 1000.0, obj, imb, nsplit);
            fflush(stdout);
        }
        runKmeansPostProcess(cDev.as<float>(), (int64_t)k, (int)d, spherical, int_centroids, stream);
        if (update_index) {
            index.reset();
            index.train(k, cDev.as<float>());
            index.add(k, cDev.as<float>());
        } else {
            index.replaceVectorsDevice(k, cDev.as<float>());
        }
        // faiss/Clustering.cpp:356; not with a communicator: a rank that left the loop would strand the others in
        // their next all-reduce
        if (!comm)
            InterruptCallback::check();
        // early stop when the objective did not change (early_stop_threshold = 0, faiss/Clustering.cpp:360-377)
        if (it > 0) {
            const float prev = iteration_stats[iteration_stats.size() - 2].obj;
            if (prev != 0 && std::fabs((double)prev - (double)obj) / std::fabs((double)prev) <= 0.0)
                break;
        }
    }
    if (verbose)
        printf("\n");
    CUDA_VERIFY(cudaMemcpyAsync(centroids.data(), cDev.data, sizeof(float) * k * d, cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    return obj;
}

// the assignment step runs on the L2 / inner-product tensor-core path; the other metrics are not clustered
static void checkClusteringMetric(const GpuIndexFlat& index) {
    if (!(index.metric_type == METRIC_L2 || index.metric_type == METRIC_INNER_PRODUCT))
        FB_THROW_FMT("unsupported metric type %d", (int)index.metric_type);
}

void Clustering::train(idx_t nx, const float* x_in, GpuIndexFlat& index) {
    checkClusteringMetric(index);
    FB_THROW_IF_NOT_FMT(
            nx >= (idx_t)k,
            "Number of training points (%ld) should be at least as large as number of clusters (%zd)",
            (long)nx,
            k);
    FB_THROW_IF_NOT_FMT((size_t)index.d == d, "Index dimension %d not the same as data dimension %d", index.d, (int)d);
    // input centroids (hot start / frozen) are not part of this path; refuse instead of ignoring the flag
    FB_THROW_IF_NOT_MSG(!frozen_centroids, "Clustering: frozen_centroids (input centroids) is not supported by faiss_b200");
    GpuResources* res = index.getResources().get();
    const int device = index.getDevice();
    DeviceScope scope(device);
    cudaStream_t stream = res->getDefaultStream(device);
    const double t0 = now_ms();
    splitSeconds = 0;

    // training set resident on the device for the whole run
    DeviceView<float> xall(res, device, x_in, (size_t)nx * d, stream);
    const float* x = xall.ptr;
    GpuMemoryReservation sub;
    if ((size_t)nx > k * (size_t)max_points_per_centroid) {
        // subsample_training_set (faiss/impl/ClusteringHelpers.cpp:36-99): first k*max_ppc of rand_perm(seed)
        FB_THROW_IF_NOT_MSG(nx <= (idx_t)0x7fffffff, "Dataset too large for standard subsampling");
        if (verbose)
            printf("Sampling a subset of %zd / %ld for training\n", k * max_points_per_centroid, (long)nx);
        x = subsampleRowsDevice(res, device, nx, (int)d, (idx_t)(k * max_points_per_centroid), seed, x, sub, stream);
    } else if ((size_t)nx < k * (size_t)min_points_per_centroid) {
        fprintf(stderr,
                "WARNING clustering %ld points to %zd centroids: please provide at least %ld training points\n",
                (long)nx,
                k,
                (long)(k * min_points_per_centroid));
    }

    if ((size_t)nx == k) {
        centroids.resize(d * k);
        CUDA_VERIFY(cudaMemcpyAsync(centroids.data(), x, sizeof(float) * d * k, cudaMemcpyDeviceToHost, stream));
        CUDA_VERIFY(cudaStreamSynchronize(stream));
        iteration_stats.push_back({0.f, 0.0, 0.0, 1.0, 0});
        index.reset();
        index.add(k, centroids.data());
        return;
    }
    if (verbose)
        printf("Clustering %ld points in %zdD to %zd clusters, redo %d times, %d iterations\n",
               (long)nx, d, k, nredo, niter);

    const bool lower_is_better = !is_similarity_metric(index.metric_type);
    float best_obj = lower_is_better ? HUGE_VALF : -HUGE_VALF;
    std::vector<ClusteringIterationStats> best_stats;
    std::vector<float> best_centroids;
    double t_search_tot = 0;
    for (int redo = 0; redo < nredo; redo++) {
        const float obj = lloyd_(nx, x, nx, 0, index, redo, nullptr, t0, t_search_tot);
        if (nredo > 1) {
            if ((lower_is_better && obj < best_obj) || (!lower_is_better && obj > best_obj)) {
                best_centroids = centroids;
                best_stats = iteration_stats;
                best_obj = obj;
            }
            index.reset();
        }
    }
    if (nredo > 1) {
        centroids = best_centroids;
        iteration_stats = best_stats;
        index.reset();
        index.add(k, best_centroids.data());
    }
}

void Clustering::trainSharded(idx_t nLocal, const float* x_in, GpuIndexFlat& index, const Communicator& comm) {
    checkClusteringMetric(index);
    FB_THROW_IF_NOT_FMT((size_t)index.d == d, "Index dimension %d not the same as data dimension %d", index.d, (int)d);
    FB_THROW_IF_NOT_MSG(!frozen_centroids, "Clustering: frozen_centroids (input centroids) is not supported by faiss_b200");
    FB_THROW_IF_NOT_MSG(nredo == 1, "sharded clustering supports nredo == 1");
    GpuResources* res = index.getResources().get();
    const int device = index.getDevice();
    DeviceScope scope(device);
    cudaStream_t stream = res->getDefaultStream(device);
    const double t0 = now_ms();
    splitSeconds = 0;

    DeviceView<float> xall(res, device, x_in, (size_t)nLocal * d, stream);
    std::vector<int64_t> sizes = comm.allGatherHostI64(nLocal, stream);
    idx_t nTotal = 0, off = 0;
    for (int r = 0; r < comm.size(); r++) {
        if (r < comm.rank())
            off += sizes[r];
        nTotal += sizes[r];
    }
    FB_THROW_IF_NOT_FMT(
            nTotal >= (idx_t)k,
            "Number of training points (%ld) should be at least as large as number of clusters (%zd)",
            (long)nTotal,
            k);
    FB_THROW_IF_NOT_MSG(nTotal <= (idx_t)0x7fffffff, "Dataset too large for the reference's int permutation");

    double tSearch = 0;
    lloyd_(nLocal, xall.ptr, nTotal, off, index, 0, &comm, t0, tSearch);
}

// ------------------------------------------------------------------------------------------
// IvfLists
// ------------------------------------------------------------------------------------------
IvfLists::IvfLists(GpuResources* res, int device, int64_t nlist, int codeSize, bool pqInterleaved)
        : res_(res),
          device_(device),
          nlist_(nlist),
          codeSize_(codeSize),
          interleaved_(pqInterleaved),
          hStart_(nlist, 0),
          hCap_(nlist, 0),
          hLen_(nlist, 0) {
    AllocRequest r;
    r.type = AllocType::IVFLists;
    r.device = device;
    r.space = MemorySpace::Device;
    r.stream = res->getDefaultStream(device);
    r.size = sizeof(int64_t) * nlist;
    dStart_ = (int64_t*)res_->allocMemory(r);
    r.size = sizeof(int) * nlist;
    dLen_ = (int*)res_->allocMemory(r);
    dCounts_ = (int*)res_->allocMemory(r);
    uploadMeta_(r.stream);
}

IvfLists::~IvfLists() {
    res_->deallocMemory(device_, dStart_);
    res_->deallocMemory(device_, dLen_);
    res_->deallocMemory(device_, dCounts_);
    if (codes_)
        res_->deallocMemory(device_, codes_);
    if (ids_)
        res_->deallocMemory(device_, ids_);
}

void IvfLists::uploadMeta_(cudaStream_t stream) {
    CUDA_VERIFY(cudaMemcpyAsync(dStart_, hStart_.data(), sizeof(int64_t) * nlist_, cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaMemcpyAsync(dLen_, hLen_.data(), sizeof(int) * nlist_, cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

void IvfLists::reset() {
    cudaStream_t stream = res_->getDefaultStream(device_);
    if (codes_)
        res_->deallocMemory(device_, codes_);
    if (ids_)
        res_->deallocMemory(device_, ids_);
    codes_ = nullptr;
    ids_ = nullptr;
    arenaElems_ = 0;
    std::fill(hStart_.begin(), hStart_.end(), 0);
    std::fill(hCap_.begin(), hCap_.end(), 0);
    std::fill(hLen_.begin(), hLen_.end(), 0);
    uploadMeta_(stream);
}

int IvfLists::maxListLength() const {
    int m = 0;
    for (int v : hLen_)
        m = std::max(m, v);
    return m;
}

// move every list to a new arena with the given capacities (multiples of 32 elements: 16-byte
// aligned list starts for any code size, whole groups for the interleaved PQ layout)
void IvfLists::relayout_(const std::vector<int64_t>& newCap, cudaStream_t stream) {
    std::vector<int64_t> newStart(nlist_);
    int64_t total = 0;
    for (int64_t l = 0; l < nlist_; l++) {
        newStart[l] = total;
        total += round_up(newCap[l], 32);
    }
    AllocRequest r;
    r.type = AllocType::IVFLists;
    r.device = device_;
    r.space = MemorySpace::Device;
    r.stream = stream;
    r.size = std::max<int64_t>(total, 16) * codeSize_;
    uint8_t* nc = (uint8_t*)res_->allocMemory(r);
    if (interleaved_) // tail lanes of the last group are read (and masked) by the scan: keep them defined
        CUDA_VERIFY(cudaMemsetAsync(nc, 0, r.size, stream));
    r.size = std::max<int64_t>(total, 16) * sizeof(idx_t);
    idx_t* ni = nullptr;
    try {
        ni = (idx_t*)res_->allocMemory(r);
    } catch (...) {
        res_->deallocMemory(device_, nc);
        throw;
    }
    if (codes_) {
        auto ds = res_->temp(device_, sizeof(int64_t) * nlist_);
        CUDA_VERIFY(cudaMemcpyAsync(ds.data, newStart.data(), sizeof(int64_t) * nlist_, cudaMemcpyHostToDevice, stream));
        copy_lists_kernel<<<(unsigned)nlist_, 256, 0, stream>>>(
                codes_, ids_, dStart_, dLen_, ds.as<int64_t>(), codeSize_, interleaved_ ? 32 : 1, nc, ni);
        CUDA_CHECK_LAST();
        CUDA_VERIFY(cudaStreamSynchronize(stream));
        res_->deallocMemory(device_, codes_);
        res_->deallocMemory(device_, ids_);
    }
    codes_ = nc;
    ids_ = ni;
    arenaElems_ = total;
    hStart_ = newStart;
    for (int64_t l = 0; l < nlist_; l++)
        hCap_[l] = round_up(newCap[l], 32);
    uploadMeta_(stream);
}

void IvfLists::reserve(size_t totalVecs, cudaStream_t stream) {
    // faiss/gpu/impl/IVFBase.cu reserveMemory: spread evenly
    int64_t per = (int64_t)ceil_div((int64_t)totalVecs, nlist_);
    std::vector<int64_t> cap(nlist_);
    bool grow = false;
    for (int64_t l = 0; l < nlist_; l++) {
        cap[l] = std::max<int64_t>(hCap_[l], per);
        grow |= cap[l] > hCap_[l];
    }
    if (grow)
        relayout_(cap, stream);
}

void IvfLists::reserveLists(const int64_t* lens, cudaStream_t stream) {
    std::vector<int64_t> cap(nlist_);
    bool grow = false;
    for (int64_t l = 0; l < nlist_; l++) {
        FB_THROW_IF_NOT_MSG(lens[l] >= 0 && lens[l] < (int64_t(1) << 31), "invalid inverted list length");
        cap[l] = std::max<int64_t>(hCap_[l], lens[l]);
        grow |= cap[l] > hCap_[l];
    }
    if (grow)
        relayout_(cap, stream);
}

size_t IvfLists::reclaim(cudaStream_t stream) {
    size_t before = (size_t)arenaElems_ * (codeSize_ + sizeof(idx_t));
    std::vector<int64_t> cap(nlist_);
    for (int64_t l = 0; l < nlist_; l++)
        cap[l] = hLen_[l];
    relayout_(cap, stream);
    size_t after = (size_t)arenaElems_ * (codeSize_ + sizeof(idx_t));
    return before > after ? before - after : 0;
}

idx_t IvfLists::append(idx_t n, const uint8_t* rowsDev, const idx_t* idsDev, const idx_t* assignDev, cudaStream_t stream) {
    if (n == 0)
        return 0;
    // batch histogram on the device, mirrored to the host for capacity planning
    CUDA_VERIFY(cudaMemsetAsync(dCounts_, 0, sizeof(int) * nlist_, stream));
    runIvfCountAssign(assignDev, n, nlist_, dCounts_, stream);
    std::vector<int> hc(nlist_);
    CUDA_VERIFY(cudaMemcpyAsync(hc.data(), dCounts_, sizeof(int) * nlist_, cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    bool grow = false;
    idx_t stored = 0;
    std::vector<int64_t> cap(nlist_);
    for (int64_t l = 0; l < nlist_; l++) {
        int64_t need = (int64_t)hLen_[l] + hc[l];
        stored += hc[l];
        FB_THROW_IF_NOT_MSG(need < (int64_t(1) << 31), "inverted list too long");
        if (need > hCap_[l]) {
            grow = true;
            cap[l] = std::max<int64_t>(need + need / 4, 16); // 1.25x geometric slack
        } else {
            cap[l] = hCap_[l];
        }
    }
    if (grow)
        relayout_(cap, stream);
    auto offsets = res_->temp(device_, sizeof(int) * n);
    runIvfAppendOffsets(assignDev, n, nlist_, dLen_, offsets.as<int>(), nullptr, stream);
    if (interleaved_)
        runIvfPqScatterInterleaved(rowsDev, idsDev, assignDev, offsets.as<int>(), n, codeSize_, dStart_, codes_, ids_, stream);
    else
        runIvfScatter(rowsDev, idsDev, assignDev, offsets.as<int>(), n, codeSize_, dStart_, codes_, ids_, stream);
    for (int64_t l = 0; l < nlist_; l++)
        hLen_[l] += hc[l];
    CUDA_VERIFY(cudaMemcpyAsync(dLen_, hLen_.data(), sizeof(int) * nlist_, cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    return stored;
}

void IvfLists::setListFromHost(int64_t l, int64_t len, const uint8_t* codes, const idx_t* ids, cudaStream_t stream) {
    FB_THROW_IF_NOT(l >= 0 && l < nlist_);
    if (len > hCap_[l]) {
        std::vector<int64_t> cap(hCap_.begin(), hCap_.end());
        cap[l] = len;
        relayout_(cap, stream);
    }
    if (len > 0) {
        if (interleaved_) {
            auto tmp = res_->temp(device_, (size_t)len * codeSize_);
            CUDA_VERIFY(cudaMemcpyAsync(tmp.data, codes, (size_t)len * codeSize_, cudaMemcpyDefault, stream));
            runIvfPqListToInterleaved(tmp.as<uint8_t>(), len, codeSize_, codes_ + hStart_[l] * codeSize_, stream);
            CUDA_VERIFY(cudaStreamSynchronize(stream));
        } else {
            CUDA_VERIFY(cudaMemcpyAsync(codes_ + hStart_[l] * codeSize_, codes, (size_t)len * codeSize_, cudaMemcpyDefault, stream));
        }
        CUDA_VERIFY(cudaMemcpyAsync(ids_ + hStart_[l], ids, (size_t)len * sizeof(idx_t), cudaMemcpyDefault, stream));
    }
    hLen_[l] = (int)len;
    CUDA_VERIFY(cudaMemcpyAsync(dLen_ + l, &hLen_[l], sizeof(int), cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

void IvfLists::getListToHost(int64_t l, uint8_t* codes, idx_t* ids, cudaStream_t stream) const {
    FB_THROW_IF_NOT(l >= 0 && l < nlist_);
    int64_t len = hLen_[l];
    if (len == 0)
        return;
    if (codes) {
        if (interleaved_) {
            auto tmp = res_->temp(device_, (size_t)len * codeSize_);
            runIvfPqListFromInterleaved(codes_ + hStart_[l] * codeSize_, len, codeSize_, tmp.as<uint8_t>(), stream);
            CUDA_VERIFY(cudaMemcpyAsync(codes, tmp.data, (size_t)len * codeSize_, cudaMemcpyDeviceToHost, stream));
            CUDA_VERIFY(cudaStreamSynchronize(stream));
        } else {
            CUDA_VERIFY(cudaMemcpyAsync(codes, codes_ + hStart_[l] * codeSize_, (size_t)len * codeSize_, cudaMemcpyDeviceToHost, stream));
        }
    }
    if (ids)
        CUDA_VERIFY(cudaMemcpyAsync(ids, ids_ + hStart_[l], (size_t)len * sizeof(idx_t), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

// ------------------------------------------------------------------------------------------
// GpuIndexIVF
// ------------------------------------------------------------------------------------------
GpuIndexIVF::GpuIndexIVF(
        std::shared_ptr<GpuResources> resources,
        int dims,
        MetricType metric,
        idx_t nlist_,
        int codeSize,
        GpuIndexIVFConfig config,
        bool pqInterleaved)
        : GpuIndex(std::move(resources), dims, metric, 0, config), nlist(nlist_), ivfConfig_(config) {
    // faiss/gpu/GpuIndexIVF.cu:34-38: only L2 and inner product
    if (!(metric == METRIC_L2 || metric == METRIC_INNER_PRODUCT))
        FB_THROW_FMT("unsupported metric type %d", (int)metric);
    FB_THROW_IF_NOT_MSG(nlist > 0, "nlist must be > 0");
    // faiss/gpu/GpuIndexIVF.cu:72-80: spherical k-means for inner product, 10 iterations
    if (metric == METRIC_INNER_PRODUCT)
        cp.spherical = true;
    cp.niter = 10;
    GpuIndexFlatConfig fc = config.flatConfig;
    fc.device = config.device;
    quantizer = new GpuIndexFlat(resources_, dims, metric, fc);
    own_fields = true;
    this->is_trained = false;
    lists_.reset(new IvfLists(resources_.get(), config.device, nlist, codeSize, pqInterleaved));
}

// the constructors taking `Index* coarseQuantizer` (faiss/gpu/GpuIndexIVFFlat.h:48-59, GpuIndexIVFPQ.h:69-82,
// GpuIndexIVF.cu:84-100): the quantiser is shared, not owned; the index is trained iff the quantiser already
// holds nlist centroids (the PQ of a GpuIndexIVFPQ still needs train()).  Only this library's GpuIndexFlat is
// accepted (a CPU quantiser would put a host search on the path: allowCpuCoarseQuantizer stays unsupported).
void GpuIndexIVF::setQuantizer(GpuIndexFlat* coarse) {
    FB_THROW_IF_NOT_MSG(coarse != nullptr, "null coarse quantizer");
    FB_THROW_IF_NOT_MSG(coarse->d == d, "coarse quantizer dimension mismatch");
    FB_THROW_IF_NOT_MSG(coarse->metric_type == metric_type, "coarse quantizer metric mismatch");
    FB_THROW_IF_NOT_MSG(coarse->getDevice() == config_.device, "coarse quantizer lives on another device");
    FB_THROW_IF_NOT_MSG(this->ntotal == 0, "cannot swap the quantizer of a populated index");
    if (own_fields)
        delete quantizer;
    quantizer = coarse;
    own_fields = false;
    coarseEpoch++;
    this->is_trained = quantizer->is_trained && quantizer->ntotal == nlist && quantizerOnlyTraining_();
}

GpuIndexIVF::~GpuIndexIVF() {
    lists_.reset();
    if (own_fields)
        delete quantizer;
}

idx_t GpuIndexIVF::getListLength(idx_t listId) const {
    FB_THROW_IF_NOT(listId >= 0 && listId < nlist);
    return lists_->listLength(listId);
}

std::vector<uint8_t> GpuIndexIVF::getListVectorData(idx_t listId) const {
    DeviceScope scope(config_.device);
    std::vector<uint8_t> out((size_t)getListLength(listId) * lists_->codeSize());
    lists_->getListToHost(listId, out.data(), nullptr, stream_());
    return out;
}

std::vector<idx_t> GpuIndexIVF::getListIndices(idx_t listId) const {
    DeviceScope scope(config_.device);
    std::vector<idx_t> out((size_t)getListLength(listId));
    lists_->getListToHost(listId, nullptr, out.data(), stream_());
    return out;
}

void GpuIndexIVF::reserveMemory(size_t numVecs) {
    DeviceScope scope(config_.device);
    lists_->reserve(numVecs, stream_());
}

void GpuIndexIVF::setListSizes(const idx_t* lens) {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(lens != nullptr, "null list-size array");
    lists_->reserveLists(lens, stream_());
}

size_t GpuIndexIVF::reclaimMemory() {
    DeviceScope scope(config_.device);
    return lists_->reclaim(stream_());
}

void GpuIndexIVF::reset() {
    DeviceScope scope(config_.device);
    lists_->reset();
    this->ntotal = 0;
}

void GpuIndexIVF::setCoarseCentroids(const float* c) {
    DeviceScope scope(config_.device);
    quantizer->reset();
    quantizer->add(nlist, c);
    coarseEpoch++;
    quantizer->is_trained = true;
}

void GpuIndexIVF::getCoarseCentroids(float* out) const {
    quantizer->reconstruct_n(0, nlist, out);
}

void GpuIndexIVF::setList(idx_t listId, idx_t len, const uint8_t* codes, const idx_t* ids) {
    DeviceScope scope(config_.device);
    idx_t before = lists_->listLength(listId);
    lists_->setListFromHost(listId, len, codes, ids, stream_());
    this->ntotal += len - before;
}

void GpuIndexIVF::trainQuantizer_(idx_t n, const float* xDev) {
    if (n == 0)
        return;
    if (quantizer->is_trained && quantizer->ntotal == nlist) {
        if (verbose)
            printf("IVF quantizer does not need training.\n");
        return;
    }
    if (verbose)
        printf("Training IVF quantizer on %ld vectors in %dD\n", (long)n, d);
    quantizer->reset();
    Clustering clus(d, (int)nlist, cp);
    clus.verbose = verbose;
    clus.train(n, xDev, *quantizer);
    quantizer->is_trained = true;
    coarseEpoch++;
    FB_THROW_IF_NOT(quantizer->ntotal == nlist);
}

void GpuIndexIVF::train(idx_t n, const float* x) {
    DeviceScope scope(config_.device);
    if (this->is_trained) {
        FB_THROW_IF_NOT(quantizer->is_trained && quantizer->ntotal == nlist);
        return;
    }
    DeviceView<float> xv(resources_.get(), config_.device, x, (size_t)n * d, stream_());
    trainQuantizer_(n, xv.ptr);
    trainEncoder_(n, xv.ptr);
    this->is_trained = true;
}

void GpuIndexIVF::addImpl_(idx_t n, const float* xDev, const idx_t* idsDev) {
    auto stream = stream_();
    auto assign = resources_->temp(config_.device, sizeof(idx_t) * n);
    auto dis = resources_->temp(config_.device, sizeof(float) * n);
    quantizer->searchDevice(n, xDev, 1, dis.as<float>(), assign.as<idx_t>());
    GpuMemoryReservation hold;
    const uint8_t* rows = encode_(n, xDev, assign.as<idx_t>(), hold);
    lists_->append(n, rows, idsDev, assign.as<idx_t>(), stream);
    // vectors that could not be assigned (NaN) are still counted, as upstream (IVFBase.cu addVectors)
    this->ntotal += n;
}

GpuMemoryReservation GpuIndexIVF::coarseResiduals_(idx_t n, const float* xDev, const idx_t* assignDev) const {
    GpuResources* res = resources_.get();
    const int device = config_.device;
    const bool training = assignDev == nullptr;
    auto alloc = [&](size_t bytes) {
        return training ? res->device_alloc(device, bytes, AllocType::Other) : res->temp(device, bytes);
    };
    auto resid = alloc(sizeof(float) * n * d);
    GpuMemoryReservation assign, dis;
    if (training) {
        assign = alloc(sizeof(idx_t) * n);
        dis = alloc(sizeof(float) * n);
        quantizer->searchDevice(n, xDev, 1, dis.as<float>(), assign.as<idx_t>());
        assignDev = assign.as<idx_t>();
    }
    runCalcResidual(xDev, quantizer->vectorsDevice(), assignDev, n, d, resid.as<float>(), stream_());
    return resid;
}

void GpuIndexIVF::searchImpl_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, const SearchCall& call) const {
    // per-call SearchParametersIVF override the index fields (faiss/gpu/GpuIndexIVF.cu:383-406)
    size_t use_nprobe = nprobe, use_max_codes = max_codes;
    if (call.params) {
        auto* ivfParams = dynamic_cast<const SearchParametersIVF*>(call.params);
        FB_THROW_IF_NOT_MSG(ivfParams != nullptr, "IVF search: search parameters must be SearchParametersIVF");
        use_nprobe = ivfParams->nprobe;
        use_max_codes = ivfParams->max_codes;
        FB_THROW_IF_NOT_MSG(ivfParams->quantizer_params == nullptr, "quantizer search parameters are not supported on the GPU path");
    }
    validateNProbe(use_nprobe);
    FB_THROW_IF_NOT_FMT(
            use_max_codes == 0,
            "GPU IVF index does not currently support max_codes (passed %zu, must be 0)",
            use_max_codes);
    const int np = (int)std::min<size_t>(use_nprobe, (size_t)nlist);
    auto cD = resources_->temp(config_.device, sizeof(float) * n * np);
    auto cI = resources_->temp(config_.device, sizeof(idx_t) * n * np);
    // coarse quantisation = a Flat search with k = nprobe over the centroids (IVFBase.cu:509-545)
    quantizer->searchDevice(n, xDev, np, cD.as<float>(), cI.as<idx_t>());
    scanImpl_(n, xDev, cI.as<idx_t>(), cD.as<float>(), np, k, dDev, iDev, call);
}

GpuMemoryReservation GpuIndexIVF::selMask_(const IDSelector& sel, idx_t&) const {
    const int64_t slots = lists_->arenaElems();
    auto mask = resources_->temp(config_.device, sizeof(uint32_t) * slotMaskWords(slots));
    std::vector<uint8_t> valid; // a callback is only called for the occupied slots
    if (sel.usesCallback()) {
        valid.assign((size_t)slots, 0);
        for (idx_t l = 0; l < nlist; l++)
            std::fill_n(valid.begin() + lists_->listStart(l), lists_->listLength(l), 1);
    }
    buildSlotMask(
            resources_.get(), config_.device, sel, slots, lists_->ids(), valid.empty() ? nullptr : valid.data(),
            mask.as<uint32_t>(), stream_());
    return mask;
}

void GpuIndexIVF::search_preassigned(
        idx_t n,
        const float* x,
        idx_t k,
        const idx_t* assign,
        const float* centroid_dis,
        float* distances,
        idx_t* labels) const {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(this->is_trained, "GpuIndexIVF not trained");
    validateKSelect(k);
    if (n == 0 || k == 0)
        return;
    validateNProbe(nprobe);
    auto stream = stream_();
    const int np = (int)nprobe;
    DeviceView<float> xv(resources_.get(), config_.device, x, (size_t)n * d, stream);
    DeviceView<idx_t> av(resources_.get(), config_.device, assign, (size_t)n * np, stream);
    DeviceView<float> cv(resources_.get(), config_.device, centroid_dis, (size_t)n * np, stream);
    DeviceOut<float> dv(resources_.get(), config_.device, distances, (size_t)n * k);
    DeviceOut<idx_t> lv(resources_.get(), config_.device, labels, (size_t)n * k);
    scanImpl_(n, xv.ptr, av.ptr, cv.ptr, np, (int)k, dv.ptr, lv.ptr, SearchCall());
    dv.finish(stream);
    lv.finish(stream);
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

// ---- retrieval: ids -> arena slots -> decoded entries (ivf_reconstruct.cu)
IvfStoredLayout GpuIndexIVF::listLayout_() const {
    IvfStoredLayout a;
    a.d = d;
    a.codeSize = lists_->codeSize();
    a.interleaved = lists_->interleaved();
    a.listStart = lists_->dStart();
    a.listLen = lists_->dLen();
    a.nlist = nlist;
    a.arenaElems = lists_->arenaElems();
    a.codes = lists_->codes();
    a.ids = lists_->ids();
    return a;
}

int GpuIndexIVF::coarse_code_size() const {
    int nbyte = 0;
    for (idx_t nl = nlist - 1; nl > 0; nl >>= 8)
        nbyte++;
    return nbyte;
}

// rows per call of the ids -> slots pass: all of them for a device output; pages of kRetrievalPageBytes for a host
// output, so the device staging stays bounded (each page repeats the pass over the stored ids)
idx_t GpuIndexIVF::retrievalPageRows_(const float* out, idx_t n) const {
    if (getDeviceForAddress(out) == config_.device)
        return std::max<idx_t>(n, 1);
    return std::max<idx_t>(1, (idx_t)(kRetrievalPageBytes / (sizeof(float) * d)));
}

void GpuIndexIVF::reconstruct_n(idx_t i0, idx_t ni, float* recons) const {
    FB_THROW_IF_NOT(ni == 0 || (i0 >= 0 && i0 + ni <= this->ntotal));
    if (ni == 0)
        return;
    DeviceScope scope(config_.device);
    auto stream = stream_();
    const IvfStoredLayout a = storedLayout_();
    const idx_t page = retrievalPageRows_(recons, ni);
    for (idx_t r0 = 0; r0 < ni; r0 += page) {
        const idx_t nr = std::min(page, ni - r0);
        auto slots = resources_->temp(config_.device, sizeof(idx_t) * nr);
        runIvfSlotsOfRange(a, i0 + r0, nr, slots.as<idx_t>(), stream);
        // rows of ids not stored keep the caller's contents: a staged page starts as a copy of them
        DeviceInOut<float> out(resources_.get(), config_.device, recons + (size_t)r0 * d, (size_t)nr * d, stream);
        runIvfReconstruct(a, slots.as<idx_t>(), nr, false, out.ptr, stream);
        out.finish(stream);
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
}

void GpuIndexIVF::reconstruct_batch(idx_t n, const idx_t* keys, float* recons) const {
    if (n == 0)
        return;
    DeviceScope scope(config_.device);
    auto stream = stream_();
    const IvfStoredLayout a = storedLayout_();
    DeviceView<idx_t> kv(resources_.get(), config_.device, keys, (size_t)n, stream);
    auto slots = resources_->temp(config_.device, sizeof(idx_t) * n);
    // every key is resolved before any row is written
    FB_THROW_IF_NOT_MSG(
            runIvfSlotsOfKeys(resources_.get(), config_.device, a, kv.ptr, n, slots.as<idx_t>(), stream), "key not found");
    const idx_t page = retrievalPageRows_(recons, n);
    for (idx_t r0 = 0; r0 < n; r0 += page) {
        const idx_t nr = std::min(page, n - r0);
        DeviceOut<float> out(resources_.get(), config_.device, recons + (size_t)r0 * d, (size_t)nr * d);
        runIvfReconstruct(a, slots.as<idx_t>() + r0, nr, true, out.ptr, stream);
        out.finish(stream);
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
}

void GpuIndexIVF::reconstruct(idx_t key, float* recons) const {
    reconstruct_batch(1, &key, recons);
}

void GpuIndexIVF::searchWithSlots_(
        idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, const SearchParameters* params,
        size_t resultBytes, const std::function<void(idx_t, idx_t, const idx_t*)>& page) const {
    DeviceScope scope(config_.device);
    const int64_t slotsTotal = lists_->arenaElems();
    auto identity = resources_->device_alloc(config_.device, sizeof(idx_t) * std::max<int64_t>(1, slotsTotal), AllocType::Other);
    runIvfIdentitySlots(identity.as<idx_t>(), slotsTotal, stream_());
    searchPaged_(n, x, k, distances, labels, params, resultBytes, [&](idx_t nb, const float* xDev, float* dDev, idx_t* iDev, const SearchCall& call) {
        auto slots = resources_->temp(config_.device, sizeof(idx_t) * nb * k);
        const IvfSlotOutput so{identity.as<idx_t>(), lists_->ids(), slots.as<idx_t>()};
        SearchCall withSlots = call;
        withSlots.slots = &so;
        searchImpl_(nb, xDev, (int)k, dDev, iDev, withSlots);
        page(call.row0, nb, slots.as<idx_t>());
    });
}

void GpuIndexIVF::search_and_reconstruct(
        idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, float* recons, const SearchParameters* params) const {
    FB_THROW_IF_NOT_MSG(n == 0 || recons, "null pointer passed to search_and_reconstruct");
    const IvfStoredLayout a = storedLayout_();
    searchWithSlots_(n, x, k, distances, labels, params, sizeof(float) * d, [&](idx_t i0, idx_t nb, const idx_t* slots) {
        auto stream = stream_();
        DeviceOut<float> rv(resources_.get(), config_.device, recons + (size_t)i0 * k * d, (size_t)nb * k * d);
        runIvfReconstruct(a, slots, nb * k, true, rv.ptr, stream);
        rv.finish(stream);
        CUDA_VERIFY(cudaStreamSynchronize(stream)); // the staging buffer dies here
    });
}

void GpuIndexIVF::search_and_return_codes(
        idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, uint8_t* codes, bool include_listno,
        const SearchParameters* params) const {
    FB_THROW_IF_NOT_MSG(n == 0 || codes, "null pointer passed to search_and_return_codes");
    const IvfStoredLayout a = listLayout_();
    const int listnoBytes = include_listno ? coarse_code_size() : 0;
    const size_t rowBytes = (size_t)listnoBytes + a.codeSize;
    searchWithSlots_(n, x, k, distances, labels, params, rowBytes, [&](idx_t i0, idx_t nb, const idx_t* slots) {
        auto stream = stream_();
        DeviceOut<uint8_t> cv(resources_.get(), config_.device, codes + (size_t)i0 * k * rowBytes, (size_t)nb * k * rowBytes);
        runIvfGatherCodes(a, slots, nb * k, listnoBytes, cv.ptr, stream);
        cv.finish(stream);
        CUDA_VERIFY(cudaStreamSynchronize(stream)); // the staging buffer dies here
    });
}

// ------------------------------------------------------------------------------------------
// GpuIndexIVFFlat
// ------------------------------------------------------------------------------------------
GpuIndexIVFFlat::GpuIndexIVFFlat(
        std::shared_ptr<GpuResources> resources,
        int dims,
        idx_t nlist,
        MetricType metric,
        GpuIndexIVFConfig config)
        : GpuIndexIVF(std::move(resources), dims, metric, nlist, (int)(sizeof(float) * dims), config) {}

GpuIndexIVFFlat::GpuIndexIVFFlat(
        std::shared_ptr<GpuResources> resources,
        GpuIndexFlat* coarseQuantizer,
        int dims,
        idx_t nlist,
        MetricType metric,
        GpuIndexIVFConfig config)
        : GpuIndexIVFFlat(std::move(resources), dims, nlist, metric, config) {
    setQuantizer(coarseQuantizer);
}

const uint8_t* GpuIndexIVFFlat::encode_(idx_t, const float* xDev, const idx_t*, GpuMemoryReservation&) {
    return reinterpret_cast<const uint8_t*>(xDev);
}

void GpuIndexIVFFlat::scanImpl_(
        idx_t n,
        const float* xDev,
        const idx_t* probes,
        const float*,
        int np,
        int k,
        float* dDev,
        idx_t* iDev,
        const SearchCall& call) const {
    runIvfFlatScan(
            resources_.get(), config_.device, xDev, n, d, probes, np, lists_->dStart(), lists_->dLen(),
            reinterpret_cast<const float*>(lists_->codes()), scanIds_(call), lists_->arenaElems(), k, metric_type, dDev,
            iDev, stream_(), call.mask, call.slots);
}

IvfStoredLayout GpuIndexIVFFlat::storedLayout_() const {
    IvfStoredLayout a = listLayout_();
    a.kind = IVF_STORED_FLAT;
    return a;
}

// ------------------------------------------------------------------------------------------
// GpuIndexIVFPQ
// ------------------------------------------------------------------------------------------
// device layout from (M, nbits): interleaved-by-32 for 8-bit codes with M in {16, 32} and for 4-bit codes whose
// M/2 nibble-pair bytes are 16 or 32; every other shape keeps the CPU's vector-major bitstring
static bool ivfPqInterleavedLayout(idx_t M, idx_t nbits) {
    if (nbits == 8)
        return ivfPqInterleavedSupported((int)M);
    return nbits == 4 && M % 2 == 0 && ivfPqInterleavedSupported((int)(M / 2));
}
// ProductQuantizer::code_size = ceil(M * nbits / 8) (faiss/impl/ProductQuantizer.cpp set_derived_values)
static int ivfPqCodeSize(idx_t M, idx_t nbits) {
    return nbits >= 1 && nbits <= 8 ? (int)((M * nbits + 7) / 8) : (int)M;
}

GpuIndexIVFPQ::GpuIndexIVFPQ(
        std::shared_ptr<GpuResources> resources,
        int dims,
        idx_t nlist,
        idx_t subQuantizers,
        idx_t bitsPerCode,
        MetricType metric,
        GpuIndexIVFPQConfig config)
        : GpuIndexIVF(
                  std::move(resources),
                  dims,
                  metric,
                  nlist,
                  ivfPqCodeSize(subQuantizers, bitsPerCode),
                  config,
                  ivfPqInterleavedLayout(subQuantizers, bitsPerCode)),
          M_((int)subQuantizers),
          nbits_((int)bitsPerCode),
          usePrecomputed_(config.usePrecomputedTables),
          precomputedExplicit_(config.usePrecomputedTables),
          term2_(resources_.get(), config.device, AllocType::Quantizer),
          pqCentroids_(resources_.get(), config.device, AllocType::Quantizer),
          pqCentroidsT_(resources_.get(), config.device, AllocType::Quantizer) {
    // faiss/gpu/GpuIndexIVFPQ.cu:124-131, verifyPQSettings_ :566-617 (the non-cuVS rules)
    if (config.interleavedLayout)
        FB_THROW_IF_NOT_FMT(
                bitsPerCode == 4 || bitsPerCode == 5 || bitsPerCode == 6 || bitsPerCode == 8,
                "Bits per code must be between 4, 5, 6 or 8 (passed %d)",
                (int)bitsPerCode);
    else
        FB_THROW_IF_NOT_MSG(bitsPerCode == 8, "GPU: only pq.nbits == 8 is supported");
    FB_THROW_IF_NOT_MSG(subQuantizers > 0 && dims % subQuantizers == 0,
                        "Number of sub-quantizers must be an integer divisor of the number of dimensions");
    FB_THROW_IF_NOT_MSG(nlist > 0, "nlist must be > 0");
    FB_THROW_IF_NOT_FMT(
            sizeof(float) * subQuantizers * (size_t(1) << bitsPerCode) <= 160 * 1024,
            "Number of sub-quantizers %d: lookup table does not fit shared memory",
            (int)subQuantizers);
}

GpuIndexIVFPQ::GpuIndexIVFPQ(
        std::shared_ptr<GpuResources> resources,
        GpuIndexFlat* coarseQuantizer,
        int dims,
        idx_t nlist,
        idx_t subQuantizers,
        idx_t bitsPerCode,
        MetricType metric,
        GpuIndexIVFPQConfig config)
        : GpuIndexIVFPQ(std::move(resources), dims, nlist, subQuantizers, bitsPerCode, metric, config) {
    setQuantizer(coarseQuantizer);
}

GpuIndexIVFPQ::~GpuIndexIVFPQ() {}

void GpuIndexIVFPQ::setPQCentroids(const float* c) {
    DeviceScope scope(config_.device);
    auto stream = stream_();
    const int ksub = ksub_();
    pqCentroids_.resize((size_t)ksub * d, stream);
    CUDA_VERIFY(cudaMemcpyAsync(pqCentroids_.data(), c, sizeof(float) * ksub * d, cudaMemcpyDefault, stream));
    // transposed copy [ksub][M][dsub]
    std::vector<float> h((size_t)ksub * d), ht((size_t)ksub * d);
    CUDA_VERIFY(cudaMemcpyAsync(h.data(), pqCentroids_.data(), sizeof(float) * ksub * d, cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    const int dsub = d / M_;
    for (int m = 0; m < M_; m++)
        for (int cc = 0; cc < ksub; cc++)
            memcpy(&ht[((size_t)cc * M_ + m) * dsub], &h[((size_t)m * ksub + cc) * dsub], sizeof(float) * dsub);
    pqCentroidsT_.resize((size_t)ksub * d, stream);
    CUDA_VERIFY(cudaMemcpyAsync(pqCentroidsT_.data(), ht.data(), sizeof(float) * ksub * d, cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    pqEpoch_++;
}

bool GpuIndexIVFPQ::precomputedActive_() const {
    if (nbits_ != 8 || metric_type != METRIC_L2 || !lists_->interleaved())
        return false;
    if (precomputedExplicit_)
        return usePrecomputed_;
    // auto: the CPU reference's size rule, and only with short lists: with long lists (N=100M / nlist=4096, 24k
    // vectors per list) the LUT build is a small share of the scan and the direct LUT needs no [nlist][256][M] table
    // reads; with short lists (nlist=65536) the LUT build dominates the CTA
    const size_t bytes = sizeof(float) * (size_t)nlist * 256 * M_;
    return bytes <= (size_t(1) << 31) && this->ntotal / nlist < 4096;
}

void GpuIndexIVFPQ::ensureTerm2_() const {
    const uint64_t key = (coarseEpoch << 32) ^ pqEpoch_;
    if (term2Key_ == key && term2_.size() == (size_t)nlist * 256 * M_)
        return;
    auto stream = stream_();
    term2_.resize((size_t)nlist * 256 * M_, stream);
    runIvfPqPrecomputeTerm2(quantizer->vectorsDevice(), pqCentroidsT_.data(), nlist, d, M_, term2_.data(), stream);
    term2Key_ = key;
}

void GpuIndexIVFPQ::getPQCentroids(float* out) const {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(pqCentroids_.size() > 0, "PQ not trained");
    auto stream = stream_();
    CUDA_VERIFY(cudaMemcpyAsync(out, pqCentroids_.data(), sizeof(float) * ksub_() * d, cudaMemcpyDefault, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

// ProductQuantizer::train, Train_default (faiss/impl/ProductQuantizer.cpp:130-195): M independent
// k-means on the column slices, each with a fresh Clustering(dsub, ksub, cp).  x: device [n, d];
// pqOut: host [M][ksub][dsub].
void trainProductQuantizer(
        std::shared_ptr<GpuResources> resources,
        int device,
        idx_t n,
        const float* xDev,
        int d,
        int M,
        int ksub,
        const ClusteringParameters& cp,
        float* pqOut) {
    GpuResources* res = resources.get();
    DeviceScope scope(device);
    cudaStream_t stream = res->getDefaultStream(device);
    const int dsub = d / M;
    auto slice = res->device_alloc(device, sizeof(float) * n * dsub, AllocType::Other);
    GpuIndexFlatConfig fc;
    fc.device = device;
    GpuIndexFlatL2 pqIndex(resources, dsub, fc);
    for (int m = 0; m < M; m++) {
        slice_cols_kernel<<<(unsigned)ceil_div(n * dsub, 256), 256, 0, stream>>>(xDev, n, d, m * dsub, dsub, slice.as<float>());
        CUDA_CHECK_LAST();
        Clustering clus(dsub, ksub, cp);
        clus.verbose = false;
        pqIndex.reset();
        clus.train(n, slice.as<float>(), pqIndex);
        memcpy(pqOut + (size_t)m * ksub * dsub, clus.centroids.data(), sizeof(float) * ksub * dsub);
    }
}

const float* subsampleRowsDevice(
        GpuResources* res,
        int device,
        idx_t& n,
        int d,
        idx_t nmax,
        int64_t seed,
        const float* xDev,
        GpuMemoryReservation& hold,
        cudaStream_t stream) {
    if (n <= nmax)
        return xDev;
    std::vector<int> perm(n);
    rand_perm(perm.data(), n, seed);
    auto pd = res->temp(device, sizeof(int) * nmax);
    CUDA_VERIFY(cudaMemcpyAsync(pd.data, perm.data(), sizeof(int) * nmax, cudaMemcpyHostToDevice, stream));
    hold = res->device_alloc(device, sizeof(float) * nmax * d, AllocType::Other);
    gather_rows_int_kernel<<<(unsigned)nmax, std::min(256, d), 0, stream>>>(xDev, pd.as<int>(), nmax, d, hold.as<float>());
    CUDA_CHECK_LAST();
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    n = nmax;
    return hold.as<float>();
}

void GpuIndexIVFPQ::trainEncoder_(idx_t n, const float* xDev) {
    auto stream = stream_();
    const int ksub = ksub_();
    // fvecs_maybe_subsample (faiss/utils/utils.cpp:464-489) with pq.cp.seed
    GpuMemoryReservation sub;
    const float* x = subsampleRowsDevice(
            resources_.get(), config_.device, n, d, (idx_t)pq_cp.max_points_per_centroid * ksub, pq_cp.seed, xDev,
            sub, stream);
    if (verbose)
        printf("computing residuals\n");
    auto resid = coarseResiduals_(n, x, nullptr);
    if (verbose)
        printf("training %d x %d product quantizer on %ld vectors in %dD\n", M_, ksub, (long)n, d);
    std::vector<float> pq((size_t)ksub * d);
    trainProductQuantizer(resources_, config_.device, n, resid.as<float>(), d, M_, ksub, pq_cp, pq.data());
    setPQCentroids(pq.data());
}

const uint8_t* GpuIndexIVFPQ::encode_(idx_t n, const float* xDev, const idx_t* assignDev, GpuMemoryReservation& hold) {
    FB_THROW_IF_NOT_MSG(pqCentroids_.size() > 0, "PQ not trained");
    auto stream = stream_();
    auto resid = coarseResiduals_(n, xDev, assignDev);
    hold = resources_->temp(config_.device, (size_t)n * M_);
    runPQEncode(resid.as<float>(), n, d, M_, ksub_(), pqCentroids_.data(), hold.as<uint8_t>(), stream);
    if (nbits_ != 8) {
        auto codes = std::move(hold);
        hold = resources_->temp(config_.device, (size_t)n * lists_->codeSize());
        runPQPack(codes.as<uint8_t>(), n, M_, nbits_, hold.as<uint8_t>(), stream);
    }
    return hold.as<uint8_t>();
}

void GpuIndexIVFPQ::scanImpl_(
        idx_t n,
        const float* xDev,
        const idx_t* probes,
        const float* coarseDis,
        int np,
        int k,
        float* dDev,
        idx_t* iDev,
        const SearchCall& call) const {
    FB_THROW_IF_NOT_MSG(pqCentroids_.size() > 0, "PQ not trained");
    if (lists_->interleaved()) {
        runIvfPqScanInterleaved(
                resources_.get(), config_.device, xDev, n, d, probes, coarseDis, np, quantizer->vectorsDevice(),
                pqCentroidsT_.data(), precomputedActive_() ? (ensureTerm2_(), term2_.data()) : nullptr,
                lists_->codeSize(), nibbleLayout_(), lists_->dStart(), lists_->dLen(), lists_->codes(), scanIds_(call),
                lists_->arenaElems(), k, metric_type, dDev, iDev, stream_(), call.mask, call.slots);
        return;
    }
    runIvfPqScan(
            resources_.get(), config_.device, xDev, n, d, probes, coarseDis, np, quantizer->vectorsDevice(),
            pqCentroids_.data(), M_, nbits_, lists_->dStart(), lists_->dLen(), lists_->codes(), scanIds_(call), k,
            metric_type, dDev, iDev, stream_(), call.mask, call.slots);
}

// IndexIVFPQ::reconstruct_from_offset (faiss/IndexIVFPQ.cpp:358-372): pq.decode, then + the list's centroid
IvfStoredLayout GpuIndexIVFPQ::storedLayout_() const {
    FB_THROW_IF_NOT_MSG(pqCentroids_.size() > 0, "PQ not trained");
    IvfStoredLayout a = listLayout_();
    a.kind = IVF_STORED_PQ;
    a.M = M_;
    a.nbits = nbits_;
    a.pq = pqCentroids_.data();
    a.centroids = quantizer->vectorsDevice();
    return a;
}

// ------------------------------------------------------------------------------------------
// GpuIndexIVFScalarQuantizer
// ------------------------------------------------------------------------------------------
static bool sqTypeSupported(int qtype) { // faiss/gpu/impl/GpuScalarQuantizer.cuh:20-33
    return qtype >= SQ_QT_8bit && qtype <= SQ_QT_6bit;
}
static bool sqUniform(int qtype) {
    return qtype == SQ_QT_8bit_uniform || qtype == SQ_QT_4bit_uniform;
}

int GpuIndexIVFScalarQuantizer::codeSizeFor(int qtype, int d) {
    FB_THROW_IF_NOT_MSG(sqTypeSupported(qtype), "Unsupported scalar QuantizerType on GPU");
    switch (qtype) {
        case SQ_QT_4bit:
        case SQ_QT_4bit_uniform:
            return (d + 1) / 2;
        case SQ_QT_6bit:
            return (d * 6 + 7) / 8;
        case SQ_QT_fp16:
            return 2 * d;
        default:
            return d;
    }
}

GpuIndexIVFScalarQuantizer::GpuIndexIVFScalarQuantizer(
        std::shared_ptr<GpuResources> resources,
        int dims,
        idx_t nlist,
        int qtype,
        MetricType metric,
        bool encodeResidual,
        GpuIndexIVFScalarQuantizerConfig config)
        : GpuIndexIVF(std::move(resources), dims, metric, nlist, codeSizeFor(qtype, dims), config),
          by_residual(encodeResidual),
          qtype_(qtype),
          params_(resources_.get(), config.device, AllocType::Quantizer) {
    // faiss/gpu/GpuIndexIVFScalarQuantizer.cu:97-124: the per-dimension decode tables live in shared memory
    const size_t maxTable = 200 * 1024;
    FB_THROW_IF_NOT_FMT(
            ivfSqScanTableBytes(dims) <= maxTable,
            "GpuIndexIVFScalarQuantizer: Insufficient shared memory available on the GPU with %d dimensions; "
            "maximum dimensions possible is %d",
            dims,
            (int)((maxTable / sizeof(float) - 4) / 2));
    if (trainedSize() == 0)
        setTrained(nullptr, 0);
}

GpuIndexIVFScalarQuantizer::GpuIndexIVFScalarQuantizer(
        std::shared_ptr<GpuResources> resources,
        GpuIndexFlat* coarseQuantizer,
        int dims,
        idx_t nlist,
        int qtype,
        MetricType metric,
        bool encodeResidual,
        GpuIndexIVFScalarQuantizerConfig config)
        : GpuIndexIVFScalarQuantizer(std::move(resources), dims, nlist, qtype, metric, encodeResidual, config) {
    setQuantizer(coarseQuantizer);
}

size_t GpuIndexIVFScalarQuantizer::trainedSize() const {
    switch (qtype_) {
        case SQ_QT_8bit_uniform:
        case SQ_QT_4bit_uniform:
            return 2;
        case SQ_QT_8bit:
        case SQ_QT_4bit:
        case SQ_QT_6bit:
            return 2 * (size_t)d;
        default:
            return 0;
    }
}

void GpuIndexIVFScalarQuantizer::setTrained(const float* t, size_t n) {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_FMT(n == trainedSize(), "scalar quantizer expects %zu trained values, got %zu", trainedSize(), n);
    trained_.assign(t, t + n);
    // host tables [4][d]: vmin | vdiff for the encoder (the CPU's values), m | b for the scan's folded decode
    std::vector<float> h((size_t)4 * d);
    float* vmin = h.data();
    float* vdiff = vmin + d;
    float* m = vdiff + d;
    float* b = m + d;
    const float levels = (qtype_ == SQ_QT_4bit || qtype_ == SQ_QT_4bit_uniform) ? 15.f : qtype_ == SQ_QT_6bit ? 63.f : 255.f;
    for (int i = 0; i < d; i++) {
        if (n == 0) { // fp16, 8bit_direct: the code is the value
            vmin[i] = 0.f;
            vdiff[i] = 1.f;
            m[i] = 0.f;
            b[i] = 1.f;
            continue;
        }
        vmin[i] = sqUniform(qtype_) ? trained_[0] : trained_[i];
        vdiff[i] = sqUniform(qtype_) ? trained_[1] : trained_[d + i];
        b[i] = vdiff[i] / levels;
        m[i] = vmin[i] + 0.5f * b[i];
    }
    auto stream = stream_();
    params_.resize(h.size(), stream);
    CUDA_VERIFY(cudaMemcpyAsync(params_.data(), h.data(), sizeof(float) * h.size(), cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

void GpuIndexIVFScalarQuantizer::train(idx_t n, const float* x) {
    if (!this->is_trained)
        FB_THROW_IF_NOT_MSG(
                trainedSize() == 0 || rangestat == 0, "GpuIndexIVFScalarQuantizer: only RS_minmax training runs on the GPU");
    GpuIndexIVF::train(n, x);
}

// IndexIVF::train (faiss/IndexIVF.cpp:1296-1329) with train_encoder_num_vectors() = 100000
// (faiss/IndexScalarQuantizer.cpp:158-160) and ScalarQuantizer::train, RS_minmax
void GpuIndexIVFScalarQuantizer::trainEncoder_(idx_t n, const float* xDev) {
    const size_t nt = trainedSize();
    if (nt == 0)
        return;
    FB_THROW_IF_NOT(n > 0);
    auto stream = stream_();
    GpuResources* res = resources_.get();
    const int device = config_.device;
    GpuMemoryReservation sub;
    idx_t ns = n;
    const float* xs = subsampleRowsDevice(res, device, ns, d, 100000, 1234, xDev, sub, stream);
    GpuMemoryReservation resid;
    if (by_residual) {
        resid = coarseResiduals_(ns, xs, nullptr);
        xs = resid.as<float>();
    }
    auto mm = res->temp(device, sizeof(float) * 2 * d);
    runSqMinMax(xs, ns, d, mm.as<float>(), mm.as<float>() + d, stream);
    std::vector<float> h((size_t)2 * d);
    CUDA_VERIFY(cudaMemcpyAsync(h.data(), mm.data, sizeof(float) * 2 * d, cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    std::vector<float> t(nt);
    // training.cpp:221-234 (uniform: one range over all n*d values) and :345-365 (per dimension)
    if (sqUniform(qtype_)) {
        float vmin = HUGE_VALF, vmax = -HUGE_VALF;
        for (int j = 0; j < d; j++) {
            vmin = std::min(vmin, h[j]);
            vmax = std::max(vmax, h[d + j]);
        }
        const float vexp = (vmax - vmin) * rangestat_arg;
        vmin -= vexp;
        vmax += vexp;
        t[0] = vmin;
        t[1] = vmax - vmin;
    } else {
        for (int j = 0; j < d; j++) {
            float vmin = h[j], vmax = h[d + j];
            const float vexp = (vmax - vmin) * rangestat_arg;
            vmin -= vexp;
            vmax += vexp;
            t[j] = vmin;
            t[d + j] = vmax - vmin;
        }
    }
    setTrained(t.data(), nt);
}

const uint8_t* GpuIndexIVFScalarQuantizer::encode_(
        idx_t n, const float* xDev, const idx_t* assignDev, GpuMemoryReservation& hold) {
    FB_THROW_IF_NOT_MSG(params_.size() == (size_t)4 * d, "scalar quantizer not trained");
    GpuMemoryReservation resid;
    if (by_residual) { // IndexIVFScalarQuantizer::encode_vectors (faiss/IndexScalarQuantizer.cpp:162-200)
        resid = coarseResiduals_(n, xDev, assignDev);
        xDev = resid.as<float>();
    }
    hold = resources_->temp(config_.device, (size_t)n * lists_->codeSize());
    runSqEncode(
            xDev, n, d, qtype_, lists_->codeSize(), params_.data(), params_.data() + d, hold.as<uint8_t>(), stream_());
    return hold.as<uint8_t>();
}

void GpuIndexIVFScalarQuantizer::scanImpl_(
        idx_t n,
        const float* xDev,
        const idx_t* probes,
        const float* coarseDis,
        int np,
        int k,
        float* dDev,
        idx_t* iDev,
        const SearchCall& call) const {
    FB_THROW_IF_NOT_MSG(params_.size() == (size_t)4 * d, "scalar quantizer not trained");
    const bool needCentroids = by_residual && metric_type == METRIC_L2;
    runIvfSqScan(
            resources_.get(), config_.device, xDev, n, d, probes, coarseDis, np,
            needCentroids ? quantizer->vectorsDevice() : nullptr, by_residual, qtype_, params_.data() + 2 * d,
            lists_->dStart(), lists_->dLen(), lists_->codes(), scanIds_(call), lists_->arenaElems(), lists_->codeSize(), k,
            metric_type, dDev, iDev, stream_(), call.mask, call.slots);
}

// IndexIVFScalarQuantizer::reconstruct_from_offset (faiss/IndexScalarQuantizer.cpp:400-425): sq.decode, then + the
// list's centroid when by_residual
IvfStoredLayout GpuIndexIVFScalarQuantizer::storedLayout_() const {
    FB_THROW_IF_NOT_MSG(params_.size() == (size_t)4 * d, "scalar quantizer not trained");
    IvfStoredLayout a = listLayout_();
    a.kind = IVF_STORED_SQ;
    const bool nibble = qtype_ == SQ_QT_4bit || qtype_ == SQ_QT_4bit_uniform;
    a.sqCodec = nibble ? SQC_NIBBLE : qtype_ == SQ_QT_6bit ? SQC_SIX : qtype_ == SQ_QT_fp16 ? SQC_HALF : SQC_BYTE;
    a.levels = qtype_ == SQ_QT_fp16 || qtype_ == SQ_QT_8bit_direct ? 0.f : nibble ? 15.f : qtype_ == SQ_QT_6bit ? 63.f : 255.f;
    a.vmin = params_.data();
    a.vdiff = params_.data() + d;
    a.centroids = by_residual ? quantizer->vectorsDevice() : nullptr;
    return a;
}

// ------------------------------------------------------------------------------------------
// GpuIndexCagra
// ------------------------------------------------------------------------------------------
GpuIndexCagra::GpuIndexCagra(std::shared_ptr<GpuResources> resources, int dims, MetricType metric, GpuIndexCagraConfig config)
        : GpuIndex(std::move(resources), dims, metric, 0.f, config),
          cagraConfig_(config),
          data_(resources_.get(), config.device, AllocType::FlatData),
          graph_(resources_.get(), config.device, AllocType::Other) {
    FB_THROW_IF_NOT_MSG(
            metric == METRIC_L2 || metric == METRIC_INNER_PRODUCT,
            "GpuIndexCagra supports METRIC_L2 and METRIC_INNER_PRODUCT only");
    this->is_trained = false;
}

void GpuIndexCagra::train(idx_t n, const float* x) {
    DeviceScope scope(config_.device);
    if (this->is_trained)
        return;
    const GpuIndexCagraConfig& c = cagraConfig_;
    FB_THROW_IF_NOT_MSG(
            c.build_algo == graph_build_algo::IVF_PQ,
            "GpuIndexCagra builds with graph_build_algo IVF_PQ only (NN_DESCENT and ITERATIVE_SEARCH are not implemented)");
    FB_THROW_IF_NOT_MSG(!c.guarantee_connectivity, "GpuIndexCagra: guarantee_connectivity is not implemented");
    FB_THROW_IF_NOT_MSG(c.store_dataset, "GpuIndexCagra: store_dataset = false is not implemented (the search reads the stored rows)");
    FB_THROW_IF_NOT_MSG(
            c.ivf_pq_params.codebook_kind == codebook_gen::PER_SUBSPACE,
            "GpuIndexCagra: codebook_kind PER_CLUSTER is not implemented");
    FB_THROW_IF_NOT_MSG(!c.ivf_pq_params.force_random_rotation, "GpuIndexCagra: force_random_rotation is not implemented");
    FB_THROW_IF_NOT_MSG(c.refine_rate >= 1.f, "GpuIndexCagra: refine_rate must be >= 1");
    FB_THROW_IF_NOT_MSG(n >= 2, "GpuIndexCagra needs at least 2 vectors to build a graph");
    FB_THROW_IF_NOT_MSG(n < (idx_t(1) << 31) - 1, "GpuIndexCagra holds fewer than 2^31 - 1 vectors");
    FB_THROW_IF_NOT_MSG(c.graph_degree >= 1, "GpuIndexCagra: graph_degree must be >= 1");
    // K0 <= N - 1 (a row has no more distinct neighbours) and K <= K0 (the prune only drops edges)
    const int K0 = (int)std::min<idx_t>((idx_t)c.intermediate_graph_degree, n - 1);
    const int K = (int)std::min<idx_t>((idx_t)c.graph_degree, K0);
    FB_THROW_IF_NOT_FMT(K0 <= 1024, "GpuIndexCagra: intermediate_graph_degree %d > 1024", K0);
    auto stream = stream_();
    try {
        DeviceView<float> xv(resources_.get(), config_.device, x, (size_t)n * d, stream);
        data_.clear();
        data_.reserve((size_t)n * d, stream, true);
        data_.append(xv.ptr, (size_t)n * d, stream);
        cagraBuildGraph(resources_, config_.device, data_.data(), n, d, metric_type, c, K0, K, graph_, lastBuildSeconds);
    } catch (...) {
        reset();
        throw;
    }
    graphDegree_ = K;
    this->ntotal = n;
    this->is_trained = true;
}

void GpuIndexCagra::add(idx_t n, const float* x) {
    train(n, x);
}

void GpuIndexCagra::addImpl_(idx_t, const float*, const idx_t*) {
    FB_THROW_MSG("adding vectors is not supported by GpuIndexCagra.");
}

void GpuIndexCagra::reset() {
    DeviceScope scope(config_.device);
    data_.clear();
    graph_.clear();
    graphDegree_ = 0;
    this->ntotal = 0;
    this->is_trained = false;
}

void GpuIndexCagra::copyFrom(idx_t n, const float* xb, const idx_t* graph, int degree) {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(n >= 1 && n < (idx_t(1) << 31) - 1, "GpuIndexCagra::copyFrom: bad number of vectors");
    FB_THROW_IF_NOT_MSG(degree >= 1, "GpuIndexCagra::copyFrom: graph degree must be >= 1");
    auto stream = stream_();
    std::vector<idx_t> g((size_t)n * degree);
    CUDA_VERIFY(cudaMemcpy(g.data(), graph, g.size() * sizeof(idx_t), cudaMemcpyDefault));
    std::vector<uint32_t> g32(g.size());
    for (size_t i = 0; i < g.size(); i++) {
        FB_THROW_IF_NOT_FMT(g[i] >= -1 && g[i] < n, "GpuIndexCagra::copyFrom: graph entry %ld out of range", (long)g[i]);
        g32[i] = g[i] < 0 ? 0xFFFFFFFFu : (uint32_t)g[i];
    }
    reset();
    DeviceView<float> xv(resources_.get(), config_.device, xb, (size_t)n * d, stream);
    data_.reserve((size_t)n * d, stream, true);
    data_.append(xv.ptr, (size_t)n * d, stream);
    graph_.reserve(g32.size(), stream, true);
    graph_.append(g32.data(), g32.size(), stream);
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    graphDegree_ = degree;
    this->ntotal = n;
    this->is_trained = true;
}

std::vector<idx_t> GpuIndexCagra::get_knngraph() const {
    DeviceScope scope(config_.device);
    FB_THROW_IF_NOT_MSG(this->is_trained, "GpuIndexCagra: the index is not built");
    std::vector<uint32_t> g32(graph_.size());
    CUDA_VERIFY(cudaMemcpy(g32.data(), graph_.data(), g32.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    std::vector<idx_t> g(g32.size());
    for (size_t i = 0; i < g.size(); i++)
        g[i] = g32[i] == 0xFFFFFFFFu ? -1 : (idx_t)g32[i];
    return g;
}

void GpuIndexCagra::copyTo(float* xb, idx_t* graph) const {
    auto g = get_knngraph();
    DeviceScope scope(config_.device);
    CUDA_VERIFY(cudaMemcpy(xb, data_.data(), sizeof(float) * (size_t)ntotal * d, cudaMemcpyDefault));
    CUDA_VERIFY(cudaMemcpy(graph, g.data(), sizeof(idx_t) * g.size(), cudaMemcpyDefault));
}

GpuMemoryReservation GpuIndexCagra::selMask_(const IDSelector&, idx_t&) const {
    FB_THROW_MSG("GpuIndexCagra does not support SearchParameters::sel");
}

void GpuIndexCagra::searchImpl_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, const SearchCall& call) const {
    const SearchParametersCagra defaults;
    const auto* sp = dynamic_cast<const SearchParametersCagra*>(call.params);
    if (!sp)
        sp = &defaults;
    FB_THROW_IF_NOT_MSG(
            sp->algo == search_algo::SINGLE_CTA || sp->algo == search_algo::AUTO,
            "GpuIndexCagra implements search_algo SINGLE_CTA (and AUTO) only; MULTI_CTA and MULTI_KERNEL are not implemented");
    FB_THROW_IF_NOT_FMT(sp->itopk_size <= 512, "GpuIndexCagra: itopk_size %zu > 512", sp->itopk_size);
    FB_THROW_IF_NOT_FMT((size_t)k <= sp->itopk_size, "GpuIndexCagra: k %d > itopk_size %zu", k, sp->itopk_size);
    FB_THROW_IF_NOT_MSG(sp->search_width >= 1, "GpuIndexCagra: search_width must be >= 1");
    FB_THROW_IF_NOT_MSG(sp->num_random_samplings >= 1, "GpuIndexCagra: num_random_samplings must be >= 1");
    FB_THROW_IF_NOT_MSG(
            sp->team_size == 0 || sp->team_size == 4 || sp->team_size == 8 || sp->team_size == 16 || sp->team_size == 32,
            "GpuIndexCagra: team_size must be 0, 4, 8, 16 or 32");
    FB_THROW_IF_NOT_MSG(
            sp->thread_block_size == 0 || sp->thread_block_size == 64 || sp->thread_block_size == 128 ||
                    sp->thread_block_size == 256 || sp->thread_block_size == 512 || sp->thread_block_size == 1024,
            "GpuIndexCagra: thread_block_size must be 0, 64, 128, 256, 512 or 1024");
    FB_THROW_IF_NOT_MSG(
            sp->hashmap_max_fill_rate >= 0.1f && sp->hashmap_max_fill_rate <= 0.9f,
            "GpuIndexCagra: hashmap_max_fill_rate must be in [0.1, 0.9]");
    FB_THROW_IF_NOT_MSG(sp->hashmap_min_bitlen <= 16, "GpuIndexCagra: hashmap_min_bitlen must be <= 16");

    CagraSearchArgs a{};
    a.data = data_.data();
    a.graph = graph_.data();
    a.n = ntotal;
    a.d = d;
    a.graphDegree = graphDegree_;
    a.metric = metric_type;
    a.k = k;
    a.itopk = (int)round_up(std::max<size_t>(sp->itopk_size, 1), 32);
    a.bufSize = next_pow2(a.itopk);
    a.searchWidth = (int)sp->search_width;
    const int64_t gather = (int64_t)a.searchWidth * a.graphDegree;
    const int64_t numInit = (int64_t)sp->num_random_samplings * gather;
    FB_THROW_IF_NOT_FMT(gather <= 4096, "GpuIndexCagra: search_width * graph_degree = %ld > 4096", (long)gather);
    FB_THROW_IF_NOT_FMT(numInit <= 8192, "GpuIndexCagra: num_random_samplings * search_width * graph_degree = %ld > 8192", (long)numInit);
    a.numInit = (int)numInit;
    a.candSize = next_pow2((int)std::max(numInit, gather));
    // automatic cap: twice the iterations that expand every itopk entry once, plus a margin
    const size_t autoIter = 2 * (size_t)a.itopk / a.searchWidth + 16;
    a.maxIterations = (int)std::min<size_t>(std::max(sp->max_iterations ? sp->max_iterations : autoIter, sp->min_iterations), 1 << 20);
    a.teamSize = sp->team_size ? (int)sp->team_size : std::min(32, std::max(4, next_pow2((d + 15) / 16)));
    a.blockSize = sp->thread_block_size ? (int)sp->thread_block_size : (a.itopk <= 64 ? 64 : a.itopk <= 256 ? 128 : 256);
    // the visited set holds every id inserted between two refills: at least the initial samples, and itopk plus a few
    // iterations of gathers
    const double need = std::max<double>((double)numInit + a.itopk, 4.0 * (a.itopk + gather));
    int bits = std::max<int>(8, (int)sp->hashmap_min_bitlen);
    while ((double)(1 << bits) * sp->hashmap_max_fill_rate < need)
        bits++;
    FB_THROW_IF_NOT_FMT(bits <= 16, "GpuIndexCagra: the visited set would need 2^%d entries", bits);
    a.hashBits = bits;
    a.hashLimit = (int)((double)(1 << bits) * sp->hashmap_max_fill_rate);
    a.seed = sp->seed;
    FB_THROW_IF_NOT_MSG(cagraSearchSmemBytes(a) <= 227 * 1024, "GpuIndexCagra: the search does not fit shared memory");

    auto stream = stream_();
    auto count = resources_->temp(config_.device, sizeof(unsigned long long));
    CUDA_VERIFY(cudaMemsetAsync(count.data, 0, sizeof(unsigned long long), stream));
    a.distanceCount = count.as<unsigned long long>();
    const idx_t batch = sp->max_queries ? (idx_t)sp->max_queries : n;
    for (idx_t b0 = 0; b0 < n; b0 += batch) {
        InterruptCallback::check(); // between query batches
        a.queries = xDev + (size_t)b0 * d;
        a.nq = std::min(batch, n - b0);
        a.rowOffset = call.row0 + b0;
        a.outD = dDev + (size_t)b0 * k;
        a.outI = iDev + (size_t)b0 * k;
        runCagraSearch(a, stream);
    }
    unsigned long long hCount = 0;
    CUDA_VERIFY(cudaMemcpyAsync(&hCount, count.data, sizeof(hCount), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    if (call.row0 == 0)
        lastSearchDistanceCount = 0;
    lastSearchDistanceCount += (int64_t)hCount;
}

// ------------------------------------------------------------------------------------------
// IndexShards
// ------------------------------------------------------------------------------------------
IndexShards::IndexShards(int d_, bool threaded_, bool successive_ids_)
        : Index(d_), threaded(threaded_), successive_ids(successive_ids_) {}

IndexShards::~IndexShards() {
    if (own_indices)
        for (auto* s : shards_)
            delete s;
}

void IndexShards::add_shard(Index* idx) {
    if (shards_.empty() && d == 0)
        d = idx->d;
    FB_THROW_IF_NOT_FMT(idx->d == d || d == 0, "addIndex: dimension mismatch for newly added index; expecting dim %d, new index has dim %d", d, idx->d);
    if (!shards_.empty()) {
        FB_THROW_IF_NOT_MSG(idx->metric_type == shards_[0]->metric_type, "addIndex: newly added index is of different metric type than old index");
    }
    shards_.push_back(idx);
    syncWithSubIndexes();
}

void IndexShards::remove_shard(Index* idx) {
    auto it = std::find(shards_.begin(), shards_.end(), idx);
    if (it != shards_.end())
        shards_.erase(it);
    syncWithSubIndexes();
}

void IndexShards::syncWithSubIndexes() { // faiss/IndexShards.cpp:87-111
    if (shards_.empty()) {
        is_trained = false;
        ntotal = 0;
        return;
    }
    metric_type = shards_[0]->metric_type;
    is_trained = shards_[0]->is_trained;
    ntotal = 0;
    for (auto* s : shards_) {
        FB_THROW_IF_NOT(metric_type == s->metric_type);
        FB_THROW_IF_NOT(d == s->d);
        FB_THROW_IF_NOT(is_trained == s->is_trained);
        ntotal += s->ntotal;
    }
}

template <typename F>
void IndexShards::runOnIndex(F f) const {
    // one worker per shard when threaded (faiss/impl/ThreadedIndex-inl.h:119-194); exceptions are
    // collected and the first is rethrown with the shard number
    const int ns = (int)shards_.size();
    std::vector<std::string> errors(ns);
    std::vector<char> failed(ns, 0);
    auto body = [&](int i) {
        try {
            f(i, shards_[i]);
        } catch (const std::exception& e) {
            failed[i] = 1;
            errors[i] = e.what();
        }
    };
    if (threaded && ns > 1) {
        std::vector<std::thread> th;
        for (int i = 0; i < ns; i++)
            th.emplace_back(body, i);
        for (auto& t : th)
            t.join();
    } else {
        for (int i = 0; i < ns; i++)
            body(i);
    }
    for (int i = 0; i < ns; i++) {
        if (failed[i])
            FB_THROW_FMT("Exception thrown from index %d: %s", i, errors[i].c_str());
    }
}

void IndexShards::train(idx_t n, const float* x) {
    // every shard trains on the full set (faiss/IndexShards.cpp:113-128)
    runOnIndex([n, x](int, Index* s) { s->train(n, x); });
    syncWithSubIndexes();
}

void IndexShards::add(idx_t n, const float* x) {
    add_with_ids(n, x, nullptr);
}

void IndexShards::add_with_ids(idx_t n, const float* x, const idx_t* xids) {
    // faiss/IndexShards.cpp:135-195
    FB_THROW_IF_NOT_MSG(!(successive_ids && xids), "It makes no sense to pass in ids and request them to be shifted");
    if (successive_ids) {
        FB_THROW_IF_NOT_MSG(!xids, "It makes no sense to pass in ids and request them to be shifted");
        FB_THROW_IF_NOT_MSG(this->ntotal == 0, "when adding to IndexShards with successive_ids, only add() in a single pass is supported");
    }
    const idx_t nshard = count();
    std::vector<idx_t> aids;
    const idx_t* ids = xids;
    if (!ids && !successive_ids) {
        aids.resize(n);
        for (idx_t i = 0; i < n; i++)
            aids[i] = this->ntotal + i;
        ids = aids.data();
    }
    const int dd = d;
    runOnIndex([n, ids, x, nshard, dd](int no, Index* index) {
        idx_t i0 = (idx_t)no * n / nshard;
        idx_t i1 = ((idx_t)no + 1) * n / nshard;
        const float* x0 = x + i0 * dd;
        if (index->verbose)
            printf("begin add shard %d on %ld points\n", no, (long)n);
        if (ids)
            index->add_with_ids(i1 - i0, x0, ids + i0);
        else
            index->add(i1 - i0, x0);
    });
    syncWithSubIndexes();
}

void IndexShards::reset() {
    runOnIndex([](int, Index* s) { s->reset(); });
    syncWithSubIndexes();
}

void merge_knn_results_host(
        idx_t n,
        idx_t k,
        int nshard,
        MetricType metric,
        const float* all_distances,
        const idx_t* all_labels,
        float* distances,
        idx_t* labels) {
    // S-way merge of sorted per-shard lists, ties -> smaller id; -1 labels are skipped
    // (faiss/utils/Heap.cpp:166-238)
    if (k == 0)
        return;
    const bool l2 = !is_similarity_metric(metric); // lower is better (faiss/IndexShards.cpp:246 tests METRIC_L2 only)
    const size_t stride = (size_t)n * k;
    for (idx_t i = 0; i < n; i++) {
        std::vector<idx_t> ptr(nshard, 0);
        for (idx_t j = 0; j < k; j++) {
            int bestS = -1;
            float bestD = 0;
            idx_t bestI = -1;
            for (int s = 0; s < nshard; s++) {
                if (ptr[s] >= k)
                    continue;
                const float* D = all_distances + stride * s + (size_t)i * k;
                const idx_t* I = all_labels + stride * s + (size_t)i * k;
                if (I[ptr[s]] < 0)
                    continue;
                float dv = D[ptr[s]];
                idx_t iv = I[ptr[s]];
                bool better = bestS < 0 || (l2 ? dv < bestD : dv > bestD) || (dv == bestD && iv < bestI);
                if (better) {
                    bestS = s;
                    bestD = dv;
                    bestI = iv;
                }
            }
            if (bestS < 0) {
                distances[(size_t)i * k + j] = l2 ? FLT_MAX : -FLT_MAX;
                labels[(size_t)i * k + j] = -1;
            } else {
                distances[(size_t)i * k + j] = bestD;
                labels[(size_t)i * k + j] = bestI;
                ptr[bestS]++;
            }
        }
    }
}

void IndexShards::search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const {
    // faiss/IndexShards.cpp:197-264
    FB_THROW_IF_NOT(k > 0);
    const idx_t nshard = count();
    FB_THROW_IF_NOT_MSG(nshard > 0, "no shards");
    lastSearchPath = 0;
    if (ncclFastPath_(n, x, k, distances, labels)) {
        lastSearchPath = 1;
        return;
    }
    std::vector<idx_t> translations(nshard, 0);
    if (successive_ids) {
        translations[0] = 0;
        for (idx_t s = 0; s + 1 < nshard; s++)
            translations[s + 1] = translations[s] + shards_[s]->ntotal;
    }
    std::vector<float> all_distances((size_t)nshard * k * n);
    std::vector<idx_t> all_labels((size_t)nshard * k * n);
    float* ad = all_distances.data();
    idx_t* al = all_labels.data();
    runOnIndex([n, k, x, ad, al, &translations](int no, Index* index) {
        if (index->verbose)
            printf("begin query shard %d on %ld points\n", no, (long)n);
        index->search(n, x, k, ad + (size_t)no * k * n, al + (size_t)no * k * n);
        idx_t tr = translations[no];
        if (tr != 0) {
            idx_t* l = al + (size_t)no * k * n;
            for (idx_t i = 0; i < n * k; i++)
                if (l[i] >= 0)
                    l[i] += tr;
        }
    });
    merge_knn_results_host(n, k, (int)nshard, metric_type, ad, al, distances, labels);
}


// ------------------------------------------------------------------------------------------
// IndexShardsIVF
// ------------------------------------------------------------------------------------------
IndexShardsIVF::IndexShardsIVF(GpuIndexFlat* quantizer_, idx_t nlist_, bool threaded_, bool successive_ids_)
        : IndexShards(quantizer_ ? quantizer_->d : 0, threaded_, successive_ids_), quantizer(quantizer_), nlist(nlist_) {
    FB_THROW_IF_NOT_MSG(quantizer != nullptr, "null quantizer");
    metric_type = quantizer->metric_type;
}

void IndexShardsIVF::add_shard(Index* idx) {
    auto* ivf = dynamic_cast<GpuIndexIVF*>(idx);
    FB_THROW_IF_NOT_MSG(ivf != nullptr, "IndexShardsIVF: shards must be IVF indexes");
    FB_THROW_IF_NOT_MSG(ivf->nlist == nlist, "IndexShardsIVF: shard has a different nlist");
    IndexShards::add_shard(idx);
}

void IndexShardsIVF::search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const {
    FB_THROW_IF_NOT(k > 0);
    const int nshard = count();
    FB_THROW_IF_NOT_MSG(nshard > 0, "no shards");
    lastSearchPath = 0;
    auto* index0 = dynamic_cast<GpuIndexIVF*>(shards_[0]);
    const idx_t nprobe = std::min<idx_t>((idx_t)index0->nprobe, nlist);
    // ONE coarse quantisation for all shards (faiss/IndexShardsIVF.cpp:183-188)
    std::vector<float> Dq((size_t)n * nprobe);
    std::vector<idx_t> Iq((size_t)n * nprobe);
    quantizer->search(n, x, nprobe, Dq.data(), Iq.data());
    std::vector<idx_t> translations(nshard, 0);
    if (successive_ids)
        for (int s = 0; s + 1 < nshard; s++)
            translations[s + 1] = translations[s] + shards_[s]->ntotal;
    std::vector<float> all_distances((size_t)nshard * k * n);
    std::vector<idx_t> all_labels((size_t)nshard * k * n);
    float* ad = all_distances.data();
    idx_t* al = all_labels.data();
    const float* dq = Dq.data();
    const idx_t* iq = Iq.data();
    runOnIndex([=, &translations](int no, Index* indexIn) {
        auto* index = dynamic_cast<GpuIndexIVF*>(indexIn);
        FB_THROW_IF_NOT_MSG((idx_t)index->nprobe == nprobe, "inconsistent nprobe (every shard must use the same nprobe <= nlist)");
        index->search_preassigned(n, x, k, iq, dq, ad + (size_t)no * k * n, al + (size_t)no * k * n);
        const idx_t tr = translations[no];
        if (tr != 0) {
            idx_t* l = al + (size_t)no * k * n;
            for (idx_t i = 0; i < n * k; i++)
                if (l[i] >= 0)
                    l[i] += tr;
        }
    });
    merge_knn_results_host(n, k, nshard, metric_type, ad, al, distances, labels);
}

// ------------------------------------------------------------------------------------------
// DistributedIndexShards
// ------------------------------------------------------------------------------------------
DistributedIndexShards::DistributedIndexShards(std::shared_ptr<GpuResources> resources, GpuIndex* local, bool successive)
        : Index(local->d, local->metric_type), successive_ids(successive), resources_(std::move(resources)), local_(local) {
    FB_THROW_IF_NOT_MSG(local_ != nullptr, "null local shard");
    comm_ = resources_->getCommunicator(local_->getDevice());
    FB_THROW_IF_NOT_MSG(
            comm_ != nullptr,
            "no NCCL communicator for the shard's device: call ncclInitRank / ncclInitAll on the resources first");
    syncWithSubIndexes();
}

DistributedIndexShards::~DistributedIndexShards() {
    if (dOffsets_) {
        DeviceScope scope(local_->getDevice());
        cudaFree(dOffsets_);
    }
    if (own_local)
        delete local_;
}

int DistributedIndexShards::rank() const {
    return comm_->rank();
}
int DistributedIndexShards::worldSize() const {
    return comm_->size();
}

void DistributedIndexShards::syncWithSubIndexes() {
    const int device = local_->getDevice();
    DeviceScope scope(device);
    cudaStream_t stream = resources_->getDefaultStream(device);
    // one tiny collective: every rank's (ntotal, "can take the pooled tensor-core path") pair
    const bool flatTc = dynamic_cast<GpuIndexFlat*>(local_) != nullptr && local_->shardPoolingEligible(1, 16);
    std::vector<int64_t> v = comm_->allGatherHostI64(local_->ntotal * 2 + (flatTc ? 1 : 0), stream);
    const int S = comm_->size();
    sizes_.assign(S, 0);
    allFlatTc_ = true;
    this->ntotal = 0;
    maxTiles_ = 0;
    std::vector<idx_t> offs(S, 0);
    idx_t run = 0;
    for (int r = 0; r < S; r++) {
        sizes_[r] = v[r] >> 1;
        allFlatTc_ = allFlatTc_ && (v[r] & 1);
        if (r == comm_->rank())
            idOffset_ = successive_ids ? run : 0;
        offs[r] = successive_ids ? run : 0;
        run += sizes_[r];
        maxTiles_ = std::max<int64_t>(maxTiles_, ceil_div(sizes_[r], (idx_t)256));
    }
    this->ntotal = run;
    this->is_trained = local_->is_trained;
    if (!dOffsets_)
        CUDA_VERIFY(cudaMalloc(&dOffsets_, sizeof(idx_t) * S));
    CUDA_VERIFY(cudaMemcpyAsync(dOffsets_, offs.data(), sizeof(idx_t) * S, cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

void DistributedIndexShards::train(idx_t n, const float* x) {
    local_->train(n, x);
    this->is_trained = local_->is_trained;
}

void DistributedIndexShards::add(idx_t n, const float* x) {
    FB_THROW_IF_NOT_MSG(
            !successive_ids || local_->ntotal == 0,
            "when adding to IndexShards with successive_ids, only add() in a single pass is supported");
    local_->add(n, x);
    syncWithSubIndexes();
}

void DistributedIndexShards::add_with_ids(idx_t n, const float* x, const idx_t* xids) {
    FB_THROW_IF_NOT_MSG(!(successive_ids && xids), "It makes no sense to pass in ids and request them to be shifted");
    local_->add_with_ids(n, x, xids);
    syncWithSubIndexes();
}

void DistributedIndexShards::reset() {
    local_->reset();
    syncWithSubIndexes();
}

void DistributedIndexShards::search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const {
    searchCollective(n, x, k, distances, labels, true);
}

void DistributedIndexShards::searchCollective(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, bool wantResult) const {
    FB_THROW_IF_NOT(k > 0);
    validateKSelect(k);
    if (n == 0)
        return;
    const int device = local_->getDevice();
    DeviceScope scope(device);
    GpuResources* res = resources_.get();
    cudaStream_t stream = res->getDefaultStream(device);
    const int S = comm_->size();
    // the pooled-threshold protocol only if EVERY rank takes the tensor-core Flat path for this (k, n):
    // decided from data every rank holds identically (gathered sizes and flags), never from local state
    bool pooled = allFlatTc_ && n >= 16;
    for (int r = 0; r < S && pooled; r++)
        pooled = flatTcSupported(d, (int)k, sizes_[r]);
    FlatTcShard ctx{comm_.get(), maxTiles_};
    // query pages bound the gathered staging ([S][page][k] x 12 bytes)
    const idx_t maxQ = std::max<idx_t>(1, std::min<idx_t>(idx_t(1) << 18, (idx_t)((size_t(768) << 20) / ((size_t)S * k * 12))));
    for (idx_t i0 = 0; i0 < n; i0 += maxQ) {
        const idx_t nb = std::min(maxQ, n - i0);
        DeviceView<float> xv(res, device, x + (size_t)i0 * d, (size_t)nb * d, stream);
        auto locD = res->temp(device, sizeof(float) * nb * k);
        auto locI = res->temp(device, sizeof(idx_t) * nb * k);
        SearchCall call;
        call.row0 = i0;
        local_->searchShardDevice(nb, xv.ptr, (int)k, locD.as<float>(), locI.as<idx_t>(), pooled ? &ctx : nullptr, call);
        auto allD = res->temp(device, sizeof(float) * (size_t)S * nb * k);
        auto allI = res->temp(device, sizeof(idx_t) * (size_t)S * nb * k);
        // ONE exchange: the per-shard [nb,k] distance and label blocks, fused into a single NCCL launch
        KernelTiming::begin("shards_exchange", stream);
        comm_->allGatherPair(locD.as<float>(), allD.as<float>(), (size_t)nb * k, locI.as<idx_t>(), allI.as<idx_t>(), (size_t)nb * k, stream);
        KernelTiming::end("shards_exchange", stream);
        if (wantResult) {
            DeviceOut<float> dv(res, device, distances + (size_t)i0 * k, (size_t)nb * k);
            DeviceOut<idx_t> lv(res, device, labels + (size_t)i0 * k, (size_t)nb * k);
            KernelTiming::begin("shards_merge", stream);
            runMergeTopKListMajor(allD.as<float>(), allI.as<idx_t>(), nb, S, (int)k, dOffsets_, (int)k, metric_type, dv.ptr, lv.ptr, stream);
            KernelTiming::end("shards_merge", stream);
            dv.finish(stream);
            lv.finish(stream);
            if (dv.staged || lv.staged || xv.hold.data)
                CUDA_VERIFY(cudaStreamSynchronize(stream));
        } else {
            CUDA_VERIFY(cudaStreamSynchronize(stream)); // staging buffers die here
        }
    }
}

// ------------------------------------------------------------------------------------------
// IndexShards: in-process NCCL fast path
// ------------------------------------------------------------------------------------------
bool IndexShards::ncclFastPath_(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const {
    const int S = count();
    if (S < 2 || k > kMaxK)
        return false;
    std::vector<GpuIndex*> gs(S);
    std::vector<int> seen;
    for (int i = 0; i < S; i++) {
        gs[i] = dynamic_cast<GpuIndex*>(shards_[i]);
        if (!gs[i])
            return false;
        const int dev = gs[i]->getDevice();
        if (std::find(seen.begin(), seen.end(), dev) != seen.end())
            return false; // two shards on one device: the clique has one rank per device
        seen.push_back(dev);
        auto c = gs[i]->getResources()->getCommunicator(dev);
        if (!c || c->size() != S || c->rank() != i)
            return false; // shard order must be rank order (the id translation follows it)
    }
    // (re)build the per-device wrappers when the shard set or the sizes changed; construction and
    // syncWithSubIndexes are collectives, so they run on one thread per device like the search
    bool stale = (int)dist_.size() != S;
    for (int i = 0; i < S && !stale; i++)
        stale = dist_[i]->local() != gs[i] || dist_[i]->successive_ids != successive_ids || dist_[i]->shardSize(i) != gs[i]->ntotal;
    std::vector<std::string> errors(S);
    auto runAll = [&](auto body) {
        std::vector<std::thread> th;
        for (int i = 0; i < S; i++)
            th.emplace_back([&, i] {
                try {
                    body(i);
                } catch (const std::exception& e) {
                    errors[i] = e.what();
                }
            });
        for (auto& t : th)
            t.join();
        for (int i = 0; i < S; i++)
            if (!errors[i].empty())
                FB_THROW_FMT("Exception thrown from index %d: %s", i, errors[i].c_str());
    };
    if (stale) {
        dist_.clear();
        dist_.resize(S);
        runAll([&](int i) { dist_[i].reset(new DistributedIndexShards(gs[i]->getResources(), gs[i], successive_ids)); });
    }
    runAll([&](int i) { dist_[i]->searchCollective(n, x, k, distances, labels, i == 0); });
    return true;
}

} // namespace fb200
