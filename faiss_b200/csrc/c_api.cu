// faiss_b200 -- the C ABI (include/faiss_b200_c.h).  Exceptions -> status codes + thread-local
// message, exactly as the reference does (c_api/macros_impl.h:22-36, c_api/error_impl.cpp:15).
#include <cstring>
#include <sstream>

#include "comm.h"
#include "distance.h"
#include "faiss_b200_c.h"
#include "icm_encode.h"
#include "index.h"
#include "rq_encode.h"

using namespace fb200;

static thread_local std::string g_last_error;

#define CATCH_AND_HANDLE                              \
    catch (const fb200::FaissException& e) {          \
        g_last_error = e.what();                      \
        return -2;                                    \
    }                                                 \
    catch (const std::exception& e) {                 \
        g_last_error = e.what();                      \
        return -4;                                    \
    }                                                 \
    catch (...) {                                     \
        g_last_error = "unknown exception";           \
        return -1;                                    \
    }                                                 \
    return 0;

struct FaissStandardGpuResources_H {
    std::shared_ptr<StandardGpuResources> res;
};
struct FaissIndex_H {
    Index* index;
    // keeps the resources alive as long as an index uses them
    std::shared_ptr<StandardGpuResources> res;
};

static Index* IX(const FaissIndex* p) {
    if (!p || !p->index)
        FB_THROW_MSG("null index handle");
    return p->index;
}
template <typename T>
static T* AS(const FaissIndex* p, const char* what) {
    T* t = dynamic_cast<T*>(IX(p));
    if (!t)
        FB_THROW_FMT("index handle is not a %s", what);
    return t;
}
static std::shared_ptr<StandardGpuResources> RES(FaissStandardGpuResources* r) {
    if (!r || !r->res)
        FB_THROW_MSG("null resources handle");
    return r->res;
}
// every value of faiss/MetricType.h; the C++ constructors reject what they do not implement (METRIC_NaNEuclidean
// anywhere, everything but L2 / IP in the IVF indexes)
static MetricType MT(FaissMetricType m) {
    const MetricType mt = (MetricType)(int)m;
    if (!is_implemented_metric(mt) && mt != fb200::METRIC_NaNEuclidean)
        FB_THROW_MSG("unsupported metric type");
    return mt;
}
// the entry points whose kernels are L2 / inner product only: the IVF constructors, k-means and the IVF seams
// (faiss/gpu/GpuIndexIVF.cu:34-38)
static MetricType MT_L2IP(FaissMetricType m) {
    if (m != ::METRIC_L2 && m != ::METRIC_INNER_PRODUCT)
        FB_THROW_FMT("unsupported metric type %d", (int)m);
    return m == ::METRIC_L2 ? fb200::METRIC_L2 : fb200::METRIC_INNER_PRODUCT;
}

extern "C" {

const char* faiss_get_last_error(void) {
    return g_last_error.c_str();
}
const char* faiss_b200_version(void) {
    return "faiss_b200 0.1 (sm_90a)";
}

// ---------------------------------------------------------------- resources
int faiss_StandardGpuResources_new(FaissStandardGpuResources** p) {
    try {
        auto* h = new FaissStandardGpuResources_H();
        h->res = std::make_shared<StandardGpuResources>();
        *p = h;
    }
    CATCH_AND_HANDLE
}
void faiss_StandardGpuResources_free(FaissStandardGpuResources* r) {
    delete r;
}
int faiss_StandardGpuResources_noTempMemory(FaissStandardGpuResources* r) {
    try {
        RES(r)->noTempMemory();
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_setTempMemory(FaissStandardGpuResources* r, size_t size) {
    try {
        RES(r)->setTempMemory(size);
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_setPinnedMemory(FaissStandardGpuResources* r, size_t size) {
    try {
        RES(r)->setPinnedMemory(size);
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_setDefaultStream(FaissStandardGpuResources* r, int device, void* stream) {
    try {
        RES(r)->setDefaultStream(device, (cudaStream_t)stream);
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_setDefaultNullStreamAllDevices(FaissStandardGpuResources* r) {
    try {
        RES(r)->setDefaultNullStreamAllDevices();
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_getDefaultStream(FaissStandardGpuResources* r, int device, void** out) {
    try {
        *out = (void*)RES(r)->getDefaultStream(device);
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_syncDefaultStream(FaissStandardGpuResources* r, int device) {
    try {
        DeviceScope s(device);
        RES(r)->syncDefaultStream(device);
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_getMemoryInfo(FaissStandardGpuResources* r, char* buf, size_t buflen) {
    try {
        auto info = RES(r)->getMemoryInfo();
        std::ostringstream os;
        os << "{";
        bool firstD = true;
        for (auto& dv : info) {
            if (!firstD)
                os << ",";
            firstD = false;
            os << "\"" << dv.first << "\":{";
            bool first = true;
            for (auto& kv : dv.second) {
                if (!first)
                    os << ",";
                first = false;
                os << "\"" << kv.first << "\":[" << kv.second.first << "," << kv.second.second << "]";
            }
            os << "}";
        }
        os << "}";
        std::string s = os.str();
        FB_THROW_IF_NOT_MSG(s.size() + 1 <= buflen, "buffer too small");
        memcpy(buf, s.c_str(), s.size() + 1);
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_getTempMemoryAvailable(FaissStandardGpuResources* r, int device, size_t* out) {
    try {
        RES(r)->initializeForDevice(device);
        *out = RES(r)->getTempMemoryAvailable(device);
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- generic index
void faiss_Index_free(FaissIndex* p) {
    if (p) {
        delete p->index;
        delete p;
    }
}
int faiss_Index_d(const FaissIndex* p) {
    return p && p->index ? p->index->d : 0;
}
int faiss_Index_is_trained(const FaissIndex* p) {
    return p && p->index ? (int)p->index->is_trained : 0;
}
idx_t faiss_Index_ntotal(const FaissIndex* p) {
    return p && p->index ? p->index->ntotal : 0;
}
FaissMetricType faiss_Index_metric_type(const FaissIndex* p) {
    return p && p->index ? (FaissMetricType)(int)p->index->metric_type : ::METRIC_L2;
}
float faiss_Index_metric_arg(const FaissIndex* p) {
    return p && p->index ? p->index->metric_arg : 0.f;
}
void faiss_Index_set_metric_arg(FaissIndex* p, float v) {
    if (p && p->index)
        p->index->metric_arg = v;
}
int faiss_Index_verbose(const FaissIndex* p) {
    return p && p->index ? (int)p->index->verbose : 0;
}
void faiss_Index_set_verbose(FaissIndex* p, int v) {
    if (p && p->index)
        p->index->verbose = v != 0;
}
int faiss_Index_train(FaissIndex* p, idx_t n, const float* x) {
    try {
        IX(p)->train(n, x);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_add(FaissIndex* p, idx_t n, const float* x) {
    try {
        IX(p)->add(n, x);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_add_with_ids(FaissIndex* p, idx_t n, const float* x, const idx_t* xids) {
    try {
        IX(p)->add_with_ids(n, x, xids);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_search(const FaissIndex* p, idx_t n, const float* x, idx_t k, float* D, idx_t* I) {
    try {
        IX(p)->search(n, x, k, D, I);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_assign(FaissIndex* p, idx_t n, const float* x, idx_t* labels, idx_t k) {
    try {
        IX(p)->assign(n, x, labels, k);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_reset(FaissIndex* p) {
    try {
        IX(p)->reset();
    }
    CATCH_AND_HANDLE
}
int faiss_Index_reconstruct(const FaissIndex* p, idx_t key, float* out) {
    try {
        IX(p)->reconstruct(key, out);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_reconstruct_n(const FaissIndex* p, idx_t i0, idx_t ni, float* out) {
    try {
        IX(p)->reconstruct_n(i0, ni, out);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_reconstruct_batch(const FaissIndex* p, idx_t n, const idx_t* keys, float* out) {
    try {
        IX(p)->reconstruct_batch(n, keys, out);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_compute_residual(const FaissIndex* p, const float* x, float* r, idx_t key) {
    try {
        IX(p)->compute_residual(x, r, key);
    }
    CATCH_AND_HANDLE
}
int faiss_Index_compute_residual_n(const FaissIndex* p, idx_t n, const float* x, float* r, const idx_t* keys) {
    try {
        IX(p)->compute_residual_n(n, x, r, keys);
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- GpuIndexFlat
int faiss_GpuIndexFlat_new(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        int d,
        FaissMetricType metric,
        int device,
        int use_tc) {
    try {
        GpuIndexFlatConfig c;
        c.device = device;
        c.useTensorCores = use_tc != 0;
        auto res = RES(r);
        auto* h = new FaissIndex_H();
        h->res = res;
        h->index = new GpuIndexFlat(res, d, MT(metric), c);
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexFlat_new_with_config(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        int d,
        FaissMetricType metric,
        int device,
        int use_tc,
        int use_float16) {
    try {
        GpuIndexFlatConfig c;
        c.device = device;
        c.useTensorCores = use_tc != 0;
        c.useFloat16 = use_float16 != 0;
        auto res = RES(r);
        auto* h = new FaissIndex_H();
        h->res = res;
        h->index = new GpuIndexFlat(res, d, MT(metric), c);
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexFlatL2_new(FaissGpuIndex** p, FaissStandardGpuResources* r, int d, int device) {
    return faiss_GpuIndexFlat_new(p, r, d, ::METRIC_L2, device, 1);
}
int faiss_GpuIndexFlatIP_new(FaissGpuIndex** p, FaissStandardGpuResources* r, int d, int device) {
    return faiss_GpuIndexFlat_new(p, r, d, ::METRIC_INNER_PRODUCT, device, 1);
}
int faiss_GpuIndexFlat_copyFrom(FaissGpuIndex* p, idx_t n, const float* xb) {
    try {
        AS<GpuIndexFlat>(p, "GpuIndexFlat")->copyFrom(n, xb);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexFlat_copyTo(const FaissGpuIndex* p, float* out) {
    try {
        AS<GpuIndexFlat>(p, "GpuIndexFlat")->copyTo(out);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndex_setMinPagingSize(FaissGpuIndex* p, size_t size) { // faiss/gpu/GpuIndex.h:66-69
    try {
        AS<GpuIndex>(p, "GpuIndex")->setMinPagingSize(size);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndex_getMinPagingSize(const FaissGpuIndex* p, size_t* out) {
    try {
        *out = AS<GpuIndex>(p, "GpuIndex")->getMinPagingSize();
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexFlat_setUseTensorCores(FaissGpuIndex* p, int enable) {
    try {
        AS<GpuIndexFlat>(p, "GpuIndexFlat")->setUseTensorCores(enable != 0);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexFlat_lastSearchInfo(const FaissGpuIndex* p, int* out2) {
    try {
        auto* f = AS<GpuIndexFlat>(p, "GpuIndexFlat");
        out2[0] = f->lastSearchUsedTensorCores;
        out2[1] = f->lastSearchFallbackQueries;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexFlat_lastSearchOperandBits(const FaissGpuIndex* p, int* bits) {
    try {
        *bits = AS<GpuIndexFlat>(p, "GpuIndexFlat")->lastSearchOperandBits;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexFlat_lastSearchRepairedQueries(const FaissGpuIndex* p, int* count) {
    try {
        *count = AS<GpuIndexFlat>(p, "GpuIndexFlat")->lastSearchRepairedQueries;
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- GpuIndexIVF
int faiss_GpuIndexIVF_set_nprobe(FaissGpuIndex* p, size_t nprobe) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->nprobe = nprobe;
    }
    CATCH_AND_HANDLE
}
size_t faiss_GpuIndexIVF_nprobe(const FaissGpuIndex* p) {
    auto* i = p ? dynamic_cast<GpuIndexIVF*>(p->index) : nullptr;
    return i ? i->nprobe : 0;
}
size_t faiss_GpuIndexIVF_nlist(const FaissGpuIndex* p) {
    auto* i = p ? dynamic_cast<GpuIndexIVF*>(p->index) : nullptr;
    return i ? (size_t)i->nlist : 0;
}
int faiss_GpuIndexIVF_set_clustering(FaissGpuIndex* p, int niter, int seed, int maxppc) {
    try {
        auto* i = AS<GpuIndexIVF>(p, "GpuIndexIVF");
        if (niter > 0)
            i->cp.niter = niter;
        if (seed >= 0)
            i->cp.seed = seed;
        if (maxppc > 0)
            i->cp.max_points_per_centroid = maxppc;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_reserveMemory(FaissGpuIndex* p, size_t n) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->reserveMemory(n);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_reclaimMemory(FaissGpuIndex* p, size_t* out) {
    try {
        size_t r = AS<GpuIndexIVF>(p, "GpuIndexIVF")->reclaimMemory();
        if (out)
            *out = r;
    }
    CATCH_AND_HANDLE
}
size_t faiss_GpuIndexIVF_get_list_size(const FaissGpuIndex* p, size_t l) {
    auto* i = p ? dynamic_cast<GpuIndexIVF*>(p->index) : nullptr;
    if (!i || (idx_t)l >= i->nlist)
        return 0;
    return (size_t)i->getListLength((idx_t)l);
}
int faiss_GpuIndexIVF_getListVectorData(const FaissGpuIndex* p, size_t l, uint8_t* out) {
    try {
        auto v = AS<GpuIndexIVF>(p, "GpuIndexIVF")->getListVectorData((idx_t)l);
        if (!v.empty())
            memcpy(out, v.data(), v.size());
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_getListIndices(const FaissGpuIndex* p, size_t l, idx_t* out) {
    try {
        auto v = AS<GpuIndexIVF>(p, "GpuIndexIVF")->getListIndices((idx_t)l);
        if (!v.empty())
            memcpy(out, v.data(), v.size() * sizeof(idx_t));
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_setCoarseCentroids(FaissGpuIndex* p, const float* c) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->setCoarseCentroids(c);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_getCoarseCentroids(const FaissGpuIndex* p, float* out) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->getCoarseCentroids(out);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_setList(FaissGpuIndex* p, size_t l, idx_t len, const uint8_t* codes, const idx_t* ids) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->setList((idx_t)l, len, codes, ids);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_setListSizes(FaissGpuIndex* p, const idx_t* lens) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->setListSizes(lens);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_set_is_trained(FaissGpuIndex* p, int v) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->is_trained = v != 0;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_search_preassigned(
        const FaissGpuIndex* p,
        idx_t n,
        const float* x,
        idx_t k,
        const idx_t* assign,
        const float* cdis,
        float* D,
        idx_t* I) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")->search_preassigned(n, x, k, assign, cdis, D, I);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFFlat_new(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        int d,
        idx_t nlist,
        FaissMetricType metric,
        int device) {
    try {
        GpuIndexIVFConfig c;
        c.device = device;
        auto res = RES(r);
        auto* h = new FaissIndex_H();
        h->res = res;
        h->index = new GpuIndexIVFFlat(res, d, nlist, MT_L2IP(metric), c);
        *p = h;
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- GpuIndexIVFPQ
int faiss_GpuIndexIVFPQ_new(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        int d,
        idx_t nlist,
        idx_t M,
        idx_t nbits,
        FaissMetricType metric,
        int device) {
    try {
        GpuIndexIVFPQConfig c;
        c.device = device;
        auto res = RES(r);
        auto* h = new FaissIndex_H();
        h->res = res;
        h->index = new GpuIndexIVFPQ(res, d, nlist, M, nbits, MT_L2IP(metric), c);
        *p = h;
    }
    CATCH_AND_HANDLE
}
// GpuIndexIVFPQConfig::interleavedLayout (faiss/gpu/GpuIndexIVFPQ.h:36-40): with it nbits may be 4, 5, 6 or 8
int faiss_GpuIndexIVFPQ_new_with_config(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        FaissGpuIndex* coarse,
        int d,
        idx_t nlist,
        idx_t M,
        idx_t nbits,
        FaissMetricType metric,
        int device,
        int interleaved_layout) {
    try {
        auto res = RES(r);
        GpuIndexIVFPQConfig cfg;
        cfg.device = device;
        cfg.interleavedLayout = interleaved_layout != 0;
        auto* h = new FaissIndex_H{nullptr, res};
        try {
            h->index = coarse ? new GpuIndexIVFPQ(res, AS<GpuIndexFlat>(coarse, "GpuIndexFlat"), d, nlist, M, nbits, MT_L2IP(metric), cfg)
                              : new GpuIndexIVFPQ(res, d, nlist, M, nbits, MT_L2IP(metric), cfg);
        } catch (...) {
            delete h;
            throw;
        }
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFPQ_setPQCentroids(FaissGpuIndex* p, const float* c) {
    try {
        AS<GpuIndexIVFPQ>(p, "GpuIndexIVFPQ")->setPQCentroids(c);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFPQ_getPQCentroids(const FaissGpuIndex* p, float* out) {
    try {
        AS<GpuIndexIVFPQ>(p, "GpuIndexIVFPQ")->getPQCentroids(out);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFPQ_set_pq_clustering(FaissGpuIndex* p, int niter, int seed, int maxppc) {
    try {
        auto* i = AS<GpuIndexIVFPQ>(p, "GpuIndexIVFPQ");
        if (niter > 0)
            i->pq_cp.niter = niter;
        if (seed >= 0)
            i->pq_cp.seed = seed;
        if (maxppc > 0)
            i->pq_cp.max_points_per_centroid = maxppc;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFPQ_setPrecomputedCodes(FaissGpuIndex* p, int enable) {
    try {
        AS<GpuIndexIVFPQ>(p, "GpuIndexIVFPQ")->setPrecomputedCodes(enable != 0);
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- GpuIndexIVFScalarQuantizer
int faiss_GpuIndexIVFScalarQuantizer_new(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        int d,
        idx_t nlist,
        int qtype,
        FaissMetricType metric,
        int encodeResidual,
        int device) {
    try {
        GpuIndexIVFScalarQuantizerConfig c;
        c.device = device;
        auto res = RES(r);
        auto* h = new FaissIndex_H{nullptr, res};
        try {
            h->index = new GpuIndexIVFScalarQuantizer(res, d, nlist, qtype, MT_L2IP(metric), encodeResidual != 0, c);
        } catch (...) {
            delete h;
            throw;
        }
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFScalarQuantizer_new_with_quantizer(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        FaissGpuIndex* coarse,
        int d,
        idx_t nlist,
        int qtype,
        FaissMetricType metric,
        int encodeResidual,
        int device) {
    try {
        GpuIndexIVFScalarQuantizerConfig c;
        c.device = device;
        auto res = RES(r);
        auto* h = new FaissIndex_H{nullptr, res};
        try {
            h->index = new GpuIndexIVFScalarQuantizer(
                    res, AS<GpuIndexFlat>(coarse, "GpuIndexFlat"), d, nlist, qtype, MT_L2IP(metric), encodeResidual != 0, c);
        } catch (...) {
            delete h;
            throw;
        }
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFScalarQuantizer_set_trained(FaissGpuIndex* p, const float* t, size_t n) {
    try {
        AS<GpuIndexIVFScalarQuantizer>(p, "GpuIndexIVFScalarQuantizer")->setTrained(t, n);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFScalarQuantizer_get_trained(const FaissGpuIndex* p, float* out, size_t* n) {
    try {
        FB_THROW_IF_NOT_MSG(n != nullptr, "null length pointer");
        const auto& t = AS<GpuIndexIVFScalarQuantizer>(p, "GpuIndexIVFScalarQuantizer")->getTrained();
        if (out)
            std::copy(t.begin(), t.end(), out);
        *n = t.size();
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFScalarQuantizer_code_size(const FaissGpuIndex* p, size_t* out) {
    try {
        auto* i = AS<GpuIndexIVFScalarQuantizer>(p, "GpuIndexIVFScalarQuantizer");
        *out = (size_t)GpuIndexIVFScalarQuantizer::codeSizeFor(i->qtype(), i->d);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFScalarQuantizer_qtype(const FaissGpuIndex* p, int* out) {
    try {
        *out = AS<GpuIndexIVFScalarQuantizer>(p, "GpuIndexIVFScalarQuantizer")->qtype();
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFScalarQuantizer_by_residual(const FaissGpuIndex* p, int* out) {
    try {
        *out = AS<GpuIndexIVFScalarQuantizer>(p, "GpuIndexIVFScalarQuantizer")->by_residual ? 1 : 0;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFScalarQuantizer_set_rangestat(FaissGpuIndex* p, int rangestat, float arg) {
    try {
        auto* i = AS<GpuIndexIVFScalarQuantizer>(p, "GpuIndexIVFScalarQuantizer");
        FB_THROW_IF_NOT_MSG(rangestat >= 0 && rangestat <= 3, "invalid rangestat");
        i->rangestat = rangestat;
        i->rangestat_arg = arg;
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- IndexShards
int faiss_IndexShards_new(FaissIndexShards** p, idx_t d) {
    return faiss_IndexShards_new_with_options(p, d, 0, 1);
}
int faiss_IndexShards_new_with_options(FaissIndexShards** p, idx_t d, int threaded, int successive_ids) {
    try {
        auto* h = new FaissIndex_H();
        h->index = new IndexShards((int)d, threaded != 0, successive_ids != 0);
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_IndexShards_add_shard(FaissIndexShards* p, FaissIndex* shard) {
    try {
        AS<IndexShards>(p, "IndexShards")->add_shard(IX(shard));
    }
    CATCH_AND_HANDLE
}
int faiss_IndexShards_remove_shard(FaissIndexShards* p, FaissIndex* shard) {
    try {
        AS<IndexShards>(p, "IndexShards")->remove_shard(IX(shard));
    }
    CATCH_AND_HANDLE
}
FaissIndex* faiss_IndexShards_at(FaissIndexShards*, int) {
    // handles are owned by the caller; the C++ object can be reached through the shard handles
    return nullptr;
}
int faiss_IndexShards_own_indices(const FaissIndexShards* p) {
    auto* s = p ? dynamic_cast<IndexShards*>(p->index) : nullptr;
    return s ? (int)s->own_indices : 0;
}
void faiss_IndexShards_set_own_indices(FaissIndexShards* p, int v) {
    // ownership of sub-indexes stays with their C handles; refuse to double-free
    (void)p;
    (void)v;
}
int faiss_IndexShards_successive_ids(const FaissIndexShards* p) {
    auto* s = p ? dynamic_cast<IndexShards*>(p->index) : nullptr;
    return s ? (int)s->successive_ids : 0;
}
void faiss_IndexShards_set_successive_ids(FaissIndexShards* p, int v) {
    auto* s = p ? dynamic_cast<IndexShards*>(p->index) : nullptr;
    if (s)
        s->successive_ids = v != 0;
}

// ---------------------------------------------------------------- search parameters, interrupt, shared quantiser
struct FaissSearchParameters_H {
    SearchParameters* p;
};
int faiss_SearchParametersIVF_new_with(FaissSearchParametersIVF** out, size_t nprobe, size_t max_codes) {
    return faiss_SearchParametersIVF_new_with_sel(out, nullptr, nprobe, max_codes);
}

// ---------------------------------------------------------------- IDSelector
} // extern "C"
struct FaissIDSelector_H {
    IDSelector* sel;
};
static const IDSelector* SEL(const FaissIDSelector* p) {
    if (!p || !p->sel)
        FB_THROW_MSG("null IDSelector handle");
    return p->sel;
}
template <typename F>
static int newSelector(FaissIDSelector** out, F make) {
    try {
        FB_THROW_IF_NOT_MSG(out != nullptr, "null output pointer");
        std::unique_ptr<IDSelector> s(make());
        *out = new FaissIDSelector_H{s.release()};
    }
    CATCH_AND_HANDLE
}
extern "C" {
void faiss_IDSelector_free(FaissIDSelector* p) {
    if (p) {
        delete p->sel;
        delete p;
    }
}
int faiss_IDSelector_is_member(const FaissIDSelector* p, idx_t id) {
    if (!p || !p->sel)
        return -1;
    return p->sel->is_member(id) ? 1 : 0;
}
int faiss_IDSelectorRange_new(FaissIDSelectorRange** out, idx_t imin, idx_t imax) {
    return newSelector(out, [&] { return IDSelector::range(imin, imax); });
}
int faiss_IDSelectorArray_new(FaissIDSelectorArray** out, size_t n, const idx_t* ids) {
    return newSelector(out, [&] { return IDSelector::array(n, ids); });
}
int faiss_IDSelectorBatch_new(FaissIDSelectorBatch** out, size_t n, const idx_t* indices) {
    return newSelector(out, [&] { return IDSelector::batch(n, indices); });
}
int faiss_IDSelectorBitmap_new(FaissIDSelectorBitmap** out, size_t n, const uint8_t* bitmap) {
    return newSelector(out, [&] { return IDSelector::bitmapOf(n, bitmap); });
}
int faiss_IDSelectorNot_new(FaissIDSelectorNot** out, const FaissIDSelector* sel) {
    return newSelector(out, [&] { return IDSelector::negation(SEL(sel)); });
}
int faiss_IDSelectorAnd_new(FaissIDSelectorAnd** out, const FaissIDSelector* lhs, const FaissIDSelector* rhs) {
    return newSelector(out, [&] { return IDSelector::binary(IDSelector::AND, SEL(lhs), SEL(rhs)); });
}
int faiss_IDSelectorOr_new(FaissIDSelectorOr** out, const FaissIDSelector* lhs, const FaissIDSelector* rhs) {
    return newSelector(out, [&] { return IDSelector::binary(IDSelector::OR, SEL(lhs), SEL(rhs)); });
}
int faiss_IDSelectorXOr_new(FaissIDSelectorXOr** out, const FaissIDSelector* lhs, const FaissIDSelector* rhs) {
    return newSelector(out, [&] { return IDSelector::binary(IDSelector::XOR, SEL(lhs), SEL(rhs)); });
}
int faiss_b200_IDSelectorCallback_new(FaissIDSelector** out, int (*is_member)(void* ctx, idx_t id), void* ctx) {
    return newSelector(out, [&] { return IDSelector::callback(is_member, ctx); });
}
int faiss_SearchParameters_new(FaissSearchParameters** out, FaissIDSelector* sel) {
    try {
        FB_THROW_IF_NOT_MSG(out != nullptr, "null output pointer");
        auto sp = std::make_unique<SearchParameters>();
        sp->sel = sel ? SEL(sel) : nullptr;
        *out = new FaissSearchParameters_H{sp.release()};
    }
    CATCH_AND_HANDLE
}
int faiss_SearchParametersIVF_new_with_sel(FaissSearchParametersIVF** out, FaissIDSelector* sel, size_t nprobe, size_t max_codes) {
    try {
        FB_THROW_IF_NOT_MSG(out != nullptr, "null output pointer");
        auto sp = std::make_unique<SearchParametersIVF>();
        sp->sel = sel ? SEL(sel) : nullptr;
        sp->nprobe = nprobe;
        sp->max_codes = max_codes;
        *out = new FaissSearchParameters_H{sp.release()};
    }
    CATCH_AND_HANDLE
}
// ---------------------------------------------------------------- GpuIndexCagra
void faiss_GpuIndexCagraConfig_init(FaissGpuIndexCagraConfig* c) {
    const GpuIndexCagraConfig d;
    c->device = d.device;
    c->intermediate_graph_degree = d.intermediate_graph_degree;
    c->graph_degree = d.graph_degree;
    c->build_algo = (int)d.build_algo;
    c->nn_descent_niter = d.nn_descent_niter;
    c->refine_rate = d.refine_rate;
    c->store_dataset = d.store_dataset;
    c->guarantee_connectivity = d.guarantee_connectivity;
    c->n_lists = d.ivf_pq_params.n_lists;
    c->kmeans_n_iters = d.ivf_pq_params.kmeans_n_iters;
    c->kmeans_trainset_fraction = d.ivf_pq_params.kmeans_trainset_fraction;
    c->pq_bits = d.ivf_pq_params.pq_bits;
    c->pq_dim = d.ivf_pq_params.pq_dim;
    c->codebook_kind = (int)d.ivf_pq_params.codebook_kind;
    c->force_random_rotation = d.ivf_pq_params.force_random_rotation;
    c->conservative_memory_allocation = d.ivf_pq_params.conservative_memory_allocation;
    c->n_probes = d.ivf_pq_search_params.n_probes;
    c->max_internal_batch_size = d.ivf_pq_search_params.max_internal_batch_size;
}
int faiss_GpuIndexCagra_new(FaissGpuIndex** p, FaissStandardGpuResources* r, int d, FaissMetricType metric, const FaissGpuIndexCagraConfig* cc) {
    try {
        FB_THROW_IF_NOT_MSG(p != nullptr && cc != nullptr, "null argument");
        auto res = RES(r);
        GpuIndexCagraConfig c;
        c.device = cc->device;
        c.intermediate_graph_degree = cc->intermediate_graph_degree;
        c.graph_degree = cc->graph_degree;
        c.build_algo = (graph_build_algo)cc->build_algo;
        c.nn_descent_niter = cc->nn_descent_niter;
        c.refine_rate = cc->refine_rate;
        c.store_dataset = cc->store_dataset != 0;
        c.guarantee_connectivity = cc->guarantee_connectivity != 0;
        c.ivf_pq_params.n_lists = cc->n_lists;
        c.ivf_pq_params.kmeans_n_iters = cc->kmeans_n_iters;
        c.ivf_pq_params.kmeans_trainset_fraction = cc->kmeans_trainset_fraction;
        c.ivf_pq_params.pq_bits = cc->pq_bits;
        c.ivf_pq_params.pq_dim = cc->pq_dim;
        c.ivf_pq_params.codebook_kind = (codebook_gen)cc->codebook_kind;
        c.ivf_pq_params.force_random_rotation = cc->force_random_rotation != 0;
        c.ivf_pq_params.conservative_memory_allocation = cc->conservative_memory_allocation != 0;
        c.ivf_pq_search_params.n_probes = cc->n_probes;
        c.ivf_pq_search_params.max_internal_batch_size = cc->max_internal_batch_size;
        std::unique_ptr<Index> ix(new GpuIndexCagra(res, d, MT_L2IP(metric), c));
        *p = new FaissIndex_H{ix.release(), res};
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexCagra_graph_degree(const FaissGpuIndex* p, int* degree) {
    try {
        *degree = AS<GpuIndexCagra>(p, "GpuIndexCagra")->graphDegree();
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexCagra_get_knngraph(const FaissGpuIndex* p, idx_t* graph) {
    try {
        auto g = AS<GpuIndexCagra>(p, "GpuIndexCagra")->get_knngraph();
        std::memcpy(graph, g.data(), g.size() * sizeof(idx_t));
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexCagra_copyFrom(FaissGpuIndex* p, idx_t n, const float* xb, const idx_t* graph, int degree) {
    try {
        AS<GpuIndexCagra>(p, "GpuIndexCagra")->copyFrom(n, xb, graph, degree);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexCagra_copyTo(const FaissGpuIndex* p, float* xb, idx_t* graph) {
    try {
        AS<GpuIndexCagra>(p, "GpuIndexCagra")->copyTo(xb, graph);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexCagra_lastSearchDistanceCount(const FaissGpuIndex* p, int64_t* count) {
    try {
        *count = AS<GpuIndexCagra>(p, "GpuIndexCagra")->lastSearchDistanceCount;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexCagra_lastBuildSeconds(const FaissGpuIndex* p, double* seconds3) {
    try {
        const auto* ix = AS<GpuIndexCagra>(p, "GpuIndexCagra");
        for (int i = 0; i < 3; i++)
            seconds3[i] = ix->lastBuildSeconds[i];
    }
    CATCH_AND_HANDLE
}
void faiss_SearchParametersCagraConfig_init(FaissSearchParametersCagraConfig* c) {
    const SearchParametersCagra d;
    c->max_queries = d.max_queries;
    c->itopk_size = d.itopk_size;
    c->max_iterations = d.max_iterations;
    c->algo = (int)d.algo;
    c->team_size = d.team_size;
    c->search_width = d.search_width;
    c->min_iterations = d.min_iterations;
    c->thread_block_size = d.thread_block_size;
    c->hashmap_mode = (int)d.hashmap_mode;
    c->hashmap_min_bitlen = d.hashmap_min_bitlen;
    c->hashmap_max_fill_rate = d.hashmap_max_fill_rate;
    c->num_random_samplings = d.num_random_samplings;
    c->seed = d.seed;
}
int faiss_SearchParametersCagra_new(FaissSearchParametersCagra** out, FaissIDSelector* sel, const FaissSearchParametersCagraConfig* c) {
    try {
        FB_THROW_IF_NOT_MSG(out != nullptr && c != nullptr, "null argument");
        auto sp = std::make_unique<SearchParametersCagra>();
        sp->sel = sel ? SEL(sel) : nullptr;
        sp->max_queries = c->max_queries;
        sp->itopk_size = c->itopk_size;
        sp->max_iterations = c->max_iterations;
        sp->algo = (search_algo)c->algo;
        sp->team_size = c->team_size;
        sp->search_width = c->search_width;
        sp->min_iterations = c->min_iterations;
        sp->thread_block_size = c->thread_block_size;
        sp->hashmap_mode = (hash_mode)c->hashmap_mode;
        sp->hashmap_min_bitlen = c->hashmap_min_bitlen;
        sp->hashmap_max_fill_rate = c->hashmap_max_fill_rate;
        sp->num_random_samplings = c->num_random_samplings;
        sp->seed = c->seed;
        *out = new FaissSearchParameters_H{sp.release()};
    }
    CATCH_AND_HANDLE
}
int b200_cagra_optimize(FaissStandardGpuResources* r, int device, const uint32_t* G0, int64_t n, int K0, int K, uint32_t* G) {
    try {
        auto res = RES(r);
        DeviceScope scope(device);
        res->initializeForDevice(device);
        auto stream = res->getDefaultStream(device);
        FB_THROW_IF_NOT_FMT(n >= 0 && K0 >= 1, "b200_cagra_optimize: bad shape (%ld, %d)", (long)n, K0);
        checkCagraG0(res.get(), device, G0, n, K0, stream);
        runCagraOptimize(res.get(), device, G0, n, K0, K, G, stream);
    }
    CATCH_AND_HANDLE
}

void faiss_SearchParameters_free(FaissSearchParameters* p) {
    if (p) {
        delete p->p;
        delete p;
    }
}
int faiss_Index_search_with_params(
        const FaissIndex* p, idx_t n, const float* x, idx_t k, const FaissSearchParameters* params, float* D, idx_t* I) {
    try {
        Index* ix = IX(p);
        if (!params || !params->p) {
            ix->search(n, x, k, D, I);
        } else if (auto* g = dynamic_cast<GpuIndex*>(ix)) {
            g->search(n, x, k, D, I, params->p);
        } else {
            FB_THROW_MSG("search parameters are only supported on GPU indexes");
        }
    }
    CATCH_AND_HANDLE
}
int faiss_Index_search_and_reconstruct(
        const FaissIndex* p, idx_t n, const float* x, idx_t k, const FaissSearchParameters* params, float* D, idx_t* I,
        float* recons) {
    try {
        IX(p)->search_and_reconstruct(n, x, k, D, I, recons, params ? params->p : nullptr);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_search_and_return_codes(
        const FaissGpuIndex* p, idx_t n, const float* x, idx_t k, const FaissSearchParameters* params, float* D, idx_t* I,
        uint8_t* codes, int include_listno) {
    try {
        AS<GpuIndexIVF>(p, "GpuIndexIVF")
                ->search_and_return_codes(n, x, k, D, I, codes, include_listno != 0, params ? params->p : nullptr);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVF_code_sizes(const FaissGpuIndex* p, int* coarse_code_size, int* code_size) {
    try {
        auto* ivf = AS<GpuIndexIVF>(p, "GpuIndexIVF");
        *coarse_code_size = ivf->coarse_code_size();
        *code_size = ivf->code_size();
    }
    CATCH_AND_HANDLE
}
void faiss_b200_set_interrupt_callback(int (*want_interrupt)(void*), void* ctx) {
    InterruptCallback::set(want_interrupt, ctx);
}
int faiss_GpuIndexIVFFlat_new_with_quantizer(
        FaissGpuIndex** p, FaissStandardGpuResources* r, FaissGpuIndex* coarse, int d, idx_t nlist, FaissMetricType metric, int device) {
    try {
        auto res = RES(r);
        GpuIndexIVFConfig cfg;
        cfg.device = device;
        auto* h = new FaissIndex_H{nullptr, res};
        try {
            h->index = new GpuIndexIVFFlat(res, AS<GpuIndexFlat>(coarse, "GpuIndexFlat"), d, nlist, MT_L2IP(metric), cfg);
        } catch (...) {
            delete h;
            throw;
        }
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIndexIVFPQ_new_with_quantizer(
        FaissGpuIndex** p,
        FaissStandardGpuResources* r,
        FaissGpuIndex* coarse,
        int d,
        idx_t nlist,
        idx_t M,
        idx_t nbits,
        FaissMetricType metric,
        int device) {
    try {
        auto res = RES(r);
        GpuIndexIVFPQConfig cfg;
        cfg.device = device;
        auto* h = new FaissIndex_H{nullptr, res};
        try {
            h->index = new GpuIndexIVFPQ(res, AS<GpuIndexFlat>(coarse, "GpuIndexFlat"), d, nlist, M, nbits, MT_L2IP(metric), cfg);
        } catch (...) {
            delete h;
            throw;
        }
        *p = h;
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- NCCL communicator ownership + sharded search
int faiss_b200_nccl_unique_id(char* out128) {
    try {
        FB_THROW_IF_NOT_MSG(out128 != nullptr, "null output buffer");
        auto id = Communicator::uniqueId();
        memcpy(out128, id.data(), id.size());
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_ncclInitRank(FaissStandardGpuResources* r, int device, int nranks, int rank, const char* id128) {
    try {
        FB_THROW_IF_NOT_MSG(id128 != nullptr, "null unique id");
        RES(r)->ncclInitRank(device, nranks, rank, id128);
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_ncclInitAll(FaissStandardGpuResources* r, int ndev, const int* devices) {
    try {
        FB_THROW_IF_NOT_MSG(ndev > 0 && devices != nullptr, "no devices");
        RES(r)->ncclInitAll(std::vector<int>(devices, devices + ndev));
    }
    CATCH_AND_HANDLE
}
int faiss_StandardGpuResources_ncclRank(FaissStandardGpuResources* r, int device, int* rank, int* nranks) {
    try {
        auto c = RES(r)->getCommunicator(device);
        FB_THROW_IF_NOT_MSG(c != nullptr, "no communicator for this device");
        if (rank)
            *rank = c->rank();
        if (nranks)
            *nranks = c->size();
    }
    CATCH_AND_HANDLE
}
int faiss_IndexShardsIVF_new(FaissIndexShards** p, FaissGpuIndex* quantizer, idx_t nlist, int threaded, int successive_ids) {
    try {
        auto* h = new FaissIndex_H();
        try {
            h->index = new IndexShardsIVF(AS<GpuIndexFlat>(quantizer, "GpuIndexFlat"), nlist, threaded != 0, successive_ids != 0);
        } catch (...) {
            delete h;
            throw;
        }
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_IndexShardsIVF_add_shard(FaissIndexShards* p, FaissIndex* shard) {
    try {
        AS<IndexShardsIVF>(p, "IndexShardsIVF")->add_shard(IX(shard));
    }
    CATCH_AND_HANDLE
}
int faiss_IndexShards_lastSearchPath(const FaissIndexShards* p) {
    try {
        return AS<IndexShards>(p, "IndexShards")->lastSearchPath;
    } catch (...) {
        return -1;
    }
}
int faiss_DistributedIndexShards_new(FaissIndexShards** p, FaissStandardGpuResources* r, FaissGpuIndex* local, int successive_ids) {
    try {
        auto res = RES(r);
        auto* h = new FaissIndex_H{nullptr, res};
        try {
            h->index = new DistributedIndexShards(res, AS<GpuIndex>(local, "GpuIndex"), successive_ids != 0);
        } catch (...) {
            delete h;
            throw;
        }
        *p = h;
    }
    CATCH_AND_HANDLE
}
int faiss_DistributedIndexShards_sync(FaissIndexShards* p) {
    try {
        AS<DistributedIndexShards>(p, "DistributedIndexShards")->syncWithSubIndexes();
    }
    CATCH_AND_HANDLE
}
int faiss_DistributedIndexShards_info(const FaissIndexShards* p, int* rank, int* nranks, idx_t* id_offset) {
    try {
        auto* s = AS<DistributedIndexShards>(p, "DistributedIndexShards");
        if (rank)
            *rank = s->rank();
        if (nranks)
            *nranks = s->worldSize();
        if (id_offset)
            *id_offset = s->idOffset();
    }
    CATCH_AND_HANDLE
}
int b200_shards_search(
        FaissStandardGpuResources* r,
        FaissGpuIndex* local_shard,
        int successive_ids,
        idx_t n,
        const float* x,
        idx_t k,
        float* distances,
        idx_t* labels) {
    try {
        // one-shot form (re-reads every shard's size first: one tiny extra collective); hold a
        // DistributedIndexShards for repeated searches
        DistributedIndexShards s(RES(r), AS<GpuIndex>(local_shard, "GpuIndex"), successive_ids != 0);
        s.search(n, x, k, distances, labels);
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- clustering
int faiss_b200_kmeans(
        FaissStandardGpuResources* r,
        int device,
        size_t d,
        size_t n,
        size_t k,
        const float* x,
        int niter,
        int seed,
        int maxppc,
        float* centroids_out,
        float* obj_out) {
    return faiss_b200_kmeans_ex(r, device, d, n, k, x, niter, seed, maxppc, ::METRIC_L2, 0, centroids_out, obj_out);
}

int faiss_b200_kmeans_ex(
        FaissStandardGpuResources* r,
        int device,
        size_t d,
        size_t n,
        size_t k,
        const float* x,
        int niter,
        int seed,
        int maxppc,
        FaissMetricType metric,
        int spherical,
        float* centroids_out,
        float* obj_out) {
    try {
        auto res = RES(r);
        ClusteringParameters cp;
        if (niter > 0)
            cp.niter = niter;
        if (seed >= 0)
            cp.seed = seed;
        if (maxppc > 0)
            cp.max_points_per_centroid = maxppc;
        cp.spherical = spherical != 0;
        Clustering clus((int)d, (int)k, cp);
        GpuIndexFlatConfig fc;
        fc.device = device;
        GpuIndexFlat index(res, (int)d, MT_L2IP(metric), fc);
        clus.train((idx_t)n, x, index);
        memcpy(centroids_out, clus.centroids.data(), sizeof(float) * d * k);
        if (obj_out) {
            for (size_t i = 0; i < clus.iteration_stats.size() && (int)i < cp.niter; i++)
                obj_out[i] = clus.iteration_stats[i].obj;
        }
    }
    CATCH_AND_HANDLE
}

int faiss_b200_kmeans_sharded(
        FaissStandardGpuResources* r,
        int device,
        size_t d,
        size_t n_local,
        size_t k,
        const float* x_local,
        int niter,
        int seed,
        float* centroids_out,
        float* obj_out,
        double* stats_out) {
    try {
        auto res = RES(r);
        res->initializeForDevice(device);
        auto comm = res->getCommunicator(device);
        FB_THROW_IF_NOT_MSG(comm != nullptr, "no NCCL communicator for this device: call ncclInitRank / ncclInitAll first");
        ClusteringParameters cp;
        if (niter > 0)
            cp.niter = niter;
        if (seed >= 0)
            cp.seed = seed;
        Clustering clus((int)d, (int)k, cp);
        GpuIndexFlatConfig fc;
        fc.device = device;
        GpuIndexFlatL2 index(res, (int)d, fc);
        clus.trainSharded((idx_t)n_local, x_local, index, *comm);
        memcpy(centroids_out, clus.centroids.data(), sizeof(float) * d * k);
        if (obj_out) {
            for (size_t i = 0; i < clus.iteration_stats.size() && (int)i < cp.niter; i++)
                obj_out[i] = clus.iteration_stats[i].obj;
        }
        if (stats_out) {
            stats_out[0] = clus.iteration_stats.empty() ? 0 : clus.iteration_stats.back().time;
            stats_out[1] = clus.iteration_stats.empty() ? 0 : clus.iteration_stats.back().time_search;
            stats_out[2] = clus.splitSeconds;
            double ns = 0;
            for (auto& s : clus.iteration_stats)
                ns += s.nsplit;
            stats_out[3] = ns;
        }
    }
    CATCH_AND_HANDLE
}

int faiss_b200_pq_train(
        FaissStandardGpuResources* r,
        int device,
        size_t d,
        size_t M,
        size_t n,
        const float* x,
        int niter,
        int seed,
        float* centroids_out) {
    try {
        auto res = RES(r);
        FB_THROW_IF_NOT_MSG(M > 0 && d % M == 0, "Number of sub-quantizers must be an integer divisor of the number of dimensions");
        ClusteringParameters cp; // ProductQuantizer::cp defaults (faiss/impl/ProductQuantizer.h)
        if (niter > 0)
            cp.niter = niter;
        if (seed >= 0)
            cp.seed = seed;
        DeviceScope scope(device);
        res->initializeForDevice(device);
        cudaStream_t stream = res->getDefaultStream(device);
        GpuMemoryReservation hold;
        const float* xd = x;
        if (getDeviceForAddress(x) != device) {
            hold = res->device_alloc(device, sizeof(float) * n * d, AllocType::Other);
            CUDA_VERIFY(cudaMemcpyAsync(hold.data, x, sizeof(float) * n * d, cudaMemcpyDefault, stream));
            xd = hold.as<float>();
        }
        trainProductQuantizer(res, device, (idx_t)n, xd, (int)d, (int)M, 256, cp, centroids_out);
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- instrumentation
long long faiss_b200_launch_count(void) {
    return fb200::kernelLaunchCounter();
}
void faiss_b200_kernel_timing(int enable) {
    fb200::KernelTiming::enable(enable != 0);
}
int faiss_b200_kernel_timing_collect(const char* name, double* ms, int* launches) {
    try {
        fb200::KernelTiming::collect(name, ms, launches);
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- host utilities
int faiss_b200_rand_perm(int* perm, size_t n, int64_t seed) {
    try {
        fb200::rand_perm(perm, n, seed);
    }
    CATCH_AND_HANDLE
}
int faiss_b200_split_clusters(size_t d, size_t k, size_t n, float* hassign, float* centroids, int* nsplit_out) {
    try {
        int ns = fb200::split_clusters(d, k, n, hassign, centroids);
        if (nsplit_out)
            *nsplit_out = ns;
    }
    CATCH_AND_HANDLE
}
int faiss_b200_merge_knn_results_host(
        idx_t n,
        idx_t k,
        int nshard,
        FaissMetricType metric,
        const float* all_distances,
        const idx_t* all_labels,
        float* distances,
        idx_t* labels) {
    try {
        merge_knn_results_host(n, k, nshard, MT(metric), all_distances, all_labels, distances, labels);
    }
    CATCH_AND_HANDLE
}

// ---------------------------------------------------------------- tier 2 seams
int b200_l2_norms(FaissStandardGpuResources* r, int device, const float* x, idx_t n, int d, float* norms) {
    try {
        auto res = RES(r);
        DeviceScope s(device);
        runL2Norms(x, n, d, norms, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
// bfKnn (faiss/gpu/GpuDistance.h:33-181, GpuDistance.cu:229-571) for row-major fp32 vectors and queries: the
// FaissGpuDistanceParams entry point with the other fields at their defaults.
int faiss_b200_bfKnn(
        FaissStandardGpuResources* r,
        int device,
        FaissMetricType metric,
        idx_t k,
        int dims,
        const float* vectors,
        idx_t num_vectors,
        const float* queries,
        idx_t num_queries,
        float* out_distances,
        idx_t* out_indices) {
    return faiss_b200_bfKnn_ex(
            r, device, metric, 0.f, k, dims, vectors, num_vectors, queries, num_queries, out_distances, out_indices);
}
// GpuDistanceParams::metricArg (faiss/gpu/GpuDistance.h:41): the exponent of METRIC_Lp
int faiss_b200_bfKnn_ex(
        FaissStandardGpuResources* r,
        int device,
        FaissMetricType metric,
        float metric_arg,
        idx_t k,
        int dims,
        const float* vectors,
        idx_t num_vectors,
        const float* queries,
        idx_t num_queries,
        float* out_distances,
        idx_t* out_indices) {
    try {
        auto res = RES(r);
        FB_THROW_IF_NOT_MSG(k >= 1 && k <= kMaxK, "bfKnn: k out of range");
        GpuDistanceParams a;
        a.metric = MT(metric);
        a.metricArg = metric_arg;
        a.k = (int)k;
        a.dims = dims;
        a.vectors = vectors;
        a.numVectors = num_vectors;
        a.queries = queries;
        a.numQueries = num_queries;
        a.outDistances = out_distances;
        a.outIndices = out_indices;
        a.device = device;
        bfKnn(res, a);
    }
    CATCH_AND_HANDLE
}

// FaissGpuDistanceParams -> GpuDistanceParams; every field is checked by validateDistanceParams before any CUDA call
static GpuDistanceParams DP(const FaissGpuDistanceParams* p) {
    if (!p)
        FB_THROW_MSG("null distance parameters");
    GpuDistanceParams a;
    a.metric = MT(p->metric);
    a.metricArg = p->metricArg;
    a.k = p->k;
    a.dims = p->dims;
    a.vectors = p->vectors;
    a.vectorType = (DistanceDataType)(int)p->vectorType;
    a.vectorsRowMajor = p->vectorsRowMajor != 0;
    a.numVectors = p->numVectors;
    a.queries = p->queries;
    a.queryType = (DistanceDataType)(int)p->queryType;
    a.queriesRowMajor = p->queriesRowMajor != 0;
    a.numQueries = p->numQueries;
    a.outDistances = p->outDistances;
    a.outIndicesType = (IndicesDataType)(int)p->outIndicesType;
    a.outIndices = p->outIndices;
    a.device = p->device;
    validateDistanceParams(a);
    return a;
}
int faiss_b200_bfKnn_params(FaissStandardGpuResources* r, const FaissGpuDistanceParams* params) {
    try {
        const GpuDistanceParams a = DP(params);
        bfKnn(RES(r), a);
    }
    CATCH_AND_HANDLE
}
int faiss_b200_bfKnn_tiling(
        FaissStandardGpuResources* r,
        const FaissGpuDistanceParams* params,
        size_t vectorsMemoryLimit,
        size_t queriesMemoryLimit) {
    try {
        const GpuDistanceParams a = DP(params);
        bfKnn_tiling(RES(r), a, vectorsMemoryLimit, queriesMemoryLimit);
    }
    CATCH_AND_HANDLE
}
struct FaissGpuIcmEncoder_H {
    std::unique_ptr<GpuIcmEncoder> enc;
};
static GpuIcmEncoder* ICM(FaissGpuIcmEncoder* p) {
    if (!p || !p->enc)
        FB_THROW_MSG("null encoder handle");
    return p->enc.get();
}
int faiss_GpuIcmEncoder_new(FaissGpuIcmEncoder** p, int M, int K, int d, int ndevices, FaissStandardGpuResources** r, const int* devices) {
    try {
        FB_THROW_IF_NOT_MSG(p != nullptr && r != nullptr && devices != nullptr, "null argument");
        FB_THROW_IF_NOT_MSG(ndevices >= 1, "at least one device is needed");
        std::vector<std::shared_ptr<GpuResources>> res;
        std::vector<int> devs;
        for (int i = 0; i < ndevices; i++) {
            res.push_back(RES(r[i]));
            devs.push_back(devices[i]);
        }
        auto h = std::make_unique<FaissGpuIcmEncoder_H>();
        h->enc = std::make_unique<GpuIcmEncoder>(M, K, d, std::move(res), std::move(devs));
        *p = h.release();
    }
    CATCH_AND_HANDLE
}
void faiss_GpuIcmEncoder_free(FaissGpuIcmEncoder* p) {
    delete p;
}
int faiss_GpuIcmEncoder_set_binary_term(FaissGpuIcmEncoder* p, const float* codebooks) {
    try {
        ICM(p)->setBinaryTerm(codebooks);
    }
    CATCH_AND_HANDLE
}
int faiss_GpuIcmEncoder_encode(
        FaissGpuIcmEncoder* p, int32_t* codes, const float* x, idx_t n, size_t ils_iters, size_t nperts, size_t icm_iters,
        const int32_t* perturbations) {
    try {
        ICM(p)->encode(codes, x, n, ils_iters, nperts, icm_iters, perturbations);
    }
    CATCH_AND_HANDLE
}
int b200_icm_encode_paged(
        FaissGpuIcmEncoder* p, int32_t* codes, const float* x, idx_t n, size_t ils_iters, size_t nperts, size_t icm_iters,
        const int32_t* perturbations, size_t page_bytes) {
    try {
        ICM(p)->encode(codes, x, n, ils_iters, nperts, icm_iters, perturbations, page_bytes);
    }
    CATCH_AND_HANDLE
}
struct FaissGpuRqEncoder_H {
    std::unique_ptr<GpuRqEncoder> enc;
};
static GpuRqEncoder* RQ(const FaissGpuRqEncoder* p) {
    if (!p || !p->enc)
        FB_THROW_MSG("null encoder handle");
    return p->enc.get();
}
int faiss_b200_RqEncoder_new(FaissGpuRqEncoder** p, FaissStandardGpuResources* r, int device, int d, int M, const int* nbits) {
    try {
        FB_THROW_IF_NOT_MSG(p != nullptr && nbits != nullptr, "null argument");
        FB_THROW_IF_NOT_FMT(M >= 1, "M = %d: at least one codebook is needed", M);
        auto h = std::make_unique<FaissGpuRqEncoder_H>();
        h->enc = std::make_unique<GpuRqEncoder>(d, std::vector<int>(nbits, nbits + M), RES(r), device);
        *p = h.release();
    }
    CATCH_AND_HANDLE
}
void faiss_b200_RqEncoder_free(FaissGpuRqEncoder* p) {
    delete p;
}
int faiss_b200_RqEncoder_set_codebooks(FaissGpuRqEncoder* p, const float* codebooks) {
    try {
        RQ(p)->setCodebooks(codebooks);
    }
    CATCH_AND_HANDLE
}
int faiss_b200_RqEncoder_final_beam(const FaissGpuRqEncoder* p, int beam_in, int out_beam, int* beam) {
    try {
        FB_THROW_IF_NOT_MSG(beam != nullptr, "null argument");
        *beam = RQ(p)->finalBeam(beam_in, out_beam);
    }
    CATCH_AND_HANDLE
}
int faiss_b200_RqEncoder_refine_beam(
        FaissGpuRqEncoder* p, idx_t n, int beam_in, const float* residuals, int out_beam, int32_t* codes, float* residuals_out,
        float* distances) {
    return b200_rq_refine_beam_paged(p, n, beam_in, residuals, out_beam, codes, residuals_out, distances, kRqPageBytes);
}
int b200_rq_refine_beam_paged(
        FaissGpuRqEncoder* p, idx_t n, int beam_in, const float* residuals, int out_beam, int32_t* codes, float* residuals_out,
        float* distances, size_t page_bytes) {
    try {
        RQ(p)->refineBeam(n, beam_in, residuals, out_beam, codes, residuals_out, distances, page_bytes);
    }
    CATCH_AND_HANDLE
}
int faiss_b200_RqEncoder_refine_beam_lut(FaissGpuRqEncoder* p, idx_t n, const float* x, int out_beam, int32_t* codes, float* distances) {
    return b200_rq_refine_beam_lut_paged(p, n, x, out_beam, codes, distances, kRqPageBytes);
}
int b200_rq_refine_beam_lut_paged(
        FaissGpuRqEncoder* p, idx_t n, const float* x, int out_beam, int32_t* codes, float* distances, size_t page_bytes) {
    try {
        RQ(p)->refineBeamLUT(n, x, out_beam, codes, distances, page_bytes);
    }
    CATCH_AND_HANDLE
}
int faiss_b200_RqEncoder_compute_codes(
        FaissGpuRqEncoder* p, const float* x, idx_t n, int use_beam_lut, int max_beam, int search_type, float norm_min,
        float norm_max, const float* centroids, uint8_t* packed) {
    return b200_rq_compute_codes_paged(
            p, x, n, use_beam_lut, max_beam, search_type, norm_min, norm_max, centroids, packed, kRqPageBytes);
}
int b200_rq_compute_codes_paged(
        FaissGpuRqEncoder* p, const float* x, idx_t n, int use_beam_lut, int max_beam, int search_type, float norm_min,
        float norm_max, const float* centroids, uint8_t* packed, size_t page_bytes) {
    try {
        RQ(p)->computeCodes(x, n, use_beam_lut != 0, max_beam, search_type, norm_min, norm_max, centroids, packed, page_bytes);
    }
    CATCH_AND_HANDLE
}
int faiss_b200_RqEncoder_encode_unpacked(
        FaissGpuRqEncoder* p, const float* x, idx_t n, int use_beam_lut, int max_beam, int32_t* codes) {
    try {
        RQ(p)->encodeUnpacked(x, n, use_beam_lut != 0, max_beam, codes);
    }
    CATCH_AND_HANDLE
}
// test seam: k = -1 into a host-resident matrix with a block budget other than kPairwisePageBytes
int b200_pairwise_paged(FaissStandardGpuResources* r, const FaissGpuDistanceParams* params, size_t page_bytes) {
    try {
        const GpuDistanceParams a = DP(params);
        bfKnn(RES(r), a, page_bytes);
    }
    CATCH_AND_HANDLE
}
int b200_flat_search_exact(
        FaissStandardGpuResources* r,
        int device,
        const float* Y,
        idx_t N,
        int d,
        const float* Q,
        idx_t nq,
        int k,
        FaissMetricType metric,
        float* D,
        idx_t* I) {
    try {
        auto res = RES(r);
        DeviceScope s(device);
        FB_THROW_IF_NOT(k >= 1 && k <= kMaxK);
        runFlatExact(res.get(), device, Q, nq, Y, N, d, k, MT(metric), 0, D, I, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
int b200_topk_merge(
        FaissStandardGpuResources* r,
        int device,
        const float* D_in,
        const idx_t* I_in,
        idx_t nq,
        int nshard,
        int k_in,
        const idx_t* id_offsets,
        int k,
        FaissMetricType metric,
        float* D,
        idx_t* I) {
    try {
        auto res = RES(r);
        DeviceScope s(device);
        FB_THROW_IF_NOT(k >= 1 && k <= kMaxK);
        runMergeTopK(D_in, I_in, nq, nshard, k_in, id_offsets, k, MT(metric), D, I, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
int b200_flat_tc_scores_debug(
        FaissStandardGpuResources* r,
        int device,
        const void* Q16,
        idx_t nq,
        const void* Y16,
        idx_t N,
        int dpad,
        float* S) {
    try {
        auto res = RES(r);
        DeviceScope s(device);
        runFlatTcScoresDebug(Q16, nq, Y16, N, dpad, false, S, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
int b200_flat_tc_scores_debug_s8(FaissStandardGpuResources* r, int device, const void* Q8, idx_t nq, const void* Y8, idx_t N, float* S) {
    try {
        auto res = RES(r);
        DeviceScope s(device);
        runFlatTcScoresDebug(Q8, nq, Y8, N, 128, true, S, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
// ---- the remaining tier-2 seams of SURVEY 8(b): the reference's internal run* launchers on raw device buffers
int b200_ivf_coarse(
        FaissStandardGpuResources* r,
        int device,
        const float* centroids,
        idx_t nlist,
        int d,
        const float* Q,
        idx_t nq,
        int nprobe,
        FaissMetricType metric,
        float* coarse_dis,
        idx_t* coarse_ids) {
    try {
        // IVFBase::searchCoarseQuantizer_ (faiss/gpu/impl/IVFBase.cu:509-545) = a Flat search with k = nprobe
        auto res = RES(r);
        DeviceScope s(device);
        FB_THROW_IF_NOT(nprobe >= 1 && nprobe <= kMaxNprobe);
        runFlatExact(res.get(), device, Q, nq, centroids, nlist, d, nprobe, MT_L2IP(metric), 0, coarse_dis, coarse_ids, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
int b200_kmeans_assign(
        FaissStandardGpuResources* r,
        int device,
        const float* centroids,
        idx_t k,
        int d,
        const float* x,
        idx_t n,
        FaissMetricType metric,
        float* dis,
        idx_t* assign) {
    try {
        // Clustering's index.search(n, x, 1) (faiss/Clustering.cpp:270-290) on raw device buffers, exact SIMT arithmetic
        auto res = RES(r);
        DeviceScope s(device);
        runFlatArgmin(res.get(), device, x, n, centroids, k, d, MT_L2IP(metric), dis, assign, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
int b200_ivfflat_scan(
        FaissStandardGpuResources* r,
        int device,
        const float* Q,
        idx_t nq,
        int d,
        const idx_t* probes,
        int nprobe,
        const int64_t* list_start,
        const int* list_len,
        const float* arena_vecs,
        const idx_t* arena_ids,
        idx_t arena_elems,
        int k,
        FaissMetricType metric,
        float* D,
        idx_t* I) {
    try {
        // runIVFInterleavedScan (faiss/gpu/impl/IVFInterleaved.cu:179): lists = row-major fp32 runs of one arena
        auto res = RES(r);
        DeviceScope s(device);
        FB_THROW_IF_NOT(k >= 1 && k <= kMaxK && nprobe >= 1 && nprobe <= kMaxNprobe);
        IvfScanLayout a;
        a.kind = IVF_STORED_FLAT;
        a.d = d;
        a.listStart = list_start;
        a.listLen = list_len;
        a.arenaElems = arena_elems;
        a.codes = reinterpret_cast<const uint8_t*>(arena_vecs);
        a.ids = arena_ids;
        const IvfScanCall c{Q, nq, probes, nullptr, nprobe, k, MT_L2IP(metric), D, I, res->getDefaultStream(device)};
        runIvfScan(res.get(), device, a, c);
    }
    CATCH_AND_HANDLE
}
int b200_ivfpq_scan(
        FaissStandardGpuResources* r,
        int device,
        const float* Q,
        idx_t nq,
        int d,
        const idx_t* probes,
        const float* coarse_dis,
        int nprobe,
        const float* coarse_centroids,
        const float* pq_centroids,
        int M,
        const int64_t* list_start,
        const int* list_len,
        const uint8_t* arena_codes,
        const idx_t* arena_ids,
        int k,
        FaissMetricType metric,
        float* D,
        idx_t* I) {
    try {
        // runPQScanMultiPassNoPrecomputed (faiss/gpu/impl/PQScanMultiPassNoPrecomputed-inl.cuh:527) over vector-major
        // [len][M] codes (the CPU ArrayInvertedLists bytes); pq_centroids [M][256][d/M]
        auto res = RES(r);
        DeviceScope s(device);
        FB_THROW_IF_NOT(k >= 1 && k <= kMaxK && nprobe >= 1 && nprobe <= kMaxNprobe);
        IvfScanLayout a;
        a.kind = IVF_STORED_PQ;
        a.d = d;
        a.listStart = list_start;
        a.listLen = list_len;
        a.codes = arena_codes;
        a.ids = arena_ids;
        a.centroids = coarse_centroids;
        a.M = M;
        a.nbits = 8;
        a.pq = pq_centroids;
        const IvfScanCall c{Q, nq, probes, coarse_dis, nprobe, k, MT_L2IP(metric), D, I, res->getDefaultStream(device)};
        runIvfScan(res.get(), device, a, c);
    }
    CATCH_AND_HANDLE
}
int b200_ivf_append(
        FaissStandardGpuResources* r,
        int device,
        const uint8_t* rows,
        const idx_t* ids,
        const idx_t* assign,
        idx_t n,
        int code_size,
        idx_t nlist,
        const int64_t* list_start,
        int* list_len,
        uint8_t* arena_codes,
        idx_t* arena_ids) {
    try {
        // device-side append bookkeeping (role of IVFBase::addVectorsToLists_ + runIVFAppend, faiss/gpu/impl/IVFBase.cu:693-905,
        // IVFAppend.cu:265): stable offsets inside each list, scatter, list lengths advanced; capacity is the caller's
        auto res = RES(r);
        DeviceScope s(device);
        cudaStream_t stream = res->getDefaultStream(device);
        auto offsets = res->temp(device, sizeof(int) * std::max<idx_t>(n, 1));
        runIvfAppendOffsets(assign, n, nlist, list_len, offsets.as<int>(), nullptr, stream);
        runIvfScatter(rows, ids, assign, offsets.as<int>(), n, code_size, list_start, arena_codes, arena_ids, stream);
        runIvfCountAssign(assign, n, nlist, list_len, stream);
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
    CATCH_AND_HANDLE
}
int b200_pq_encode(
        FaissStandardGpuResources* r,
        int device,
        const float* resid,
        idx_t n,
        int d,
        int M,
        const float* pq,
        uint8_t* codes) {
    try {
        auto res = RES(r);
        DeviceScope s(device);
        runPQEncode(resid, n, d, M, 256, pq, codes, res->getDefaultStream(device));
    }
    CATCH_AND_HANDLE
}
int b200_kmeans_update(
        FaissStandardGpuResources* r,
        int device,
        const float* x,
        const idx_t* assign,
        idx_t n,
        int d,
        idx_t k,
        float* sums,
        float* counts,
        float* centroids) {
    try {
        auto res = RES(r);
        DeviceScope s(device);
        auto st = res->getDefaultStream(device);
        runKmeansAccumulate(x, assign, n, d, k, sums, counts, st);
        if (centroids)
            runKmeansFinalize(sums, counts, k, d, centroids, st);
    }
    CATCH_AND_HANDLE
}

} // extern "C"
