// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's IndexIVFScalarQuantizer, compiled by oracle/sq.mk into
// oracle/_ref/libfaiss_ref_sq.so against the UNMODIFIED reference CPU library (oracle/_ref/libfaiss_ref.so).
// Like ref_shim.cpp it contains no algorithm of its own: every function forwards to a reference entry point.
// The generic Index / IndexIVF functions of ref_shim.cpp (train, add, search, lists, centroids,
// search_preassigned) apply to these handles as well.  The product (faiss_b200/) never loads this file.

#include <faiss/IndexFlat.h>
#include <faiss/IndexScalarQuantizer.h>
#include <faiss/impl/ScalarQuantizer.h>

#include <cstring>
#include <string>

static thread_local std::string g_sq_err;

#define SQ_TRY try {
#define SQ_CATCH                      \
    }                                 \
    catch (const std::exception& e) { \
        g_sq_err = e.what();          \
        return -1;                    \
    }                                 \
    return 0;

extern "C" {

const char* ref_sq_last_error() {
    return g_sq_err.c_str();
}

// faiss/IndexScalarQuantizer.cpp:122-145 (IndexIVFScalarQuantizer constructor) over an IndexFlat quantizer
void* ref_ivfsq_new(int d, int64_t nlist, int qtype, int metric /*0=IP 1=L2*/, int by_residual) {
    try {
        auto mt = metric == 0 ? faiss::METRIC_INNER_PRODUCT : faiss::METRIC_L2;
        auto* q = new faiss::IndexFlat(d, mt);
        auto* idx = new faiss::IndexIVFScalarQuantizer(
                q, d, nlist, (faiss::ScalarQuantizer::QuantizerType)qtype, mt, by_residual != 0);
        idx->own_fields = true;
        return idx;
    } catch (const std::exception& e) {
        g_sq_err = e.what();
        return nullptr;
    }
}

// ScalarQuantizer::trained (faiss/impl/ScalarQuantizer.h)
int64_t ref_ivfsq_trained_size(void* idx) {
    return (int64_t)((faiss::IndexIVFScalarQuantizer*)idx)->sq.trained.size();
}
int ref_ivfsq_get_trained(void* idx, float* out) {
    SQ_TRY const auto& t = ((faiss::IndexIVFScalarQuantizer*)idx)->sq.trained;
    if (!t.empty())
        memcpy(out, t.data(), sizeof(float) * t.size());
    SQ_CATCH
}
int ref_ivfsq_set_trained(void* idx, const float* t, int64_t n) {
    SQ_TRY((faiss::IndexIVFScalarQuantizer*)idx)->sq.trained.assign(t, t + n);
    SQ_CATCH
}
int64_t ref_ivfsq_code_size(void* idx) {
    return (int64_t)((faiss::IndexIVFScalarQuantizer*)idx)->sq.code_size;
}
int ref_ivfsq_set_rangestat(void* idx, int rangestat, float arg) {
    SQ_TRY auto& sq = ((faiss::IndexIVFScalarQuantizer*)idx)->sq;
    sq.rangestat = (faiss::ScalarQuantizer::RangeStat)rangestat;
    sq.rangestat_arg = arg;
    SQ_CATCH
}
// IndexIVFScalarQuantizer::encode_vectors (faiss/IndexScalarQuantizer.cpp:162-200), without list numbers in the code
int ref_ivfsq_encode(void* idx, int64_t n, const float* x, const int64_t* list_nos, uint8_t* codes) {
    SQ_TRY((faiss::IndexIVFScalarQuantizer*)idx)->encode_vectors(n, x, list_nos, codes, false);
    SQ_CATCH
}

} // extern "C"
