// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's CPU all-pairs distances, built by oracle/pairwise.mk into
// oracle/_ref/libfaiss_ref_pairwise.so against the UNMODIFIED reference CPU library of oracle/Makefile.  Every
// function forwards to a reference entry point.  The product (faiss_b200/) never loads this file.

#include <faiss/MetricType.h>
#include <faiss/utils/distances.h>
#include <faiss/utils/extra_distances.h>

#include <string>

static thread_local std::string g_err;

extern "C" {

const char* ref_pairwise_last_error() {
    return g_err.c_str();
}

// faiss::pairwise_L2sqr (faiss/utils/distances.h:116-125) over row-major xq [nq, d], xb [nb, d] -> dis [nq, nb]
int ref_pairwise_L2sqr(int64_t d, int64_t nq, const float* xq, int64_t nb, const float* xb, float* dis) {
    try {
        faiss::pairwise_L2sqr(d, nq, xq, nb, xb, dis);
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
    return 0;
}

// faiss::pairwise_extra_distances (faiss/utils/extra_distances.h:25-37): every metric of VectorDistance, inner
// product included
int ref_pairwise_extra_distances(
        int64_t d,
        int64_t nq,
        const float* xq,
        int64_t nb,
        const float* xb,
        int metric,
        float metric_arg,
        float* dis) {
    try {
        faiss::pairwise_extra_distances(d, nq, xq, nb, xb, (faiss::MetricType)metric, metric_arg, dis);
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
    return 0;
}

} // extern "C"
