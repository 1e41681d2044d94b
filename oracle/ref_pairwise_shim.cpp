// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's CPU all-pairs distances, built by oracle/Makefile into
// oracle/_ref/libfaiss_ref_pairwise.so against the UNMODIFIED reference CPU library of oracle/Makefile.  Every
// function forwards to a reference entry point.  The product (faiss_b200/) never loads this file.

#include <faiss/MetricType.h>
#include <faiss/utils/distances.h>
#include <faiss/utils/extra_distances.h>

#include "ref_shim.h"

extern "C" {

// faiss::pairwise_L2sqr (faiss/utils/distances.h:116-125) over row-major xq [nq, d], xb [nb, d] -> dis [nq, nb]
int ref_pairwise_L2sqr(int64_t d, int64_t nq, const float* xq, int64_t nb, const float* xb, float* dis) {
    REF_TRY faiss::pairwise_L2sqr(d, nq, xq, nb, xb, dis);
    REF_CATCH
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
    REF_TRY faiss::pairwise_extra_distances(d, nq, xq, nb, xb, (faiss::MetricType)metric, metric_arg, dis);
    REF_CATCH
}

} // extern "C"
