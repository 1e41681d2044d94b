// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's extra metrics (L1, Linf, Lp, Canberra, BrayCurtis,
// JensenShannon, Jaccard, Gower), built by oracle/Makefile into oracle/_ref/libfaiss_ref_metrics.so
// against the UNMODIFIED reference CPU library of oracle/Makefile.  Every function forwards to a
// reference entry point; the handles are reference faiss::Index objects, so oracle/ref.py's generic
// index calls apply to them.  The product (faiss_b200/) never loads this file.

#include <faiss/IndexFlat.h>
#include <faiss/impl/FaissException.h>
#include <faiss/utils/extra_distances.h>

#include "ref_shim.h"

extern "C" {

// faiss::IndexFlat(d, metric) with Index::metric_arg set (faiss/IndexFlat.cpp:40-60 dispatches the extra
// metrics to knn_extra_metrics); null on error
void* ref_flat_new_ex(int d, int metric, float metric_arg) {
    REF_TRY auto* idx = new faiss::IndexFlat(d, (faiss::MetricType)metric);
    idx->metric_arg = metric_arg;
    return idx;
    REF_CATCH_RET(nullptr)
}

// faiss::knn_extra_metrics (faiss/utils/extra_distances.cpp:93-137) over row-major x [nx, d], y [ny, d]
int ref_knn_extra_metrics(
        const float* x,
        const float* y,
        int64_t d,
        int64_t nx,
        int64_t ny,
        int metric,
        float metric_arg,
        int64_t k,
        float* distances,
        int64_t* indexes) {
    REF_TRY faiss::knn_extra_metrics(
            x, y, (size_t)d, (size_t)nx, (size_t)ny, (faiss::MetricType)metric, metric_arg, (size_t)k, distances,
            indexes);
    REF_CATCH
}

} // extern "C"
