// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points around the reference's IndexHNSWCagra, compiled by oracle/Makefile into
// oracle/_ref/libfaiss_ref_cagra.so against the UNMODIFIED reference CPU library (oracle/_ref/libfaiss_ref.so).  The
// product (faiss_b200/) never loads this file.
//   ref_cagra_search_graph  an IndexHNSWCagra made from (xb, graph) as GpuIndexCagra::copyTo makes it
//                           (faiss/gpu/GpuIndexCagra.cu copyTo), base_level_only or with HNSW upper levels, then searched
//   ref_cagra_build_cpu     an IndexHNSWCagra built on the CPU with add, and its level-0 neighbour table

#include <faiss/IndexFlat.h>
#include <faiss/IndexHNSW.h>

#include <cmath>

#include "ref_shim.h"

extern "C" {

// metric: 0 inner product, 1 L2 (faiss::MetricType); graph [n][degree] int64, degree even
int ref_cagra_search_graph(
        int d, int metric, int64_t n, const float* xb, const int64_t* graph, int degree, int base_level_only,
        int64_t nq, const float* xq, int64_t k, int efSearch, float* D, int64_t* I) {
    REF_TRY const int M = degree / 2;
    faiss::IndexHNSWCagra index(d, M, (faiss::MetricType)metric);
    index.base_level_only = base_level_only != 0;
    index.is_trained = true;
    index.hnsw.is_similarity = metric == (int)faiss::METRIC_INNER_PRODUCT;
    index.keep_max_size_level0 = true;
    index.hnsw.reset();
    index.hnsw.assign_probas.clear();
    index.hnsw.cum_nneighbor_per_level.clear();
    index.hnsw.set_default_probas(M, 1.0 / std::log(M));
    index.init_level0 = false;
    if (!index.base_level_only) {
        index.add(n, xb);
    } else {
        index.hnsw.prepare_level_tab(n, false);
        index.storage->add(n, xb);
        index.ntotal = n;
    }
    for (int64_t i = 0; i < n; i++) {
        size_t begin, end;
        index.hnsw.neighbor_range(i, 0, &begin, &end);
        for (size_t j = begin; j < end; j++)
            index.hnsw.neighbors[j] = (faiss::HNSW::storage_idx_t)graph[i * degree + (j - begin)];
    }
    index.init_level0 = true;
    faiss::SearchParametersHNSW p;
    p.efSearch = efSearch;
    index.search(nq, xq, k, D, I, &p);
    REF_CATCH
}

// graph [n][2 * M] int64 (-1 where a row has fewer neighbours)
int ref_cagra_build_cpu(int d, int metric, int M, int64_t n, const float* xb, int64_t* graph) {
    REF_TRY faiss::IndexHNSWCagra index(d, M, (faiss::MetricType)metric);
    index.add(n, xb);
    const int degree = index.hnsw.nb_neighbors(0);
    for (int64_t i = 0; i < n; i++) {
        size_t begin, end;
        index.hnsw.neighbor_range(i, 0, &begin, &end);
        for (size_t j = begin; j < end; j++)
            graph[i * degree + (j - begin)] = index.hnsw.neighbors[j];
    }
    REF_CATCH
}

} // extern "C"
