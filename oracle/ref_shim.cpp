// TEST INFRASTRUCTURE ONLY.
//
// A thin extern "C" shim over the UNMODIFIED reference CPU library (compiled from the
// reference tree by oracle/Makefile into oracle/_ref/libfaiss_ref.so).  It exposes the
// reference's own IndexFlat / IndexIVFFlat / IndexIVFPQ / Clustering / IndexShards objects
// to the Python test-suite and to bench.py's cpu_baseline / --impl reference legs through
// ctypes.  It contains no algorithm of its own: every function forwards to a reference
// entry point (cited per function).  The product (faiss_b200/) never loads this file.

#include <faiss/Clustering.h>
#include <faiss/IndexFlat.h>
#include <faiss/IndexIVFFlat.h>
#include <faiss/IndexIVFPQ.h>
#include <faiss/IndexShards.h>
#include <faiss/impl/FaissException.h>
#include <faiss/impl/ProductQuantizer.h>
#include <faiss/invlists/InvertedLists.h>
#include <faiss/utils/Heap.h>
#include <faiss/utils/distances.h>
#include <faiss/utils/random.h>
#include <faiss/utils/utils.h>
#include <omp.h>

#include <cstring>
#include <string>

#include "ref_shim.h"

using faiss::idx_t;

// the error slot of this library and of every shim library linked against it (ref_shim.h)
static thread_local std::string g_err;

extern "C" {

void ref_set_last_error(const char* msg) {
    g_err = msg;
}
const char* ref_last_error() {
    return g_err.c_str();
}

int ref_omp_max_threads() {
    return omp_get_max_threads();
}
void ref_omp_set_threads(int n) {
    omp_set_num_threads(n);
}
const char* ref_compile_options() {
    static std::string s = faiss::get_compile_options();
    return s.c_str();
}

// faiss/utils/random.cpp:95-113
void ref_float_rand(float* x, size_t n, int64_t seed) {
    faiss::float_rand(x, n, seed);
}
// faiss/utils/random.cpp (rand_perm) -- used by Clustering init
void ref_rand_perm(int* perm, size_t n, int64_t seed) {
    faiss::rand_perm(perm, n, seed);
}

// ---------------------------------------------------------------- generic Index
void ref_index_free(void* idx) {
    delete (faiss::Index*)idx;
}
int ref_index_train(void* idx, int64_t n, const float* x) {
    REF_TRY((faiss::Index*)idx)->train(n, x);
    REF_CATCH
}
int ref_index_add(void* idx, int64_t n, const float* x) {
    REF_TRY((faiss::Index*)idx)->add(n, x);
    REF_CATCH
}
int ref_index_add_with_ids(void* idx, int64_t n, const float* x, const int64_t* ids) {
    REF_TRY((faiss::Index*)idx)->add_with_ids(n, x, ids);
    REF_CATCH
}
// faiss/Index.h:183 search()
int ref_index_search(void* idx, int64_t n, const float* x, int64_t k, float* D, int64_t* I) {
    REF_TRY((faiss::Index*)idx)->search(n, x, k, D, I);
    REF_CATCH
}
int ref_index_assign(void* idx, int64_t n, const float* x, int64_t* labels, int64_t k) {
    REF_TRY((faiss::Index*)idx)->assign(n, x, labels, k);
    REF_CATCH
}
int ref_index_reconstruct_n(void* idx, int64_t i0, int64_t ni, float* out) {
    REF_TRY((faiss::Index*)idx)->reconstruct_n(i0, ni, out);
    REF_CATCH
}
int ref_index_compute_residual_n(void* idx, int64_t n, const float* x, float* res, const int64_t* keys) {
    REF_TRY((faiss::Index*)idx)->compute_residual_n(n, x, res, keys);
    REF_CATCH
}
int ref_index_reset(void* idx) {
    REF_TRY((faiss::Index*)idx)->reset();
    REF_CATCH
}
int64_t ref_index_ntotal(void* idx) {
    return ((faiss::Index*)idx)->ntotal;
}
int ref_index_is_trained(void* idx) {
    return ((faiss::Index*)idx)->is_trained;
}

// ---------------------------------------------------------------- IndexFlat (faiss/IndexFlat.h)
void* ref_flat_new(int d, int metric /*0=IP 1=L2*/) {
    return new faiss::IndexFlat(d, metric == 0 ? faiss::METRIC_INNER_PRODUCT : faiss::METRIC_L2);
}
const float* ref_flat_xb(void* idx) {
    return ((faiss::IndexFlat*)idx)->get_xb();
}

// ---------------------------------------------------------------- IVF common (faiss/IndexIVF.h)
void ref_ivf_set_nprobe(void* idx, int64_t nprobe) {
    ((faiss::IndexIVF*)idx)->nprobe = nprobe;
}
int64_t ref_ivf_nlist(void* idx) {
    return ((faiss::IndexIVF*)idx)->nlist;
}
void ref_ivf_set_cp(void* idx, int niter, int seed, int max_points_per_centroid) {
    auto* ivf = (faiss::IndexIVF*)idx;
    if (niter > 0)
        ivf->cp.niter = niter;
    if (seed >= 0)
        ivf->cp.seed = seed;
    if (max_points_per_centroid > 0)
        ivf->cp.max_points_per_centroid = max_points_per_centroid;
}
// coarse centroids [nlist, d] (quantizer is an IndexFlat we created)
int ref_ivf_get_centroids(void* idx, float* out) {
    REF_TRY auto* ivf = (faiss::IndexIVF*)idx;
    ivf->quantizer->reconstruct_n(0, ivf->nlist, out);
    REF_CATCH
}
// install centroids into the coarse quantizer (is_trained for the coarse level)
int ref_ivf_set_centroids(void* idx, const float* c) {
    REF_TRY auto* ivf = (faiss::IndexIVF*)idx;
    ivf->quantizer->reset();
    ivf->quantizer->add(ivf->nlist, c);
    REF_CATCH
}
int64_t ref_ivf_list_size(void* idx, int64_t l) {
    return ((faiss::IndexIVF*)idx)->invlists->list_size(l);
}
int64_t ref_ivf_code_size(void* idx) {
    return ((faiss::IndexIVF*)idx)->invlists->code_size;
}
// copies list l's codes (list_size*code_size bytes) and ids (list_size int64)
int ref_ivf_get_list(void* idx, int64_t l, uint8_t* codes, int64_t* ids) {
    REF_TRY auto* il = ((faiss::IndexIVF*)idx)->invlists;
    size_t n = il->list_size(l);
    faiss::InvertedLists::ScopedCodes sc(il, l);
    faiss::InvertedLists::ScopedIds si(il, l);
    if (codes)
        memcpy(codes, sc.get(), n * il->code_size);
    if (ids)
        memcpy(ids, si.get(), n * sizeof(idx_t));
    REF_CATCH
}
// faiss/IndexIVF.cpp:401 search_preassigned
int ref_ivf_search_preassigned(
        void* idx,
        int64_t n,
        const float* x,
        int64_t k,
        const int64_t* assign,
        const float* centroid_dis,
        float* D,
        int64_t* I) {
    REF_TRY((faiss::IndexIVF*)idx)->search_preassigned(n, x, k, assign, centroid_dis, D, I, false);
    REF_CATCH
}
int ref_ivf_quantizer_search(void* idx, int64_t n, const float* x, int64_t k, float* D, int64_t* I) {
    REF_TRY((faiss::IndexIVF*)idx)->quantizer->search(n, x, k, D, I);
    REF_CATCH
}

// ---------------------------------------------------------------- IndexIVFFlat (faiss/IndexIVFFlat.h)
void* ref_ivfflat_new(int d, int64_t nlist, int metric) {
    auto mt = metric == 0 ? faiss::METRIC_INNER_PRODUCT : faiss::METRIC_L2;
    auto* q = new faiss::IndexFlat(d, mt);
    auto* idx = new faiss::IndexIVFFlat(q, d, nlist, mt);
    idx->own_fields = true;
    return idx;
}

// ---------------------------------------------------------------- IndexIVFPQ (faiss/IndexIVFPQ.h)
void* ref_ivfpq_new(int d, int64_t nlist, int M, int nbits, int metric) {
    auto mt = metric == 0 ? faiss::METRIC_INNER_PRODUCT : faiss::METRIC_L2;
    auto* q = new faiss::IndexFlat(d, mt);
    auto* idx = new faiss::IndexIVFPQ(q, d, nlist, M, nbits, mt);
    idx->own_fields = true;
    return idx;
}
int ref_ivfpq_use_precomputed_table(void* idx) {
    return ((faiss::IndexIVFPQ*)idx)->use_precomputed_table;
}
// faiss/IndexIVFPQ.cpp:375 precompute_table()
int ref_ivfpq_set_precomputed_table(void* idx, int v) {
    REF_TRY auto* p = (faiss::IndexIVFPQ*)idx;
    p->use_precomputed_table = v;
    p->precompute_table();
    REF_CATCH
}
// PQ centroids, layout [M][ksub][dsub] (faiss/impl/ProductQuantizer.h)
int ref_ivfpq_get_pq_centroids(void* idx, float* out) {
    REF_TRY auto* p = (faiss::IndexIVFPQ*)idx;
    memcpy(out, p->pq.centroids.data(), p->pq.centroids.size() * sizeof(float));
    REF_CATCH
}
int ref_ivfpq_set_pq_centroids(void* idx, const float* in) {
    REF_TRY auto* p = (faiss::IndexIVFPQ*)idx;
    memcpy(p->pq.centroids.data(), in, p->pq.centroids.size() * sizeof(float));
    p->is_trained = true;
    if (p->use_precomputed_table)
        p->precompute_table();
    REF_CATCH
}
void ref_ivfpq_set_pq_niter(void* idx, int niter, int seed) {
    auto* p = (faiss::IndexIVFPQ*)idx;
    if (niter > 0)
        p->pq.cp.niter = niter;
    if (seed >= 0)
        p->pq.cp.seed = seed;
}
// faiss/impl/ProductQuantizer.cpp compute_codes (no residual) -- used to pin the PQ encoder
int ref_pq_compute_codes(void* idx, const float* x, uint8_t* codes, int64_t n) {
    REF_TRY((faiss::IndexIVFPQ*)idx)->pq.compute_codes(x, codes, n);
    REF_CATCH
}

// InvertedLists::add_entries (faiss/invlists/InvertedLists.h) -- bulk list load: the GPU -> CPU direction
// of the cloner (index_gpu_to_cpu / GpuIndexIVFPQ::copyTo, faiss/gpu/GpuIndexIVFPQ.cu:160-217) so the CPU
// baseline searches exactly the codes the GPU index holds
int ref_ivf_add_entries(void* idx, int64_t l, int64_t n, const int64_t* ids, const uint8_t* codes) {
    REF_TRY auto* p = (faiss::IndexIVF*)idx;
    p->invlists->add_entries(l, n, ids, codes);
    p->ntotal += n;
    REF_CATCH
}
int ref_ivf_set_is_trained(void* idx, int v) {
    ((faiss::Index*)idx)->is_trained = v != 0;
    return 0;
}
int ref_ivf_set_parallel_mode(void* idx, int mode) {
    ((faiss::IndexIVF*)idx)->parallel_mode = mode;
    return 0;
}
// faiss/impl/ProductQuantizer.cpp:130-195 ProductQuantizer::train (Train_default: M independent k-means)
int ref_pq_train(int d, int M, int nbits, int64_t n, const float* x, int niter, int seed, float* centroids_out) {
    REF_TRY faiss::ProductQuantizer pq(d, M, nbits);
    if (niter > 0)
        pq.cp.niter = niter;
    if (seed >= 0)
        pq.cp.seed = seed;
    pq.train(n, x);
    memcpy(centroids_out, pq.centroids.data(), sizeof(float) * pq.centroids.size());
    REF_CATCH
}
// Clustering with spherical = true and an inner-product assignment index (what GpuIndexIVF does for
// METRIC_INNER_PRODUCT, faiss/gpu/GpuIndexIVF.cu:72-76; faiss/Clustering.cpp post_process_centroids)
int ref_kmeans_spherical_ip(int d, int64_t n, int64_t k, const float* x, int niter, int seed, float* centroids_out, float* obj_out) {
    REF_TRY faiss::ClusteringParameters cp;
    cp.niter = niter;
    cp.seed = seed;
    cp.spherical = true;
    faiss::Clustering clus(d, k, cp);
    faiss::IndexFlatIP index(d);
    clus.train(n, x, index);
    memcpy(centroids_out, clus.centroids.data(), sizeof(float) * d * k);
    for (size_t i = 0; i < clus.iteration_stats.size() && (int)i < niter; i++)
        if (obj_out)
            obj_out[i] = clus.iteration_stats[i].obj;
    REF_CATCH
}

// ---------------------------------------------------------------- Clustering (faiss/Clustering.cpp:60-380)
// Runs the reference Lloyd k-means with a CPU IndexFlatL2 as the assignment index.
// obj_out (size niter) receives ClusteringIterationStats.obj per iteration.
int ref_kmeans(
        int d,
        int64_t n,
        int64_t k,
        const float* x,
        int niter,
        int seed,
        int max_points_per_centroid,
        int min_points_per_centroid,
        float* centroids_out,
        float* obj_out,
        int64_t* nsplit_out) {
    REF_TRY faiss::ClusteringParameters cp;
    cp.niter = niter;
    cp.seed = seed;
    if (max_points_per_centroid > 0)
        cp.max_points_per_centroid = max_points_per_centroid;
    if (min_points_per_centroid >= 0)
        cp.min_points_per_centroid = min_points_per_centroid;
    faiss::Clustering clus(d, k, cp);
    faiss::IndexFlatL2 index(d);
    clus.train(n, x, index);
    memcpy(centroids_out, clus.centroids.data(), sizeof(float) * d * k);
    for (size_t i = 0; i < clus.iteration_stats.size() && (int)i < niter; i++) {
        if (obj_out)
            obj_out[i] = clus.iteration_stats[i].obj;
        if (nsplit_out)
            nsplit_out[i] = clus.iteration_stats[i].nsplit;
    }
    REF_CATCH
}

// ---------------------------------------------------------------- IndexShards (faiss/IndexShards.cpp:87-264)
void* ref_shards_new(int d, int threaded, int successive_ids) {
    return new faiss::IndexShards(d, threaded != 0, successive_ids != 0);
}
int ref_shards_add_shard(void* sh, void* idx) {
    REF_TRY((faiss::IndexShards*)sh)->add_shard((faiss::Index*)idx);
    REF_CATCH
}

// faiss/utils/Heap.cpp:166-238 merge_knn_results (CMin = L2 / ascending, CMax = IP / descending)
int ref_merge_knn_results(
        int64_t n,
        int64_t k,
        int nshard,
        int metric,
        const float* all_D,
        const int64_t* all_I,
        float* D,
        int64_t* I) {
    REF_TRY if (metric == 1) {
        faiss::merge_knn_results<idx_t, faiss::CMin<float, int>>(n, k, nshard, all_D, all_I, D, I);
    }
    else {
        faiss::merge_knn_results<idx_t, faiss::CMax<float, int>>(n, k, nshard, all_D, all_I, D, I);
    }
    REF_CATCH
}

// faiss/utils/distances.cpp:834 knn_L2sqr / :768 knn_inner_product, raw entry points
int ref_knn(int metric, const float* x, const float* y, int64_t d, int64_t nx, int64_t ny, int64_t k, float* D, int64_t* I) {
    REF_TRY if (metric == 1) faiss::knn_L2sqr(x, y, d, nx, ny, k, D, I);
    else faiss::knn_inner_product(x, y, d, nx, ny, k, D, I);
    REF_CATCH
}

} // extern "C"
