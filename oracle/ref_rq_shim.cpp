// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's ResidualQuantizer encoding, compiled by oracle/Makefile into
// oracle/_ref/libfaiss_ref_rq.so against the UNMODIFIED reference CPU library (oracle/_ref/libfaiss_ref.so).  Every
// call forwards to a reference entry point; ref_rq_refine_beam_lut first makes (query_norms, query_cp) with the calls
// compute_codes_add_centroids_mp_lut1 makes (faiss/impl/residual_quantizer_encode_steps.cpp:752-772).  The product
// (faiss_b200/) never loads this file.

#include <faiss/impl/ResidualQuantizer.h>
#include <faiss/utils/distances.h>

#include <cstring>
#include <vector>

#include "ref_shim.h"

extern "C" int sgemm_(
        const char* transa, const char* transb, int* m, int* n, int* k, const float* alpha, const float* a, int* lda,
        const float* b, int* ldb, float* beta, float* c, int* ldc);

using faiss::ResidualQuantizer;

extern "C" {

// a ResidualQuantizer(d, nbits[M]) with the given search type; with codebooks [total_K][d] it is marked trained and
// its codebook tables are computed (AdditiveQuantizer::compute_codebook_tables)
void* ref_rq_new(int d, int M, const int* nbits, int search_type, const float* codebooks) {
    REF_TRY std::vector<size_t> nb(nbits, nbits + M);
    auto* q = new ResidualQuantizer(d, nb, (faiss::AdditiveQuantizer::Search_type_t)search_type);
    if (codebooks) {
        q->codebooks.assign(codebooks, codebooks + q->total_codebook_size * d);
        q->is_trained = true;
        q->compute_codebook_tables();
    }
    return q;
    REF_CATCH_RET(nullptr)
}

void ref_rq_free(void* h) {
    delete (ResidualQuantizer*)h;
}

// max_beam_size, use_beam_LUT, norm_min, norm_max
int ref_rq_set_params(void* h, int max_beam_size, int use_beam_LUT, float norm_min, float norm_max) {
    REF_TRY auto* q = (ResidualQuantizer*)h;
    q->max_beam_size = max_beam_size;
    q->use_beam_LUT = use_beam_LUT;
    q->norm_min = norm_min;
    q->norm_max = norm_max;
    REF_CATCH
}

int64_t ref_rq_code_size(void* h) {
    return (int64_t)((ResidualQuantizer*)h)->code_size;
}

// ResidualQuantizer::train with train_type, max_beam_size and niter; the codebooks are read with ref_rq_tables
int ref_rq_train(void* h, int64_t n, const float* x, int train_type, int max_beam_size, int niter) {
    REF_TRY auto* q = (ResidualQuantizer*)h;
    q->train_type = train_type;
    q->max_beam_size = max_beam_size;
    q->cp.niter = niter;
    q->train(n, x);
    REF_CATCH
}

// codebooks [total_K][d], centroid_norms [total_K], codebook_cross_products (ref_rq_cross_size floats); each may be NULL
int ref_rq_tables(void* h, float* codebooks, float* norms, float* cross) {
    REF_TRY auto* q = (ResidualQuantizer*)h;
    if (codebooks)
        std::memcpy(codebooks, q->codebooks.data(), sizeof(float) * q->codebooks.size());
    if (norms)
        std::memcpy(norms, q->centroid_norms.data(), sizeof(float) * q->centroid_norms.size());
    if (cross)
        std::memcpy(cross, q->codebook_cross_products.data(), sizeof(float) * q->codebook_cross_products.size());
    REF_CATCH
}

int64_t ref_rq_cross_size(void* h) {
    return (int64_t)((ResidualQuantizer*)h)->codebook_cross_products.size();
}

// ResidualQuantizer::refine_beam
int ref_rq_refine_beam(
        void* h, int64_t n, int64_t beam_size, const float* residuals, int out_beam, int32_t* codes, float* residuals_out,
        float* distances) {
    REF_TRY((ResidualQuantizer*)h)->refine_beam(n, beam_size, residuals, out_beam, codes, residuals_out, distances);
    REF_CATCH
}

// ResidualQuantizer::refine_beam_LUT on the CPU's own query_norms (fvec_norms_L2sqr) and query_cp (the sgemm x·Cᵀ)
int ref_rq_refine_beam_lut(void* h, int64_t n, const float* x, int out_beam, int32_t* codes, float* distances) {
    REF_TRY auto* q = (ResidualQuantizer*)h;
    std::vector<float> norms(n), cp(n * q->total_codebook_size);
    faiss::fvec_norms_L2sqr(norms.data(), x, q->d, n);
    int ti = q->total_codebook_size, di = q->d, ni = n;
    float zero = 0, one = 1;
    sgemm_("Transposed", "Not transposed", &ti, &ni, &di, &one, q->codebooks.data(), &di, x, &di, &zero, cp.data(), &ti);
    q->refine_beam_LUT(n, norms.data(), cp.data(), out_beam, codes, distances);
    REF_CATCH
}

// ResidualQuantizer::compute_codes_add_centroids (centroids may be NULL) -> packed [n][code_size]
int ref_rq_compute_codes(void* h, const float* x, int64_t n, const float* centroids, uint8_t* packed) {
    REF_TRY((ResidualQuantizer*)h)->compute_codes_add_centroids(x, packed, n, centroids);
    REF_CATCH
}

// AdditiveQuantizer::decode
int ref_rq_decode(void* h, const uint8_t* packed, int64_t n, float* x) {
    REF_TRY((ResidualQuantizer*)h)->decode(packed, x, n);
    REF_CATCH
}

} // extern "C"
