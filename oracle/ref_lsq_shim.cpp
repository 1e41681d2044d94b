// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's LocalSearchQuantizer encoding, compiled by oracle/lsq.mk into
// oracle/_ref/libfaiss_ref_lsq.so against the UNMODIFIED reference CPU library (oracle/_ref/libfaiss_ref.so).
// Every encode forwards to a reference entry point; ref_lsq_draws makes the perturbation draws with the same
// std::mt19937 and std::uniform_int_distribution calls, in the same order, as LocalSearchQuantizer::perturb_codes
// (faiss/impl/LocalSearchQuantizer.cpp:673-688), so a device encoder can be fed the CPU's exact draws.  The product
// (faiss_b200/) never loads this file.

#include <faiss/impl/LocalSearchQuantizer.h>
#include <faiss/utils/hamming.h>

#include <omp.h>

#include <cstring>
#include <random>
#include <string>
#include <vector>

static thread_local std::string g_lsq_err;

#define LQ_TRY try {
#define LQ_CATCH                      \
    }                                 \
    catch (const std::exception& e) { \
        g_lsq_err = e.what();         \
        return -1;                    \
    }                                 \
    return 0;

using faiss::LocalSearchQuantizer;

extern "C" {

const char* ref_lsq_last_error() {
    return g_lsq_err.c_str();
}

// a LocalSearchQuantizer(d, M, nbits) with the given codebooks [M][K][d] and encoding parameters, marked trained
void* ref_lsq_new(int d, int M, int nbits, const float* codebooks, int nperts, int icm_iters, int encode_ils_iters, int random_seed) {
    try {
        auto* q = new LocalSearchQuantizer(d, M, nbits);
        q->codebooks.assign(codebooks, codebooks + (size_t)M * q->K * d);
        q->nperts = nperts;
        q->icm_iters = icm_iters;
        q->encode_ils_iters = encode_ils_iters;
        q->random_seed = random_seed;
        q->is_trained = true;
        return q;
    } catch (const std::exception& e) {
        g_lsq_err = e.what();
        return nullptr;
    }
}

// the OpenMP thread count of the CPU encoder
void ref_lsq_set_threads(int n) {
    omp_set_num_threads(n);
}

void ref_lsq_free(void* h) {
    delete (LocalSearchQuantizer*)h;
}

// LocalSearchQuantizer::compute_codes (faiss/impl/LocalSearchQuantizer.cpp:294-321: codes drawn from
// mt19937(random_seed), icm_encode in chunks of chunk_size, packed), unpacked to int32 [n][M]
int ref_lsq_compute_codes(void* h, const float* x, int64_t n, int32_t* codes) {
    LQ_TRY auto* q = (LocalSearchQuantizer*)h;
    std::vector<uint8_t> packed(q->code_size * n);
    q->compute_codes(x, packed.data(), n);
    for (int64_t i = 0; i < n; i++) {
        faiss::BitstringReader br(packed.data() + i * q->code_size, q->code_size);
        for (size_t m = 0; m < q->M; m++)
            codes[i * q->M + m] = (int32_t)br.read(q->nbits[m]);
    }
    LQ_CATCH
}

// lsq::IcmEncoder::encode (faiss/impl/LocalSearchQuantizer.cpp:812-819) on codes [n][M] in place, one chunk, with
// std::mt19937(seed); *next = the generator's next output after the call
int ref_lsq_icm_encode(void* h, int32_t* codes, const float* x, int64_t n, int64_t ils_iters, uint32_t seed, uint32_t* next) {
    LQ_TRY auto* q = (LocalSearchQuantizer*)h;
    faiss::lsq::IcmEncoder enc(q);
    enc.set_binary_term();
    std::mt19937 gen(seed);
    enc.encode(codes, x, gen, n, ils_iters);
    *next = (uint32_t)gen();
    LQ_CATCH
}

// the draws of LocalSearchQuantizer::perturb_codes for ils_iters iterations over n rows, from std::mt19937(seed)
// after `skip` outputs: out [ils_iters][n][nperts][2] = (m, k); *next = the generator's next output afterwards
int ref_lsq_draws(int64_t M, int64_t K, int64_t nperts, int64_t n, int64_t ils_iters, uint32_t seed, int64_t skip, int32_t* out, uint32_t* next) {
    LQ_TRY std::mt19937 gen(seed);
    gen.discard(skip);
    std::uniform_int_distribution<size_t> m_distrib(0, M - 1);
    std::uniform_int_distribution<int32_t> k_distrib(0, K - 1);
    int32_t* o = out;
    for (int64_t it = 0; it < ils_iters; it++) {
        for (int64_t i = 0; i < n; i++) {
            for (int64_t j = 0; j < nperts; j++) {
                o[0] = (int32_t)m_distrib(gen);
                o[1] = k_distrib(gen);
                o += 2;
            }
        }
    }
    *next = (uint32_t)gen();
    LQ_CATCH
}

} // extern "C"
