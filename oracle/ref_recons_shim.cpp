// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's IndexIVF retrieval calls, compiled by oracle/recons.mk into
// oracle/_ref/libfaiss_ref_recons.so against the UNMODIFIED reference CPU library (oracle/_ref/libfaiss_ref.so).
// Every function forwards to a reference entry point; the handles are the IndexIVF objects of ref_shim.cpp /
// ref_sq_shim.cpp.  The product (faiss_b200/) never loads this file.

#include <faiss/IndexIVF.h>

#include <string>

static thread_local std::string g_recons_err;

#define RC_TRY try {
#define RC_CATCH                      \
    }                                 \
    catch (const std::exception& e) { \
        g_recons_err = e.what();      \
        return -1;                    \
    }                                 \
    return 0;

extern "C" {

const char* ref_recons_last_error() {
    return g_recons_err.c_str();
}

// IndexIVF::search_and_reconstruct (faiss/IndexIVF.cpp:1128-1181) with SearchParametersIVF::nprobe
int ref_ivf_search_and_reconstruct(void* idx, int64_t n, const float* x, int64_t k, int64_t nprobe, float* D, int64_t* I, float* R) {
    RC_TRY faiss::SearchParametersIVF p;
    p.nprobe = (size_t)nprobe;
    ((faiss::IndexIVF*)idx)->search_and_reconstruct(n, x, k, D, I, R, &p);
    RC_CATCH
}

// IndexIVF::search_and_return_codes (faiss/IndexIVF.cpp:1183-1248)
int ref_ivf_search_and_return_codes(
        void* idx, int64_t n, const float* x, int64_t k, int64_t nprobe, float* D, int64_t* I, uint8_t* codes, int include_listno) {
    RC_TRY faiss::SearchParametersIVF p;
    p.nprobe = (size_t)nprobe;
    ((faiss::IndexIVF*)idx)->search_and_return_codes(n, x, k, D, I, codes, include_listno != 0, &p);
    RC_CATCH
}

int64_t ref_ivf_coarse_code_size(void* idx) {
    return (int64_t)((faiss::IndexIVF*)idx)->coarse_code_size();
}

// IndexIVF::set_direct_map_type(Hashtable) (make_direct_map's array map needs ids 0 .. ntotal-1; the hash map takes
// any unique ids), then IndexIVF::reconstruct per key
int ref_ivf_reconstruct_keys(void* idx, int64_t n, const int64_t* keys, float* out) {
    RC_TRY auto* ivf = (faiss::IndexIVF*)idx;
    ivf->set_direct_map_type(faiss::DirectMap::Hashtable);
    for (int64_t i = 0; i < n; i++)
        ivf->reconstruct(keys[i], out + i * ivf->d);
    RC_CATCH
}

} // extern "C"
