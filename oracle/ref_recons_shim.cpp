// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's IndexIVF retrieval calls, compiled by oracle/Makefile into
// oracle/_ref/libfaiss_ref_recons.so against the UNMODIFIED reference CPU library (oracle/_ref/libfaiss_ref.so).
// Every function forwards to a reference entry point; the handles are the IndexIVF objects of ref_shim.cpp /
// ref_sq_shim.cpp.  The product (faiss_b200/) never loads this file.

#include <faiss/IndexIVF.h>

#include "ref_shim.h"

extern "C" {

// IndexIVF::search_and_reconstruct (faiss/IndexIVF.cpp:1128-1181) with SearchParametersIVF::nprobe
int ref_ivf_search_and_reconstruct(void* idx, int64_t n, const float* x, int64_t k, int64_t nprobe, float* D, int64_t* I, float* R) {
    REF_TRY faiss::SearchParametersIVF p;
    p.nprobe = (size_t)nprobe;
    ((faiss::IndexIVF*)idx)->search_and_reconstruct(n, x, k, D, I, R, &p);
    REF_CATCH
}

// IndexIVF::search_and_return_codes (faiss/IndexIVF.cpp:1183-1248)
int ref_ivf_search_and_return_codes(
        void* idx, int64_t n, const float* x, int64_t k, int64_t nprobe, float* D, int64_t* I, uint8_t* codes, int include_listno) {
    REF_TRY faiss::SearchParametersIVF p;
    p.nprobe = (size_t)nprobe;
    ((faiss::IndexIVF*)idx)->search_and_return_codes(n, x, k, D, I, codes, include_listno != 0, &p);
    REF_CATCH
}

int64_t ref_ivf_coarse_code_size(void* idx) {
    return (int64_t)((faiss::IndexIVF*)idx)->coarse_code_size();
}

// IndexIVF::set_direct_map_type(Hashtable) (make_direct_map's array map needs ids 0 .. ntotal-1; the hash map takes
// any unique ids), then IndexIVF::reconstruct per key
int ref_ivf_reconstruct_keys(void* idx, int64_t n, const int64_t* keys, float* out) {
    REF_TRY auto* ivf = (faiss::IndexIVF*)idx;
    ivf->set_direct_map_type(faiss::DirectMap::Hashtable);
    for (int64_t i = 0; i < n; i++)
        ivf->reconstruct(keys[i], out + i * ivf->d);
    REF_CATCH
}

} // extern "C"
