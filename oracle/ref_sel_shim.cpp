// TEST INFRASTRUCTURE ONLY.
//
// extern "C" entry points for the reference's IDSelectors and for a search with SearchParameters::sel, built by
// oracle/Makefile into oracle/_ref/libfaiss_ref_sel.so against the UNMODIFIED reference CPU library of
// oracle/Makefile.  The index handles are the reference faiss::Index objects of oracle/ref.py, ref_pq.py and
// ref_sq.py (IndexFlat, IndexIVFFlat, IndexIVFPQ, IndexIVFScalarQuantizer).  Array and Bitmap selectors keep
// the caller's pointer, as the reference's do: the caller keeps those arrays alive.  The product (faiss_b200/)
// never loads this file.

#include <faiss/Index.h>
#include <faiss/IndexIVF.h>
#include <faiss/impl/FaissException.h>
#include <faiss/impl/IDSelector.h>

#include "ref_shim.h"

extern "C" {

void* ref_sel_range(int64_t imin, int64_t imax) {
    return new faiss::IDSelectorRange(imin, imax);
}
void* ref_sel_array(int64_t n, const int64_t* ids) {
    return new faiss::IDSelectorArray((size_t)n, ids);
}
void* ref_sel_batch(int64_t n, const int64_t* ids) {
    return new faiss::IDSelectorBatch((size_t)n, ids);
}
void* ref_sel_bitmap(int64_t n, const uint8_t* bitmap) {
    return new faiss::IDSelectorBitmap((size_t)n, bitmap);
}
void* ref_sel_not(void* s) {
    return new faiss::IDSelectorNot((const faiss::IDSelector*)s);
}
// op: 0 = And, 1 = Or, 2 = XOr
void* ref_sel_binary(int op, void* a, void* b) {
    auto* l = (const faiss::IDSelector*)a;
    auto* r = (const faiss::IDSelector*)b;
    if (op == 0)
        return new faiss::IDSelectorAnd(l, r);
    if (op == 1)
        return new faiss::IDSelectorOr(l, r);
    return new faiss::IDSelectorXOr(l, r);
}
void ref_sel_free(void* s) {
    delete (faiss::IDSelector*)s;
}
int ref_sel_is_member(void* s, int64_t id) {
    return ((const faiss::IDSelector*)s)->is_member(id) ? 1 : 0;
}

// faiss::Index::search(n, x, k, D, I, params) with params->sel = sel; nprobe > 0: SearchParametersIVF with that
// nprobe (faiss/IndexIVF.cpp search), else plain SearchParameters
int ref_search_sel(void* idx, int64_t n, const float* x, int64_t k, void* sel, int64_t nprobe, float* D, int64_t* I) {
    REF_TRY auto* index = (faiss::Index*)idx;
    if (nprobe > 0) {
        faiss::SearchParametersIVF p;
        p.sel = (faiss::IDSelector*)sel;
        p.nprobe = (size_t)nprobe;
        index->search(n, x, k, D, I, &p);
    } else {
        faiss::SearchParameters p;
        p.sel = (faiss::IDSelector*)sel;
        index->search(n, x, k, D, I, &p);
    }
    REF_CATCH
}

} // extern "C"
