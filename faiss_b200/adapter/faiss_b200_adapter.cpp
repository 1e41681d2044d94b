// faiss_b200 adapter implementation.  See faiss_b200_adapter.h.
#include "faiss_b200_adapter.h"

#include <faiss/impl/FaissAssert.h>
#include <faiss/impl/IDSelector.h>
#include <faiss/invlists/InvertedLists.h>

#include <cstring>
#include <vector>

// the C ABI declares its own global `idx_t` and FaissMetricType enumerators; keep them out of namespace faiss
#include "faiss_b200_c.h"

namespace faiss_b200_adapter {

namespace {
void ck(int rc) {
    if (rc != 0)
        FAISS_THROW_FMT("faiss_b200: %s", faiss_get_last_error());
}
::FaissMetricType mt(faiss::MetricType m) {
    FAISS_THROW_IF_NOT_MSG(m == faiss::METRIC_L2 || m == faiss::METRIC_INNER_PRODUCT, "faiss_b200 supports METRIC_L2 and METRIC_INNER_PRODUCT");
    return m == faiss::METRIC_L2 ? ::METRIC_L2 : ::METRIC_INNER_PRODUCT;
}
int selectorIsMember(void* ctx, ::idx_t id) {
    return static_cast<const faiss::IDSelector*>(ctx)->is_member(id) ? 1 : 0;
}

// a faiss::IDSelector as the library's selector tree: the reference's Range / Array / Batch / Bitmap / Not / And /
// Or / XOr by their contents (their is_member is final, so a subclass cannot change it), any other subclass
// (IDSelectorAll, IDSelectorTranslated, a user class) as a callback
struct SelectorHandles {
    std::vector<FaissIDSelector*> owned;
    ~SelectorHandles() {
        for (auto* h : owned)
            faiss_IDSelector_free(h);
    }
    FaissIDSelector* convert(const faiss::IDSelector* s) {
        FaissIDSelector* h = nullptr;
        if (auto* r = dynamic_cast<const faiss::IDSelectorRange*>(s)) {
            ck(faiss_IDSelectorRange_new(&h, r->imin, r->imax));
        } else if (auto* a = dynamic_cast<const faiss::IDSelectorArray*>(s)) {
            ck(faiss_IDSelectorArray_new(&h, a->n, a->ids));
        } else if (auto* b = dynamic_cast<const faiss::IDSelectorBatch*>(s)) {
            std::vector<::idx_t> ids(b->set.begin(), b->set.end());
            ck(faiss_IDSelectorBatch_new(&h, ids.size(), ids.data()));
        } else if (auto* bm = dynamic_cast<const faiss::IDSelectorBitmap*>(s)) {
            ck(faiss_IDSelectorBitmap_new(&h, bm->n, bm->bitmap));
        } else if (auto* n = dynamic_cast<const faiss::IDSelectorNot*>(s)) {
            FaissIDSelector* c = convert(n->sel);
            ck(faiss_IDSelectorNot_new(&h, c));
        } else if (auto* x = dynamic_cast<const faiss::IDSelectorAnd*>(s)) {
            FaissIDSelector* l = convert(x->lhs);
            ck(faiss_IDSelectorAnd_new(&h, l, convert(x->rhs)));
        } else if (auto* x = dynamic_cast<const faiss::IDSelectorOr*>(s)) {
            FaissIDSelector* l = convert(x->lhs);
            ck(faiss_IDSelectorOr_new(&h, l, convert(x->rhs)));
        } else if (auto* x = dynamic_cast<const faiss::IDSelectorXOr*>(s)) {
            FaissIDSelector* l = convert(x->lhs);
            ck(faiss_IDSelectorXOr_new(&h, l, convert(x->rhs)));
        } else {
            ck(faiss_b200_IDSelectorCallback_new(&h, selectorIsMember, const_cast<faiss::IDSelector*>(s)));
        }
        owned.push_back(h);
        return h;
    }
};
} // namespace

B200Resources::B200Resources() {
    ck(faiss_StandardGpuResources_new(&h_));
}
B200Resources::~B200Resources() {
    if (h_)
        faiss_StandardGpuResources_free(h_);
}
void B200Resources::ncclInitAll(const std::vector<int>& devices) {
    ck(faiss_StandardGpuResources_ncclInitAll(h_, (int)devices.size(), devices.data()));
}

// ---------------------------------------------------------------- B200Index
B200Index::~B200Index() {
    if (h_)
        faiss_Index_free(h_);
}
void B200Index::sync_() {
    ntotal = faiss_Index_ntotal(h_);
    is_trained = faiss_Index_is_trained(h_) != 0;
}
void B200Index::train(faiss::idx_t n, const float* x) {
    ck(faiss_Index_train(h_, n, x));
    sync_();
}
void B200Index::add(faiss::idx_t n, const float* x) {
    ck(faiss_Index_add(h_, n, x));
    sync_();
}
void B200Index::add_with_ids(faiss::idx_t n, const float* x, const faiss::idx_t* xids) {
    ck(faiss_Index_add_with_ids(h_, n, x, xids));
    sync_();
}
void B200Index::search(
        faiss::idx_t n, const float* x, faiss::idx_t k, float* distances, faiss::idx_t* labels, const faiss::SearchParameters* params) const {
    if (!params || !params->sel) {
        ck(faiss_Index_search(h_, n, x, k, distances, labels));
        return;
    }
    SelectorHandles sel;
    FaissSearchParameters* sp = nullptr;
    ck(faiss_SearchParameters_new(&sp, sel.convert(params->sel)));
    int rc = faiss_Index_search_with_params(h_, n, x, k, sp, distances, labels);
    faiss_SearchParameters_free(sp);
    ck(rc);
}
void B200Index::search_and_reconstruct(
        faiss::idx_t n, const float* x, faiss::idx_t k, float* distances, faiss::idx_t* labels, float* recons,
        const faiss::SearchParameters* params) const {
    if (!params || !params->sel) {
        ck(faiss_Index_search_and_reconstruct(h_, n, x, k, nullptr, distances, labels, recons));
        return;
    }
    SelectorHandles sel;
    FaissSearchParameters* sp = nullptr;
    ck(faiss_SearchParameters_new(&sp, sel.convert(params->sel)));
    int rc = faiss_Index_search_and_reconstruct(h_, n, x, k, sp, distances, labels, recons);
    faiss_SearchParameters_free(sp);
    ck(rc);
}
void B200Index::reconstruct_batch(faiss::idx_t n, const faiss::idx_t* keys, float* recons) const {
    ck(faiss_Index_reconstruct_batch(h_, n, keys, recons));
}
void B200Index::reset() {
    ck(faiss_Index_reset(h_));
    sync_();
}
void B200Index::reconstruct(faiss::idx_t key, float* recons) const {
    ck(faiss_Index_reconstruct(h_, key, recons));
}
void B200Index::reconstruct_n(faiss::idx_t i0, faiss::idx_t ni, float* recons) const {
    ck(faiss_Index_reconstruct_n(h_, i0, ni, recons));
}

// ---------------------------------------------------------------- Flat
B200IndexFlat::B200IndexFlat(B200Resources* res, int dims, faiss::MetricType metric, int device, bool useFloat16)
        : B200Index(dims, metric, device) {
    ck(faiss_GpuIndexFlat_new_with_config(&h_, res->handle(), dims, mt(metric), device, 1, useFloat16 ? 1 : 0));
    sync_();
}
B200IndexFlat::B200IndexFlat(B200Resources* res, const faiss::IndexFlat* index, int device, bool useFloat16)
        : B200IndexFlat(res, index->d, index->metric_type, device, useFloat16) {
    copyFrom(index);
}
void B200IndexFlat::copyFrom(const faiss::IndexFlat* index) { // faiss/gpu/GpuIndexFlat.cu:105-140
    FAISS_THROW_IF_NOT(index->d == d && index->metric_type == metric_type);
    ck(faiss_GpuIndexFlat_copyFrom(h_, index->ntotal, index->get_xb()));
    sync_();
}
void B200IndexFlat::copyTo(faiss::IndexFlat* index) const { // faiss/gpu/GpuIndexFlat.cu:142-176
    index->reset();
    index->d = d;
    index->metric_type = metric_type;
    index->code_size = sizeof(float) * d;
    std::vector<float> xb((size_t)ntotal * d);
    if (ntotal > 0) {
        ck(faiss_GpuIndexFlat_copyTo(h_, xb.data()));
        index->add(ntotal, xb.data());
    }
}

// ---------------------------------------------------------------- IVF
// search (recons == null) or search_and_reconstruct with the index's nprobe or the SearchParametersIVF's
void B200IndexIVF::search_(
        faiss::idx_t n, const float* x, faiss::idx_t k, float* distances, faiss::idx_t* labels, float* recons,
        const faiss::SearchParameters* params) const {
    size_t use_nprobe = nprobe;
    size_t max_codes = 0;
    SelectorHandles sel;
    FaissIDSelector* selHandle = nullptr;
    if (params) {
        if (params->sel)
            selHandle = sel.convert(params->sel);
        auto* ivf = dynamic_cast<const faiss::SearchParametersIVF*>(params);
        FAISS_THROW_IF_NOT_MSG(ivf, "IVF search: search parameters must be SearchParametersIVF");
        use_nprobe = ivf->nprobe;
        max_codes = ivf->max_codes;
    }
    FaissSearchParametersIVF* sp = nullptr;
    ck(faiss_SearchParametersIVF_new_with_sel(&sp, selHandle, use_nprobe, max_codes));
    int rc = recons ? faiss_Index_search_and_reconstruct(h_, n, x, k, sp, distances, labels, recons)
                    : faiss_Index_search_with_params(h_, n, x, k, sp, distances, labels);
    faiss_SearchParameters_free(sp);
    ck(rc);
}
void B200IndexIVF::search(
        faiss::idx_t n, const float* x, faiss::idx_t k, float* distances, faiss::idx_t* labels, const faiss::SearchParameters* params) const {
    search_(n, x, k, distances, labels, nullptr, params);
}
void B200IndexIVF::search_and_reconstruct(
        faiss::idx_t n, const float* x, faiss::idx_t k, float* distances, faiss::idx_t* labels, float* recons,
        const faiss::SearchParameters* params) const {
    search_(n, x, k, distances, labels, recons, params);
}

void B200IndexIVF::copyListsFrom_(const faiss::IndexIVF* index) {
    // IVFBase::copyInvertedListsFrom (faiss/gpu/impl/IVFBase.cu:328-451): centroids, then every list verbatim
    FAISS_THROW_IF_NOT(index->nlist == nlist && index->d == d);
    std::vector<float> cent((size_t)nlist * d);
    index->quantizer->reconstruct_n(0, nlist, cent.data());
    ck(faiss_Index_reset(h_));
    ck(faiss_GpuIndexIVF_setCoarseCentroids(h_, cent.data()));
    const faiss::InvertedLists* il = index->invlists;
    std::vector<::idx_t> lens(nlist);
    for (size_t l = 0; l < nlist; l++)
        lens[l] = il ? (::idx_t)il->list_size(l) : 0;
    ck(faiss_GpuIndexIVF_setListSizes(h_, lens.data())); // one arena relayout for the whole clone
    for (size_t l = 0; l < nlist && il; l++) {
        if (lens[l] == 0)
            continue;
        faiss::InvertedLists::ScopedCodes codes(il, l);
        faiss::InvertedLists::ScopedIds ids(il, l);
        ck(faiss_GpuIndexIVF_setList(h_, l, lens[l], codes.get(), ids.get()));
    }
    ck(faiss_GpuIndexIVF_set_is_trained(h_, index->is_trained ? 1 : 0));
    nprobe = index->nprobe;
    ck(faiss_GpuIndexIVF_set_nprobe(h_, nprobe));
    sync_();
}

void B200IndexIVF::copyListsTo_(faiss::IndexIVF* index) const {
    // IVFBase::copyInvertedListsTo: the lists come back in the ArrayInvertedLists byte format
    FAISS_THROW_IF_NOT(index->nlist == nlist);
    index->invlists->reset();
    index->ntotal = 0;
    const size_t cs = index->invlists->code_size;
    for (size_t l = 0; l < nlist; l++) {
        const size_t n = faiss_GpuIndexIVF_get_list_size(h_, l);
        if (n == 0)
            continue;
        std::vector<uint8_t> codes(n * cs);
        std::vector<faiss::idx_t> ids(n);
        ck(faiss_GpuIndexIVF_getListVectorData(h_, l, codes.data()));
        ck(faiss_GpuIndexIVF_getListIndices(h_, l, ids.data()));
        index->invlists->add_entries(l, n, ids.data(), codes.data());
        index->ntotal += n;
    }
    index->nprobe = nprobe;
}

B200IndexIVFFlat::B200IndexIVFFlat(B200Resources* res, int dims, size_t nlist_, faiss::MetricType metric, int device)
        : B200IndexIVF(dims, metric, nlist_, device) {
    ck(faiss_GpuIndexIVFFlat_new(&h_, res->handle(), dims, (::idx_t)nlist_, mt(metric), device));
    sync_();
}
B200IndexIVFFlat::B200IndexIVFFlat(B200Resources* res, const faiss::IndexIVFFlat* index, int device)
        : B200IndexIVFFlat(res, index->d, index->nlist, index->metric_type, device) {
    copyFrom(index);
}
void B200IndexIVFFlat::copyFrom(const faiss::IndexIVFFlat* index) {
    copyListsFrom_(index);
}
void B200IndexIVFFlat::copyTo(faiss::IndexIVFFlat* index) const { // faiss/gpu/GpuIndexIVFFlat.cu:127-150
    FAISS_THROW_IF_NOT(index->d == d && index->nlist == nlist);
    std::vector<float> cent((size_t)nlist * d);
    ck(faiss_GpuIndexIVF_getCoarseCentroids(h_, cent.data()));
    index->quantizer->reset();
    index->quantizer->add(nlist, cent.data());
    index->is_trained = is_trained;
    copyListsTo_(index);
}

B200IndexIVFPQ::B200IndexIVFPQ(B200Resources* res, int dims, size_t nlist_, size_t M_, size_t nbits_, faiss::MetricType metric, int device)
        : B200IndexIVF(dims, metric, nlist_, device), M(M_), nbits(nbits_) {
    ck(faiss_GpuIndexIVFPQ_new(&h_, res->handle(), dims, (::idx_t)nlist_, (::idx_t)M_, (::idx_t)nbits_, mt(metric), device));
    sync_();
}
B200IndexIVFPQ::B200IndexIVFPQ(B200Resources* res, const faiss::IndexIVFPQ* index, int device)
        : B200IndexIVFPQ(res, index->d, index->nlist, index->pq.M, index->pq.nbits, index->metric_type, device) {
    copyFrom(index);
}
void B200IndexIVFPQ::copyFrom(const faiss::IndexIVFPQ* index) { // faiss/gpu/GpuIndexIVFPQ.cu:105-158
    FAISS_THROW_IF_NOT(index->pq.M == M && index->pq.nbits == nbits);
    FAISS_THROW_IF_NOT_MSG(index->by_residual, "faiss_b200: only by_residual IVFPQ indexes are supported (as the reference GPU index)");
    copyListsFrom_(index);
    if (index->is_trained)
        ck(faiss_GpuIndexIVFPQ_setPQCentroids(h_, index->pq.centroids.data()));
    ck(faiss_GpuIndexIVF_set_is_trained(h_, index->is_trained ? 1 : 0));
    sync_();
}
void B200IndexIVFPQ::copyTo(faiss::IndexIVFPQ* index) const { // faiss/gpu/GpuIndexIVFPQ.cu:160-217
    FAISS_THROW_IF_NOT(index->d == d && index->nlist == nlist && index->pq.M == M && index->pq.nbits == nbits);
    std::vector<float> cent((size_t)nlist * d);
    ck(faiss_GpuIndexIVF_getCoarseCentroids(h_, cent.data()));
    index->quantizer->reset();
    index->quantizer->add(nlist, cent.data());
    if (is_trained)
        ck(faiss_GpuIndexIVFPQ_getPQCentroids(h_, index->pq.centroids.data()));
    index->is_trained = is_trained;
    index->by_residual = true;
    copyListsTo_(index);
    index->use_precomputed_table = 0;
    if (is_trained)
        index->precompute_table(); // the reference's auto rule
}

// ---------------------------------------------------------------- cloner
// ------------------------------------------------------------------------------------------
// B200IcmEncoder
// ------------------------------------------------------------------------------------------
B200IcmEncoder::B200IcmEncoder(
        const faiss::LocalSearchQuantizer* lsq_in,
        const std::vector<B200Resources*>& res,
        const std::vector<int>& devices)
        : faiss::lsq::IcmEncoder(lsq_in) {
    FAISS_THROW_IF_NOT_MSG(res.size() == devices.size() && !res.empty(), "one B200Resources per device");
    std::vector<FaissStandardGpuResources*> hs;
    for (auto* r : res)
        hs.push_back(r->handle());
    ck(faiss_GpuIcmEncoder_new(&h_, (int)lsq->M, (int)lsq->K, (int)lsq->d, (int)devices.size(), hs.data(), devices.data()));
}

B200IcmEncoder::~B200IcmEncoder() {
    if (h_)
        faiss_GpuIcmEncoder_free(h_);
}

void B200IcmEncoder::set_binary_term() {
    ck(faiss_GpuIcmEncoder_set_binary_term(h_, lsq->codebooks.data()));
}

void B200IcmEncoder::encode(int32_t* codes, const float* x, std::mt19937& gen, size_t n, size_t ils_iters) const {
    const size_t M = lsq->M, K = lsq->K, nperts = lsq->nperts;
    FAISS_THROW_IF_NOT(nperts <= M); // as icm_encode_impl, before any draw
    // LocalSearchQuantizer::perturb_codes (faiss/impl/LocalSearchQuantizer.cpp:673-688), once per ILS iteration
    std::uniform_int_distribution<size_t> m_distrib(0, M - 1);
    std::uniform_int_distribution<int32_t> k_distrib(0, K - 1);
    std::vector<int32_t> perts(ils_iters * n * nperts * 2);
    int32_t* p = perts.data();
    for (size_t it = 0; it < ils_iters; it++) {
        for (size_t i = 0; i < n; i++) {
            for (size_t j = 0; j < nperts; j++) {
                p[0] = (int32_t)m_distrib(gen);
                p[1] = k_distrib(gen);
                p += 2;
            }
        }
    }
    ck(faiss_GpuIcmEncoder_encode(h_, codes, x, (::idx_t)n, ils_iters, nperts, lsq->icm_iters, perts.data()));
}

B200IcmEncoderFactory::B200IcmEncoderFactory(int ngpus) {
    for (int i = 0; i < ngpus; i++) {
        res.push_back(std::make_unique<B200Resources>());
        devices.push_back(i);
    }
}

faiss::lsq::IcmEncoder* B200IcmEncoderFactory::get(const faiss::LocalSearchQuantizer* lsq) {
    std::vector<B200Resources*> rs;
    for (auto& r : res)
        rs.push_back(r.get());
    return new B200IcmEncoder(lsq, rs, devices);
}

// ------------------------------------------------------------------------------------------
// B200ResidualQuantizer
// ------------------------------------------------------------------------------------------
B200ResidualQuantizer::B200ResidualQuantizer(
        B200Resources* res,
        size_t d,
        const std::vector<size_t>& nbits,
        Search_type_t search_type,
        int device)
        : faiss::ResidualQuantizer(d, nbits, search_type), res_(res), device_(device) {
    FAISS_THROW_IF_NOT_MSG(res != nullptr, "null B200Resources");
}

B200ResidualQuantizer::B200ResidualQuantizer(B200Resources* res, size_t d, size_t M, size_t nbits, Search_type_t search_type, int device)
        : B200ResidualQuantizer(res, d, std::vector<size_t>(M, nbits), search_type, device) {}

void B200ResidualQuantizer::compute_codes_add_centroids(const float* x, uint8_t* codes_out, size_t n, const float* centroids) const {
    FAISS_THROW_IF_NOT_MSG(is_trained, "RQ is not trained yet.");
    FAISS_THROW_IF_NOT_MSG(
            approx_topk_mode == ::EXACT_TOPK,
            "B200ResidualQuantizer: the device beam search takes approx_topk_mode = EXACT_TOPK only");
    FAISS_THROW_IF_NOT_MSG(use_beam_LUT == 0 || use_beam_LUT == 1, "use_beam_LUT must be 0 or 1");
    std::vector<int> nb(nbits.begin(), nbits.end());
    FaissGpuRqEncoder* h = nullptr;
    ck(faiss_b200_RqEncoder_new(&h, res_->handle(), device_, (int)d, (int)M, nb.data()));
    std::unique_ptr<FaissGpuRqEncoder, void (*)(FaissGpuRqEncoder*)> guard(h, faiss_b200_RqEncoder_free);
    ck(faiss_b200_RqEncoder_set_codebooks(h, codebooks.data()));
    if (search_type <= ST_norm_qint4) { // packed on the device
        ck(faiss_b200_RqEncoder_compute_codes(
                h, x, (::idx_t)n, use_beam_LUT, max_beam_size, (int)search_type, norm_min, norm_max, centroids, codes_out));
        return;
    }
    // ST_norm_cqint*, ST_norm_*2x4: the CPU packs these from the decoded codes too (norms = nullptr)
    std::vector<int32_t> codes(n * M);
    ck(faiss_b200_RqEncoder_encode_unpacked(h, x, (::idx_t)n, use_beam_LUT, max_beam_size, codes.data()));
    pack_codes(n, codes.data(), codes_out, M, nullptr, centroids);
}

faiss::Index* B200ProgressiveDimIndexFactory::operator()(int dim) {
    ncall++;
    return new B200IndexFlat(&res, dim, faiss::METRIC_L2, device);
}

faiss::Index* index_cpu_to_b200(B200Resources* res, int device, const faiss::Index* index, const B200ClonerOptions* options) {
    if (auto* f = dynamic_cast<const faiss::IndexFlat*>(index))
        return new B200IndexFlat(res, f, device, options && options->useFloat16);
    if (auto* pq = dynamic_cast<const faiss::IndexIVFPQ*>(index))
        return new B200IndexIVFPQ(res, pq, device);
    if (auto* fl = dynamic_cast<const faiss::IndexIVFFlat*>(index))
        return new B200IndexIVFFlat(res, fl, device);
    FAISS_THROW_MSG("index_cpu_to_b200: this type of index is not on the faiss_b200 path (Flat, IVFFlat, IVFPQ are)");
}

faiss::Index* index_b200_to_cpu(const faiss::Index* index) {
    if (auto* f = dynamic_cast<const B200IndexFlat*>(index)) {
        auto* out = new faiss::IndexFlat(f->d, f->metric_type);
        f->copyTo(out);
        return out;
    }
    if (auto* pq = dynamic_cast<const B200IndexIVFPQ*>(index)) {
        auto* q = new faiss::IndexFlat(pq->d, pq->metric_type);
        auto* out = new faiss::IndexIVFPQ(q, pq->d, pq->nlist, pq->M, pq->nbits, pq->metric_type);
        out->own_fields = true;
        pq->copyTo(out);
        return out;
    }
    if (auto* fl = dynamic_cast<const B200IndexIVFFlat*>(index)) {
        auto* q = new faiss::IndexFlat(fl->d, fl->metric_type);
        auto* out = new faiss::IndexIVFFlat(q, fl->d, fl->nlist, fl->metric_type);
        out->own_fields = true;
        fl->copyTo(out);
        return out;
    }
    FAISS_THROW_MSG("index_b200_to_cpu: not a faiss_b200 adapter index");
}

} // namespace faiss_b200_adapter
