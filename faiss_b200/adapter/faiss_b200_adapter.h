// faiss_b200 adapter -- the backend behind the reference's OWN C++ interface.
//
// Each class derives from faiss::Index (faiss/Index.h:101-435) and forwards to the C ABI of libfaiss_b200.so
// (include/faiss_b200_c.h), so everything in Faiss that drives a `faiss::Index&` -- faiss::Clustering::train
// (faiss/Clustering.cpp:254-356), faiss::IndexShards / ThreadedIndex (faiss/IndexShards.cpp:197-264),
// ProductQuantizer::assign_index, IndexIVF's quantizer slot -- runs on the faiss_b200 kernels without a change at
// the call site.  index_cpu_to_b200 / index_b200_to_cpu are the cloner pair of faiss/gpu/GpuCloner.cpp:124-255
// (copyFrom / copyTo of GpuIndexFlat.cu:105-176, GpuIndexIVFFlat.cu:89-150, GpuIndexIVFPQ.cu:105-217; inverted
// lists are moved in the CPU ArrayInvertedLists byte format, so copyTo(copyFrom(x)) is byte-identical).
//
// Compiled against the reference's headers only (no reference source is copied); built by
// tests/adapter/build_adapter.py where /root/reference is available and exercised by tests/adapter/.
#pragma once

#include <faiss/Index.h>
#include <faiss/IndexFlat.h>
#include <faiss/IndexIVF.h>
#include <faiss/IndexIVFFlat.h>
#include <faiss/IndexIVFPQ.h>
#include <faiss/impl/LocalSearchQuantizer.h>
#include <faiss/impl/ResidualQuantizer.h>

#include <memory>
#include <random>
#include <vector>

struct FaissStandardGpuResources_H;
struct FaissIndex_H;
struct FaissGpuIcmEncoder_H;

namespace faiss_b200_adapter {

// faiss::gpu::StandardGpuResources' role: owns streams, temp memory and NCCL communicators
class B200Resources {
   public:
    B200Resources();
    ~B200Resources();
    B200Resources(const B200Resources&) = delete;
    B200Resources& operator=(const B200Resources&) = delete;
    FaissStandardGpuResources_H* handle() const {
        return h_;
    }
    void ncclInitAll(const std::vector<int>& devices);

   private:
    FaissStandardGpuResources_H* h_ = nullptr;
};

// common part: an opaque C handle + the forwarding of the faiss::Index virtuals
class B200Index : public faiss::Index {
   public:
    ~B200Index() override;
    void train(faiss::idx_t n, const float* x) override;
    void add(faiss::idx_t n, const float* x) override;
    void add_with_ids(faiss::idx_t n, const float* x, const faiss::idx_t* xids) override;
    void search(
            faiss::idx_t n,
            const float* x,
            faiss::idx_t k,
            float* distances,
            faiss::idx_t* labels,
            const faiss::SearchParameters* params = nullptr) const override;
    void reset() override;
    void reconstruct(faiss::idx_t key, float* recons) const override;
    void reconstruct_n(faiss::idx_t i0, faiss::idx_t ni, float* recons) const override;
    // one call for all keys (faiss::Index's default is one reconstruct per key)
    void reconstruct_batch(faiss::idx_t n, const faiss::idx_t* keys, float* recons) const override;
    // one call on the device: R is the entry each result was scored on, not the per-label reconstruct of
    // faiss::Index's default (which resolves an id stored twice to one fixed entry)
    void search_and_reconstruct(
            faiss::idx_t n,
            const float* x,
            faiss::idx_t k,
            float* distances,
            faiss::idx_t* labels,
            float* recons,
            const faiss::SearchParameters* params = nullptr) const override;
    FaissIndex_H* handle() const {
        return h_;
    }
    int device() const {
        return device_;
    }

   protected:
    B200Index(int d, faiss::MetricType metric, int device) : faiss::Index(d, metric), device_(device) {}
    void sync_();
    FaissIndex_H* h_ = nullptr;
    int device_;
};

class B200IndexFlat : public B200Index { // faiss::gpu::GpuIndexFlat (faiss/gpu/GpuIndexFlat.h:43-141)
   public:
    // useFloat16: GpuIndexFlatConfig::useFloat16 (faiss/gpu/GpuIndexFlat.h:26-35) -- fp16 storage, queries rounded to fp16
    B200IndexFlat(B200Resources* res, int dims, faiss::MetricType metric, int device = 0, bool useFloat16 = false);
    B200IndexFlat(B200Resources* res, const faiss::IndexFlat* index, int device = 0, bool useFloat16 = false);
    void copyFrom(const faiss::IndexFlat* index);
    void copyTo(faiss::IndexFlat* index) const;
};

class B200IndexIVF : public B200Index { // faiss::gpu::GpuIndexIVF (faiss/gpu/GpuIndexIVF.h:40-167)
   public:
    size_t nlist;
    size_t nprobe = 1;
    void search(
            faiss::idx_t n,
            const float* x,
            faiss::idx_t k,
            float* distances,
            faiss::idx_t* labels,
            const faiss::SearchParameters* params = nullptr) const override;
    void search_and_reconstruct(
            faiss::idx_t n,
            const float* x,
            faiss::idx_t k,
            float* distances,
            faiss::idx_t* labels,
            float* recons,
            const faiss::SearchParameters* params = nullptr) const override;

   protected:
    B200IndexIVF(int d, faiss::MetricType metric, size_t nlist_, int device) : B200Index(d, metric, device), nlist(nlist_) {}
    void search_(
            faiss::idx_t n,
            const float* x,
            faiss::idx_t k,
            float* distances,
            faiss::idx_t* labels,
            float* recons,
            const faiss::SearchParameters* params) const;
    void copyListsFrom_(const faiss::IndexIVF* index);
    void copyListsTo_(faiss::IndexIVF* index) const;
};

class B200IndexIVFFlat : public B200IndexIVF { // faiss/gpu/GpuIndexIVFFlat.h:24-119
   public:
    B200IndexIVFFlat(B200Resources* res, int dims, size_t nlist, faiss::MetricType metric, int device = 0);
    B200IndexIVFFlat(B200Resources* res, const faiss::IndexIVFFlat* index, int device = 0);
    void copyFrom(const faiss::IndexIVFFlat* index);
    void copyTo(faiss::IndexIVFFlat* index) const;
};

class B200IndexIVFPQ : public B200IndexIVF { // faiss/gpu/GpuIndexIVFPQ.h:56-181
   public:
    B200IndexIVFPQ(B200Resources* res, int dims, size_t nlist, size_t M, size_t nbits, faiss::MetricType metric, int device = 0);
    B200IndexIVFPQ(B200Resources* res, const faiss::IndexIVFPQ* index, int device = 0);
    void copyFrom(const faiss::IndexIVFPQ* index);
    void copyTo(faiss::IndexIVFPQ* index) const;
    size_t M, nbits;
};

// faiss::gpu::GpuIcmEncoder (faiss/gpu/GpuIcmEncoder.h): LocalSearchQuantizer's ICM encoding on the devices.  encode()
// draws the perturbations from `gen` exactly as LocalSearchQuantizer::perturb_codes does and hands them to the device,
// so `gen` ends in the state the CPU encoder leaves it in and the codes follow the CPU's random trajectory.
class B200IcmEncoder : public faiss::lsq::IcmEncoder {
   public:
    B200IcmEncoder(const faiss::LocalSearchQuantizer* lsq, const std::vector<B200Resources*>& res, const std::vector<int>& devices);
    ~B200IcmEncoder() override;
    B200IcmEncoder(const B200IcmEncoder&) = delete;
    B200IcmEncoder& operator=(const B200IcmEncoder&) = delete;
    void set_binary_term() override;
    void encode(int32_t* codes, const float* x, std::mt19937& gen, size_t n, size_t ils_iters) const override;

   private:
    FaissGpuIcmEncoder_H* h_ = nullptr;
};

// faiss::gpu::GpuIcmEncoderFactory: one B200Resources per device 0 .. ngpus - 1.  LocalSearchQuantizer deletes its
// icm_encoder_factory, so give it one made with new:  lsq.icm_encoder_factory = new B200IcmEncoderFactory(1);
struct B200IcmEncoderFactory : public faiss::lsq::IcmEncoderFactory {
    explicit B200IcmEncoderFactory(int ngpus = 1);
    faiss::lsq::IcmEncoder* get(const faiss::LocalSearchQuantizer* lsq) override;
    std::vector<std::unique_ptr<B200Resources>> res;
    std::vector<int> devices;
};

// faiss::ResidualQuantizer whose compute_codes (and so retrain_AQ_codebook under Train_refine_codebook) runs the beam
// search on the device, in the mode use_beam_LUT selects, with the codebooks of the moment uploaded on each call.  The
// search is the one compute_codes runs without an assign_index_factory; approx_topk_mode must be EXACT_TOPK.  The
// device packs ST_decompress .. ST_norm_qint4; for the other search types it returns the codes and the inherited
// pack_codes packs them on the host.  train() is the CPU's; give it a B200ProgressiveDimIndexFactory to put its
// k-means and beam assignment on the device.
class B200ResidualQuantizer : public faiss::ResidualQuantizer {
   public:
    B200ResidualQuantizer(
            B200Resources* res,
            size_t d,
            const std::vector<size_t>& nbits,
            Search_type_t search_type = ST_decompress,
            int device = 0);
    B200ResidualQuantizer(B200Resources* res, size_t d, size_t M, size_t nbits, Search_type_t search_type = ST_decompress, int device = 0);
    void compute_codes_add_centroids(const float* x, uint8_t* codes, size_t n, const float* centroids = nullptr) const override;

   private:
    B200Resources* res_;
    int device_;
};

// faiss::gpu::GpuProgressiveDimIndexFactory (faiss/gpu/GpuCloner.h:85-100) on one device: every index it makes is a
// B200IndexFlat (L2), so ProgressiveDimClustering's k-means and ResidualQuantizer's beam assignment run on the Flat
// kernels.  ncall counts the indexes made.
struct B200ProgressiveDimIndexFactory : public faiss::ProgressiveDimIndexFactory {
    explicit B200ProgressiveDimIndexFactory(int device = 0) : device(device) {}
    faiss::Index* operator()(int dim) override;
    B200Resources res;
    int device;
    int ncall = 0;
};

// faiss::gpu::index_cpu_to_gpu / index_gpu_to_cpu (faiss/gpu/GpuCloner.cpp:124-255) for the three index types on the path
// the fields of GpuClonerOptions (faiss/gpu/GpuClonerOptions.h:17-56) that act on this path
struct B200ClonerOptions {
    bool useFloat16 = false; // Flat: fp16 storage
};
faiss::Index* index_cpu_to_b200(B200Resources* res, int device, const faiss::Index* index, const B200ClonerOptions* options = nullptr);
faiss::Index* index_b200_to_cpu(const faiss::Index* index);

} // namespace faiss_b200_adapter
