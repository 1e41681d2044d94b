// faiss_b200 -- host-side index objects (L2/L3): the drop-in surface.
//
// Mirrors the reference classes (same member names, argument meaning, limits and error behaviour):
//   faiss::Index                      faiss/Index.h:101-435
//   faiss::gpu::GpuIndex              faiss/gpu/GpuIndex.h:53-297, GpuIndex.cu
//   faiss::gpu::GpuIndexFlat{,L2,IP}  faiss/gpu/GpuIndexFlat.h:26-217, GpuIndexFlat.cu:28-457
//   faiss::gpu::GpuIndexIVF           faiss/gpu/GpuIndexIVF.h:40-167, GpuIndexIVF.cu
//   faiss::gpu::GpuIndexIVFFlat       faiss/gpu/GpuIndexIVFFlat.h:24-119
//   faiss::gpu::GpuIndexIVFPQ         faiss/gpu/GpuIndexIVFPQ.h:25-181, GpuIndexIVFPQ.cu:29-622
//   faiss::Clustering                 faiss/Clustering.h:22-229, Clustering.cpp:60-380
//   faiss::IndexShards                faiss/IndexShards.h:21-106, IndexShards.cpp:87-264
// Everything device-side goes through kernels.h and flat_tc.h.
#pragma once

#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "common.h"
#include "flat_tc.h"
#include "idselector.h"
#include "kernels.h"
#include "resources.h"

namespace fb200 {

struct SearchParameters;

// ------------------------------------------------------------------------------------------
// faiss::Index
// ------------------------------------------------------------------------------------------
struct Index {
    int d;
    idx_t ntotal = 0;
    bool verbose = false;
    bool is_trained = true;
    MetricType metric_type;
    float metric_arg = 0.f;

    explicit Index(int d_ = 0, MetricType m = METRIC_L2) : d(d_), metric_type(m) {}
    virtual ~Index() = default;

    virtual void train(idx_t /*n*/, const float* /*x*/) {}
    virtual void add(idx_t n, const float* x) = 0;
    virtual void add_with_ids(idx_t n, const float* x, const idx_t* xids);
    virtual void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const = 0;
    virtual void assign(idx_t n, const float* x, idx_t* labels, idx_t k = 1) const;
    virtual void reset() = 0;
    virtual void reconstruct(idx_t key, float* recons) const;
    virtual void reconstruct_batch(idx_t n, const idx_t* keys, float* recons) const;
    virtual void reconstruct_n(idx_t i0, idx_t ni, float* recons) const;
    virtual void compute_residual(const float* x, float* residual, idx_t key) const;
    virtual void compute_residual_n(idx_t n, const float* xs, float* residuals, const idx_t* keys) const;
    // faiss::Index::search_and_reconstruct (faiss/Index.h:238-254): search, and recons [n][k][d] = the stored vector of
    // each result, all 0xFF bytes where the label is -1.  Only GpuIndexFlat and the IVF indexes implement it.
    virtual void search_and_reconstruct(
            idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, float* recons,
            const SearchParameters* params = nullptr) const;
};

// faiss::SearchParameters / SearchParametersIVF (faiss/Index.h:88-93, faiss/IndexIVF.h:68-90): per-call overrides.
// GPU indexes accept them like the reference's (faiss/gpu/GpuIndexIVF.cu:383-406), max_codes == 0.
struct SearchParameters {
    // results are restricted to the stored ids sel accepts (not owned): the row number for GpuIndexFlat, the id
    // stored in the list for the IVF indexes, whose coarse search is not filtered (as CPU IndexIVF)
    const IDSelector* sel = nullptr;
    virtual ~SearchParameters() {}
};
struct SearchParametersIVF : SearchParameters {
    size_t nprobe = 1;
    size_t max_codes = 0;
    SearchParameters* quantizer_params = nullptr;
};

// faiss::InterruptCallback (faiss/impl/AuxIndexStructures.h): a process-wide hook polled between query pages,
// add pages, search rounds and clustering iterations (the reference polls between tiles,
// faiss/gpu/impl/Distance.cu:245,266,403-405); when it returns true the running call throws
// "computation interrupted".
struct InterruptCallback {
    typedef int (*Fn)(void* ctx);
    static void set(Fn fn, void* ctx);
    static void clear();
    static bool is_interrupted();
    static void check(); // throws FaissException if the callback asks to stop
};

// ------------------------------------------------------------------------------------------
// GpuIndex
// ------------------------------------------------------------------------------------------
struct GpuIndexConfig { // faiss/gpu/GpuIndex.h:32-47
    int device = 0;
    MemorySpace memorySpace = MemorySpace::Device;
};

class GpuIndex : public Index {
   public:
    GpuIndex(std::shared_ptr<GpuResources> resources, int dims, MetricType metric, float metricArg, GpuIndexConfig config);

    int getDevice() const {
        return config_.device;
    }
    std::shared_ptr<GpuResources> getResources() {
        return resources_;
    }
    void setMinPagingSize(size_t size) {
        minPagedSize_ = size;
    }
    size_t getMinPagingSize() const {
        return minPagedSize_;
    }

    // x / ids / distances / labels may live on the host or on any device
    void add(idx_t n, const float* x) override;
    void add_with_ids(idx_t n, const float* x, const idx_t* ids) override;
    void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const override;
    // faiss::Index::search(..., const SearchParameters* params) (faiss/Index.h:207-214, faiss/gpu/GpuIndex.cu:373-448)
    void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, const SearchParameters* params) const;
    void assign(idx_t n, const float* x, idx_t* labels, idx_t k = 1) const override;
    void compute_residual(const float* x, float* residual, idx_t key) const override;
    void compute_residual_n(idx_t n, const float* xs, float* residuals, const idx_t* keys) const override;

   protected:
    // the per-call parameters of the search in flight (an index instance is not re-entrant, as upstream)
    mutable const SearchParameters* callParams_ = nullptr;
    // the row, in the whole search call, of the first query handed to searchImpl_ (set by the query paging)
    mutable idx_t callRow0_ = 0;
    // callParams_->sel evaluated once per call over the index's storage slots (idselector.h), else null
    mutable const uint32_t* callMask_ = nullptr;
    // sel over this index's slots into a device mask of slotMaskWords(slots) words (temporary memory)
    virtual GpuMemoryReservation selMask_(const IDSelector& sel) const = 0;
    virtual bool addImplRequiresIDs_() const = 0;
    virtual void addImpl_(idx_t n, const float* xDev, const idx_t* idsDev) = 0;
    virtual void searchImpl_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev) const = 0;
    // host queries above the paging threshold: pinned double buffers + async-copy stream (GpuIndex.cu:620-788)
    bool searchFromCpuPaged_(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, idx_t maxQ) const;

   public:
    // Shard-local half of a sharded search (device pointers, ids local to this shard).  `flatShard` is
    // non-null only when EVERY rank of the communicator runs the tensor-core Flat path: the ranks then pool
    // their thresholds after every round, and a shard may return fewer than k entries (-1 padded) -- those it
    // can prove are not in the global top-k.  All ranks must make the call with identical queries and k.
    virtual void searchShardDevice(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, const FlatTcShard* flatShard) const {
        (void)flatShard;
        searchImpl_(n, xDev, k, dDev, iDev);
    }
    // would this index take the tensor-core Flat path for (its current size, k)?  (sharded search: the
    // pooled-threshold protocol is used only if this holds on every rank)
    virtual bool shardPoolingEligible(int /*k*/, idx_t /*n*/) const {
        return false;
    }

   protected:
    cudaStream_t stream_() const {
        return resources_->getDefaultStream(config_.device);
    }

    std::shared_ptr<GpuResources> resources_;
    GpuIndexConfig config_;
    size_t minPagedSize_ = size_t(256) << 20; // faiss/gpu/GpuIndex.cu kMinPageSize
};

// ------------------------------------------------------------------------------------------
// GpuIndexFlat
// ------------------------------------------------------------------------------------------
struct GpuIndexFlatConfig : GpuIndexConfig { // faiss/gpu/GpuIndexFlat.h:26-35
    bool useFloat16 = false;        // store the vectors as fp16; queries are rounded to fp16 too (FlatIndex.cu:112-136)
    bool useTensorCores = true;     // false: always take the exact SIMT kernel
};

class GpuIndexFlat : public GpuIndex {
   public:
    GpuIndexFlat(
            std::shared_ptr<GpuResources> resources,
            int dims,
            MetricType metric,
            GpuIndexFlatConfig config = GpuIndexFlatConfig());
    ~GpuIndexFlat() override;

    // copyFrom / copyTo against the CPU IndexFlat payload (xb, row-major fp32)
    // (faiss/gpu/GpuIndexFlat.cu:105-176: index->get_xb(), ntotal)
    void copyFrom(idx_t n, const float* xb);
    void copyTo(float* xbOut) const;
    size_t getNumVecs() const {
        return (size_t)ntotal;
    }

    void reset() override;
    void train(idx_t n, const float* x) override;
    void add(idx_t n, const float* x) override;
    void add_with_ids(idx_t n, const float* x, const idx_t* ids) override; // unsupported, as upstream
    void reconstruct(idx_t key, float* out) const override;
    void reconstruct_n(idx_t i0, idx_t num, float* out) const override;
    void reconstruct_batch(idx_t n, const idx_t* keys, float* out) const override;
    void compute_residual(const float* x, float* residual, idx_t key) const override;
    void compute_residual_n(idx_t n, const float* xs, float* residuals, const idx_t* keys) const override;
    using GpuIndex::search;
    void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const override;
    // search, then the returned rows (fp16 storage: widened, as reconstruct)
    void search_and_reconstruct(
            idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, float* recons,
            const SearchParameters* params = nullptr) const override;

    // device-pointer entry points used by IVF / clustering (role of FlatIndex::query)
    void searchDevice(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev) const {
        lastSearchFallbackQueries = 0;
        searchImpl_(n, xDev, k, dDev, iDev);
    }
    void searchShardDevice(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, const FlatTcShard* flatShard) const override;
    bool shardPoolingEligible(int k, idx_t n) const override;
    const float* vectorsDevice() const { // fp32 rows (IVF coarse centroids); not available under useFloat16
        FB_THROW_IF_NOT_MSG(!flatConfig_.useFloat16, "fp32 row access on a float16 GpuIndexFlat");
        return vecs_.data();
    }
    bool usesFloat16() const {
        return flatConfig_.useFloat16;
    }
    void setUseTensorCores(bool v) {
        flatConfig_.useTensorCores = v;
    }
    // replace the whole content by n device rows without giving the storage back (the k-means loop installs a new
    // centroid table every iteration: reset() + add() would free and re-allocate five buffers each time)
    void replaceVectorsDevice(idx_t n, const float* xDev);
    // the fp32 storage resized to n rows, contents undefined, for the caller to fill on the default stream (bfKnn
    // converts fp16 / bf16 / column-major vectors straight into it); not available under useFloat16
    float* resizeVectorsDevice(idx_t n);
    // diagnostics of the last search (fallback queries: exact recomputes, summed over the whole call)
    mutable int lastSearchUsedTensorCores = 0;
    mutable int lastSearchFallbackQueries = 0;
    mutable int lastSearchOperandBits = 0; // tensor-core operand width of the last search: 8 or 16; 0: exact kernel

   protected:
    bool addImplRequiresIDs_() const override {
        return false;
    }
    void addImpl_(idx_t n, const float* xDev, const idx_t* idsDev) override;
    void searchImpl_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev) const override;
    GpuMemoryReservation selMask_(const IDSelector& sel) const override; // slot = row, id = row
    // the selected rows only: gathered (fp32) and searched with the exact kernel, labels mapped back
    void searchCompacted_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev, idx_t selected) const;
    void fillEmpty_(idx_t n, int k, float* dDev, idx_t* iDev) const;
    // the metric the kernels run, read at search time: METRIC_Lp with metric_arg 1 is L1 and with 2 is L2
    // (faiss/gpu/impl/Distance.cuh:223-239); only L2 and inner product can take the tensor-core path
    MetricType searchMetric_() const;
    bool tensorCoreMetric_() const {
        const MetricType m = searchMetric_();
        return m == METRIC_L2 || m == METRIC_INNER_PRODUCT;
    }
    // does a search of n queries for k results take the tensor cores?  (tiny batches stay exact)
    bool useTensorCores_(int k, idx_t n) const {
        return flatConfig_.useTensorCores && tensorCoreMetric_() && flatTcSupported(d, k, this->ntotal) && n >= 16;
    }

    const void* rows_() const { // the stored rows, as the kernels take them (with yHalf_())
        return flatConfig_.useFloat16 ? (const void*)vecs16_.data() : (const void*)vecs_.data();
    }
    int yHalf_() const {
        return flatConfig_.useFloat16 ? 1 : 0;
    }
    // useFloat16: the query block rounded to fp16 and widened again (what the reference's convertTensor does before
    // its half GEMM); returns x itself otherwise
    const float* roundedQueries_(idx_t n, const float* xDev, GpuMemoryReservation& hold) const;

    GpuIndexFlatConfig flatConfig_;
    mutable idx_t callSelected_ = 0; // rows selected by callMask_ (counted once per call, in selMask_)
    DeviceVector<float> vecs_;    // fp32 storage (default)
    DeviceVector<__half> vecs16_; // fp16 storage (useFloat16): the only copy of the vectors besides the scoring tiles
    mutable FlatTcDatabase tc_; // rebuilt lazily after the rows change
};

class GpuIndexFlatL2 : public GpuIndexFlat {
   public:
    GpuIndexFlatL2(std::shared_ptr<GpuResources> r, int dims, GpuIndexFlatConfig c = GpuIndexFlatConfig())
            : GpuIndexFlat(std::move(r), dims, METRIC_L2, c) {}
};
class GpuIndexFlatIP : public GpuIndexFlat {
   public:
    GpuIndexFlatIP(std::shared_ptr<GpuResources> r, int dims, GpuIndexFlatConfig c = GpuIndexFlatConfig())
            : GpuIndexFlat(std::move(r), dims, METRIC_INNER_PRODUCT, c) {}
};

// ------------------------------------------------------------------------------------------
// Clustering (Lloyd k-means, training set resident on the device)
// ------------------------------------------------------------------------------------------
struct ClusteringParameters { // faiss/Clustering.h:22-78
    int niter = 25;
    int nredo = 1;
    bool verbose = false;
    bool spherical = false;
    bool int_centroids = false;
    bool update_index = false;
    bool frozen_centroids = false;
    int min_points_per_centroid = 39;
    int max_points_per_centroid = 256;
    int seed = 1234;
};

struct ClusteringIterationStats { // faiss/Clustering.h:80-92
    float obj;
    double time;
    double time_search;
    double imbalance_factor;
    int nsplit;
};

struct Clustering : ClusteringParameters {
    size_t d;
    size_t k;
    std::vector<float> centroids; // (k * d), host copy, as upstream
    std::vector<ClusteringIterationStats> iteration_stats;

    Clustering(int d, int k) : d(d), k(k) {}
    Clustering(int d, int k, const ClusteringParameters& cp) : ClusteringParameters(cp), d(d), k(k) {}
    // x: host or device pointer.  `index` is the assignment index (reset / add / search k=1).
    void train(idx_t n, const float* x, GpuIndexFlat& index);
    // `train`'s Lloyd loop with the training set SHARDED over the ranks of `comm` (rank order = row order of the
    // concatenated set) and the centroid table replicated; the only addition is one all-reduce per iteration, so the
    // result equals `train` on the concatenated set (SURVEY 8(e)).  Collective: every rank calls it with its own
    // rows; sub-sampling is the caller's business.  Every rank ends with identical centroids (also in `index`).
    void trainSharded(idx_t nLocal, const float* xLocal, GpuIndexFlat& index, const Communicator& comm);
    double splitSeconds = 0; // host time inside split_clusters during the last train / trainSharded

   private:
    // One Lloyd run, initialisation to last iteration, over rows [off, off + nLocal) of an nTotal-row training set
    // (xLocal on the device); comm == nullptr for a single process.  Fills `centroids`, appends to
    // `iteration_stats` and returns the last objective.  t0 / tSearch: the run's start and its search-time total.
    float lloyd_(idx_t nLocal, const float* xLocal, idx_t nTotal, idx_t off, GpuIndexFlat& index, int redo,
                 const Communicator* comm, double t0, double& tSearch);
};

// ProductQuantizer::train, Train_default (faiss/impl/ProductQuantizer.cpp:130-195); x device [n,d], pqOut host
// [M][ksub][d/M]
void trainProductQuantizer(
        std::shared_ptr<GpuResources> resources,
        int device,
        idx_t n,
        const float* xDev,
        int d,
        int M,
        int ksub,
        const ClusteringParameters& cp,
        float* pqOut);

// helpers restated from the reference so that seeds reproduce its sampling decisions
void rand_perm(int* perm, size_t n, int64_t seed);                   // faiss/utils/random.cpp:188-199
int split_clusters(size_t d, size_t k, size_t n, float* hassign, float* centroids); // ClusteringHelpers.cpp:177-240

// ------------------------------------------------------------------------------------------
// inverted-list storage
// ------------------------------------------------------------------------------------------
class IvfLists {
   public:
    // pqInterleaved: store codes in the rotated, interleaved-by-32 PQ layout (kernels.h); the
    // host-facing accessors below always speak the flat [len][codeSize] ArrayInvertedLists format
    IvfLists(GpuResources* res, int device, int64_t nlist, int codeSize, bool pqInterleaved = false);
    ~IvfLists();
    void reset();
    void reserve(size_t totalVecs, cudaStream_t stream);
    // exact per-list capacities in ONE relayout (bulk copyFrom: all list lengths are known up front)
    void reserveLists(const int64_t* lens, cudaStream_t stream);
    // append n encoded rows (device pointers); assign[i] in [0,nlist) or -1 (skipped)
    // returns the number of rows actually stored
    idx_t append(idx_t n, const uint8_t* rowsDev, const idx_t* idsDev, const idx_t* assignDev, cudaStream_t stream);
    // bulk load of one list from host memory (copyFrom)
    void setListFromHost(int64_t l, int64_t len, const uint8_t* codes, const idx_t* ids, cudaStream_t stream);
    void getListToHost(int64_t l, uint8_t* codes, idx_t* ids, cudaStream_t stream) const;
    int64_t listLength(int64_t l) const {
        return hLen_[l];
    }
    int64_t listStart(int64_t l) const { // arena position of the list's first entry
        return hStart_[l];
    }
    size_t reclaim(cudaStream_t stream);

    const int64_t* dStart() const {
        return dStart_;
    }
    const int* dLen() const {
        return dLen_;
    }
    const uint8_t* codes() const {
        return codes_;
    }
    const idx_t* ids() const {
        return ids_;
    }
    int64_t nlist() const {
        return nlist_;
    }
    int codeSize() const {
        return codeSize_;
    }
    int maxListLength() const;
    int64_t arenaElems() const {
        return arenaElems_;
    }
    bool interleaved() const {
        return interleaved_;
    }

   private:
    void relayout_(const std::vector<int64_t>& newCap, cudaStream_t stream);
    void uploadMeta_(cudaStream_t stream);

    GpuResources* res_;
    int device_;
    int64_t nlist_;
    int codeSize_;
    bool interleaved_ = false;
    uint8_t* codes_ = nullptr;
    idx_t* ids_ = nullptr;
    int64_t arenaElems_ = 0;
    std::vector<int64_t> hStart_, hCap_;
    std::vector<int> hLen_;
    int64_t* dStart_ = nullptr;
    int* dLen_ = nullptr;
    int* dCounts_ = nullptr;
};

// ------------------------------------------------------------------------------------------
// GpuIndexIVF
// ------------------------------------------------------------------------------------------
enum IndicesOptions { INDICES_CPU = 0, INDICES_IVF = 1, INDICES_32_BIT = 2, INDICES_64_BIT = 3 };

struct GpuIndexIVFConfig : GpuIndexConfig { // faiss/gpu/GpuIndexIVF.h:23-35
    IndicesOptions indicesOptions = INDICES_64_BIT;
    GpuIndexFlatConfig flatConfig;
    bool allowCpuCoarseQuantizer = false;
};

class GpuIndexIVF : public GpuIndex {
   public:
    GpuIndexIVF(
            std::shared_ptr<GpuResources> resources,
            int dims,
            MetricType metric,
            idx_t nlist,
            int codeSize,
            GpuIndexIVFConfig config,
            bool pqInterleaved = false);
    ~GpuIndexIVF() override;

    idx_t nlist;
    size_t nprobe = 1;
    size_t max_codes = 0;
    GpuIndexFlat* quantizer = nullptr;
    // bumped whenever the coarse centroids are (re)installed through this class (train, setCoarseCentroids);
    // derived classes key centroid-dependent side tables on it
    uint64_t coarseEpoch = 0;
    bool own_fields = true;
    ClusteringParameters cp;

    idx_t getNumLists() const {
        return nlist;
    }
    idx_t getListLength(idx_t listId) const;
    std::vector<uint8_t> getListVectorData(idx_t listId) const;
    std::vector<idx_t> getListIndices(idx_t listId) const;
    void reserveMemory(size_t numVecs);
    // bulk-clone helper: exact capacity for every list in one arena relayout, before nlist x setList
    // (the role of the per-list reserve in IVFBase::copyInvertedListsFrom, faiss/gpu/impl/IVFBase.cu:328-451)
    void setListSizes(const idx_t* lens);
    size_t reclaimMemory();
    void reset() override;
    // share an existing coarse quantiser instead of the internally created one (not owned)
    void setQuantizer(GpuIndexFlat* coarse);
    // install coarse centroids [nlist,d] (copyFrom of the CPU quantizer's xb)
    void setCoarseCentroids(const float* centroidsHostOrDev);
    void getCoarseCentroids(float* out) const;
    // bulk list load (copyFrom ArrayInvertedLists): codes [len*code_size], ids [len]
    void setList(idx_t listId, idx_t len, const uint8_t* codes, const idx_t* ids);
    // the coarse quantiser (k-means, unless it already holds nlist centroids), then the encoder (trainEncoder_)
    void train(idx_t n, const float* x) override;

    // faiss/gpu/GpuIndexIVF.cu:408-488
    void search_preassigned(
            idx_t n,
            const float* x,
            idx_t k,
            const idx_t* assign,
            const float* centroid_dis,
            float* distances,
            idx_t* labels) const;

    // faiss::IndexIVF retrieval (faiss/IndexIVF.cpp:1056-1248), decoded on the device with reconstruct_from_offset's
    // arithmetic.  No direct map is kept: an id stored more than once resolves to the entry last in (list, offset)
    // order, as the CPU's reconstruct_n loop; reconstruct / reconstruct_batch throw "key not found" for an id that is
    // not stored, before writing anything.  Outputs may live on the host or the device.
    void reconstruct(idx_t key, float* recons) const override;
    void reconstruct_n(idx_t i0, idx_t ni, float* recons) const override; // rows of ids not stored are left as they are
    void reconstruct_batch(idx_t n, const idx_t* keys, float* recons) const override;
    // D and I equal search(..., params); recons decodes the entry each result came from
    void search_and_reconstruct(
            idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, float* recons,
            const SearchParameters* params = nullptr) const override;
    // codes [n][k][coarse_code_size() (include_listno) + code_size]: the CPU ArrayInvertedLists bytes of each result,
    // prefixed by its list number in little-endian bytes; all 0xFF where the label is -1
    void search_and_return_codes(
            idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, uint8_t* codes, bool include_listno,
            const SearchParameters* params = nullptr) const;
    // IndexIVF::coarse_code_size: bytes of a list number (faiss/IndexIVF.cpp encode_listno)
    int coarse_code_size() const;
    int code_size() const {
        return lists_->codeSize();
    }

   protected:
    // the decoder's view of this index's lists
    virtual IvfStoredLayout storedLayout_() const = 0;
    IvfStoredLayout listLayout_() const;
    idx_t retrievalPageRows_(const float* out, idx_t n) const;
    // search with the slot of every result: per page of queries, `page(i0, nb, slotsDev)` runs after D / I of the
    // page are on the device (slotsDev [nb][k], -1 with a missing result); resultBytes (the page's output per result)
    // bounds the page size
    void searchWithSlots_(
            idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, const SearchParameters* params,
            size_t resultBytes, const std::function<void(idx_t, idx_t, const idx_t*)>& page) const;
    // set while searchWithSlots_ runs: scanImpl_ hands the scans callSlots_->identity instead of the list ids
    mutable const IvfSlotOutput* callSlots_ = nullptr;
    const idx_t* scanIds_() const {
        return callSlots_ ? callSlots_->identity : lists_->ids();
    }

    bool addImplRequiresIDs_() const override {
        return true;
    }
    void trainQuantizer_(idx_t n, const float* xDev);
    // is a trained coarse quantiser all the training this index needs? (IVF-Flat: yes; IVF-PQ: the PQ too)
    virtual bool quantizerOnlyTraining_() const {
        return true;
    }
    // train what encodes the list entries, after the coarse quantiser (IVF-Flat: nothing)
    virtual void trainEncoder_(idx_t /*n*/, const float* /*xDev*/) {}
    // coarse k = 1 assignment, encode_, append to the lists
    void addImpl_(idx_t n, const float* xDev, const idx_t* idsDev) override;
    // the list entries (codeSize bytes each) of n rows whose coarse assignment is assignDev; the result may live in
    // `hold`.  Throws before anything is appended when the encoder is not trained.
    virtual const uint8_t* encode_(idx_t n, const float* xDev, const idx_t* assignDev, GpuMemoryReservation& hold) = 0;
    // x - (its coarse centroid).  In add, assignDev is the rows' assignment and the buffer comes from the temp stack;
    // in training assignDev is null, the k = 1 assignment runs here, and the buffers are device allocations.
    GpuMemoryReservation coarseResiduals_(idx_t n, const float* xDev, const idx_t* assignDev) const;
    void searchImpl_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev) const override;
    GpuMemoryReservation selMask_(const IDSelector& sel) const override; // slot = arena position, id = stored id
    virtual void scanImpl_(
            idx_t n,
            const float* xDev,
            const idx_t* probesDev,
            const float* coarseDisDev,
            int nprobe,
            int k,
            float* dDev,
            idx_t* iDev) const = 0;

    GpuIndexIVFConfig ivfConfig_;
    std::unique_ptr<IvfLists> lists_;
};

class GpuIndexIVFFlat : public GpuIndexIVF {
   public:
    GpuIndexIVFFlat(
            std::shared_ptr<GpuResources> resources,
            int dims,
            idx_t nlist,
            MetricType metric = METRIC_L2,
            GpuIndexIVFConfig config = GpuIndexIVFConfig());
    // faiss/gpu/GpuIndexIVFFlat.h:48-59: with an external (shared) coarse quantiser
    GpuIndexIVFFlat(
            std::shared_ptr<GpuResources> resources,
            GpuIndexFlat* coarseQuantizer,
            int dims,
            idx_t nlist,
            MetricType metric = METRIC_L2,
            GpuIndexIVFConfig config = GpuIndexIVFConfig());

   protected:
    const uint8_t* encode_(idx_t n, const float* xDev, const idx_t* assignDev, GpuMemoryReservation& hold) override;
    void scanImpl_(idx_t, const float*, const idx_t*, const float*, int, int, float*, idx_t*) const override;
    IvfStoredLayout storedLayout_() const override;
};

struct GpuIndexIVFPQConfig : GpuIndexIVFConfig { // faiss/gpu/GpuIndexIVFPQ.h:25-49
    bool useFloat16LookupTables = false;
    bool usePrecomputedTables = false;
    bool interleavedLayout = false;
    bool useMMCodeDistance = false;
};

// Code widths (verifyPQSettings_, faiss/gpu/GpuIndexIVFPQ.cu:555-617): nbits = 8 by default; with
// config.interleavedLayout also 4, 5 or 6.  Lists always hold the CPU's ceil(M * nbits / 8)-byte codes.  The
// device layout follows from (nbits, M), not from the flag: the interleaved-by-32 layout for nbits = 8 with
// M in {16, 32} and for nbits = 4 with M in {32, 64} (nibble pairs as M/2 code bytes), else vector-major.
class GpuIndexIVFPQ : public GpuIndexIVF {
   public:
    GpuIndexIVFPQ(
            std::shared_ptr<GpuResources> resources,
            int dims,
            idx_t nlist,
            idx_t subQuantizers,
            idx_t bitsPerCode,
            MetricType metric = METRIC_L2,
            GpuIndexIVFPQConfig config = GpuIndexIVFPQConfig());
    // faiss/gpu/GpuIndexIVFPQ.h:69-82: with an external (shared) coarse quantiser
    GpuIndexIVFPQ(
            std::shared_ptr<GpuResources> resources,
            GpuIndexFlat* coarseQuantizer,
            int dims,
            idx_t nlist,
            idx_t subQuantizers,
            idx_t bitsPerCode,
            MetricType metric = METRIC_L2,
            GpuIndexIVFPQConfig config = GpuIndexIVFPQConfig());
    ~GpuIndexIVFPQ() override;

    int getNumSubQuantizers() const {
        return M_;
    }
    int getBitsPerCode() const {
        return nbits_;
    }
    int getCentroidsPerSubQuantizer() const {
        return 1 << nbits_;
    }
    // Precomputed term-2 table  T2[list][code][m] = ||y||^2 + 2 <centroid_list|m, y>  (the role of
    // faiss/gpu/impl/IVFPQ.cu:362-489 and IndexIVFPQ::precompute_table, faiss/IndexIVFPQ.cpp:376-458).
    // With it the per-(query, list) lookup table is T2[list] + (-2 <x|m, y>) -- one load and one add per
    // entry instead of dsub multiply-adds, which is what matters when lists are short (nlist = 65536).
    // L2 + interleaved layout + nbits = 8 only (accepted, not honoured otherwise).  Policy: on when explicitly enabled; otherwise "auto" = the table is at
    // most precomputed_table_max_bytes (2 GiB, faiss/IndexIVFPQ.cpp:345) AND lists are short (< 4096 vectors
    // on average) -- with long lists the direct on-chip build is faster (see GpuIndexIVFPQ::precomputedActive_).
    void setPrecomputedCodes(bool enable) {
        usePrecomputed_ = enable;
        precomputedExplicit_ = true;
    }
    bool getPrecomputedCodes() const {
        return usePrecomputed_;
    }
    ClusteringParameters pq_cp; // ProductQuantizer::cp (faiss/impl/ProductQuantizer.h)
    // PQ centroids, layout [M][ksub][dsub] (ksub = 2^nbits) as in faiss::ProductQuantizer::centroids
    void setPQCentroids(const float* c);
    void getPQCentroids(float* out) const;

   protected:
    bool quantizerOnlyTraining_() const override {
        return false;
    }
    void trainEncoder_(idx_t n, const float* xDev) override; // the PQ, on residuals
    const uint8_t* encode_(idx_t n, const float* xDev, const idx_t* assignDev, GpuMemoryReservation& hold) override;
    void scanImpl_(idx_t, const float*, const idx_t*, const float*, int, int, float*, idx_t*) const override;
    IvfStoredLayout storedLayout_() const override;

    int M_, nbits_;
    int ksub_() const {
        return 1 << nbits_;
    }
    // 4-bit codes stored as M/2 nibble-pair bytes in the interleaved layout
    bool nibbleLayout_() const {
        return nbits_ == 4 && lists_->interleaved();
    }
    bool precomputedActive_() const;
    void ensureTerm2_() const;

    bool usePrecomputed_ = false;
    bool precomputedExplicit_ = false;
    uint64_t pqEpoch_ = 0;
    mutable DeviceVector<float> term2_; // [nlist][256][M]
    mutable uint64_t term2Key_ = ~uint64_t(0);
    DeviceVector<float> pqCentroids_;  // [M][ksub][dsub]
    DeviceVector<float> pqCentroidsT_; // [ksub][M][dsub] (LUT build reads it coalesced)
};

struct GpuIndexIVFScalarQuantizerConfig : GpuIndexIVFConfig { // faiss/gpu/GpuIndexIVFScalarQuantizer.h:20-27
    bool interleavedLayout = true; // accepted, not honoured: lists keep the CPU's [len][code_size] layout
};

// faiss::gpu::GpuIndexIVFScalarQuantizer (faiss/gpu/GpuIndexIVFScalarQuantizer.h:30-139); training and encoding
// follow the CPU IndexIVFScalarQuantizer (faiss/IndexScalarQuantizer.cpp:122-215, faiss/IndexIVF.cpp:1296-1329)
class GpuIndexIVFScalarQuantizer : public GpuIndexIVF {
   public:
    GpuIndexIVFScalarQuantizer(
            std::shared_ptr<GpuResources> resources,
            int dims,
            idx_t nlist,
            int qtype,
            MetricType metric = METRIC_L2,
            bool encodeResidual = true,
            GpuIndexIVFScalarQuantizerConfig config = GpuIndexIVFScalarQuantizerConfig());
    GpuIndexIVFScalarQuantizer(
            std::shared_ptr<GpuResources> resources,
            GpuIndexFlat* coarseQuantizer,
            int dims,
            idx_t nlist,
            int qtype,
            MetricType metric = METRIC_L2,
            bool encodeResidual = true,
            GpuIndexIVFScalarQuantizerConfig config = GpuIndexIVFScalarQuantizerConfig());

    // ScalarQuantizer::code_size (faiss/impl/ScalarQuantizer.cpp:451-520)
    static int codeSizeFor(int qtype, int d);
    int qtype() const {
        return qtype_;
    }
    bool by_residual;
    // ScalarQuantizer::rangestat / rangestat_arg: train() implements RS_minmax (0) only
    int rangestat = 0;
    float rangestat_arg = 0.f;

    void train(idx_t n, const float* x) override; // rejects rangestat != RS_minmax before any training work
    // ScalarQuantizer::trained: [vmin, vdiff] (uniform types), [vmin[d], vdiff[d]] (non-uniform), empty (fp16, direct)
    void setTrained(const float* t, size_t n);
    const std::vector<float>& getTrained() const {
        return trained_;
    }
    size_t trainedSize() const; // the length setTrained expects

   protected:
    bool quantizerOnlyTraining_() const override {
        return trainedSize() == 0;
    }
    void trainEncoder_(idx_t n, const float* xDev) override; // the RS_minmax ranges
    const uint8_t* encode_(idx_t n, const float* xDev, const idx_t* assignDev, GpuMemoryReservation& hold) override;
    void scanImpl_(idx_t, const float*, const idx_t*, const float*, int, int, float*, idx_t*) const override;
    IvfStoredLayout storedLayout_() const override;

    int qtype_;
    std::vector<float> trained_;
    DeviceVector<float> params_; // [4][d]: vmin | vdiff (encode) | m | b (scan decode x = m + b * code)
};

// ------------------------------------------------------------------------------------------
// GpuIndexCagra (faiss/gpu/GpuIndexCagra.h:41-380): a graph index built and searched on the device
// ------------------------------------------------------------------------------------------
enum class graph_build_algo { IVF_PQ = 0, NN_DESCENT = 1, ITERATIVE_SEARCH = 2 }; // only IVF_PQ is implemented
enum class codebook_gen { PER_SUBSPACE = 0, PER_CLUSTER = 1 };                   // only PER_SUBSPACE is implemented
enum class search_algo { SINGLE_CTA = 0, MULTI_CTA = 1, MULTI_KERNEL = 2, AUTO = 100 }; // AUTO runs SINGLE_CTA
enum class hash_mode { HASH = 0, SMALL = 1, AUTO = 100 }; // accepted; the visited set is always in shared memory

struct IVFPQBuildCagraConfig {
    uint32_t n_lists = 1024;               // clamped so that k-means gets >= 39 training rows per list
    uint32_t kmeans_n_iters = 20;
    double kmeans_trainset_fraction = 0.5; // the k-means and PQ training subsample
    uint32_t pq_bits = 8;                  // any width GpuIndexIVFPQ takes (4, 5, 6 with its interleaved layout)
    uint32_t pq_dim = 0;                   // 0: the largest divisor of d that is <= min(32, d / 2)
    codebook_gen codebook_kind = codebook_gen::PER_SUBSPACE;
    bool force_random_rotation = false;    // must stay false
    bool conservative_memory_allocation = false; // accepted, no effect
};

struct IVFPQSearchCagraConfig {
    uint32_t n_probes = 20;
    int lut_dtype = 0;                     // accepted, no effect (the LUT is fp32)
    int internal_distance_dtype = 0;       // accepted, no effect
    double preferred_shmem_carveout = 1.0; // accepted, no effect
    uint32_t max_internal_batch_size = 4096; // rows per candidate self-search page
};

struct GpuIndexCagraConfig : GpuIndexConfig {
    size_t intermediate_graph_degree = 128; // K0, clamped to N - 1
    size_t graph_degree = 64;               // K, clamped to K0
    graph_build_algo build_algo = graph_build_algo::IVF_PQ;
    size_t nn_descent_niter = 20;           // NN_DESCENT is not implemented
    IVFPQBuildCagraConfig ivf_pq_params;
    IVFPQSearchCagraConfig ivf_pq_search_params;
    float refine_rate = 2.0f;               // >= 1
    bool store_dataset = true;              // must stay true: the search reads the stored rows
    bool guarantee_connectivity = false;    // must stay false
};

struct SearchParametersCagra : SearchParameters {
    size_t max_queries = 0;     // queries per launch; 0: the whole page
    size_t itopk_size = 64;     // rounded up to a multiple of 32; <= 512 and >= k
    size_t max_iterations = 0;  // 0: 2 * itopk / search_width + 16 (itopk rounded)
    search_algo algo = search_algo::AUTO;
    size_t team_size = 0;       // lanes per distance: 4, 8, 16, 32; 0: by d
    size_t search_width = 1;
    size_t min_iterations = 0;
    size_t thread_block_size = 0; // 64 ... 1024; 0: by itopk
    hash_mode hashmap_mode = hash_mode::AUTO;
    size_t hashmap_min_bitlen = 0;
    float hashmap_max_fill_rate = 0.5f;
    uint32_t num_random_samplings = 1;
    uint64_t seed = 0x128394;
};

class GpuIndexCagra : public GpuIndex {
   public:
    GpuIndexCagra(
            std::shared_ptr<GpuResources> resources,
            int dims,
            MetricType metric = METRIC_L2,
            GpuIndexCagraConfig config = GpuIndexCagraConfig());

    // train builds the graph over x (the index stores x as its dataset); add calls train.  Either does nothing on a
    // built index.
    void train(idx_t n, const float* x) override;
    void add(idx_t n, const float* x) override;
    void reset() override;
    // IndexHNSWCagra payload: xb [n][d] and the level-0 table [n][degree]; -1 entries are skipped by the search
    void copyFrom(idx_t n, const float* xb, const idx_t* graph, int degree);
    void copyTo(float* xb, idx_t* graph) const; // xb [ntotal][d], graph [ntotal][graph degree] (host or device)
    std::vector<idx_t> get_knngraph() const;
    int graphDegree() const {
        return graphDegree_;
    }
    // distance evaluations of the last search, summed over all its queries
    mutable int64_t lastSearchDistanceCount = 0;
    // seconds spent in the last build: IVF-PQ candidates, refine, optimise
    double lastBuildSeconds[3] = {0, 0, 0};

   protected:
    bool addImplRequiresIDs_() const override {
        return false;
    }
    void addImpl_(idx_t n, const float* xDev, const idx_t* idsDev) override;
    void searchImpl_(idx_t n, const float* xDev, int k, float* dDev, idx_t* iDev) const override;
    GpuMemoryReservation selMask_(const IDSelector& sel) const override; // throws: no filtered graph search

    GpuIndexCagraConfig cagraConfig_;
    int graphDegree_ = 0;
    DeviceVector<float> data_;     // [ntotal][d]
    DeviceVector<uint32_t> graph_; // [ntotal][graphDegree_]; 0xFFFFFFFF = no edge
};

// the GpuIndexCagra build pipeline (cagra_build.cu): IVF-PQ candidates, refine, optimise into graph [n][K];
// seconds[] = the time of the three stages
void cagraBuildGraph(
        std::shared_ptr<GpuResources> res, int device, const float* xDev, idx_t n, int d, MetricType metric,
        const GpuIndexCagraConfig& cfg, int K0, int K, DeviceVector<uint32_t>& graph, double seconds[3]);

// fvecs_maybe_subsample (faiss/utils/utils.cpp:464-489) on a device matrix: when n > nmax, the rows
// rand_perm(n, seed)[0:nmax] are gathered into `hold` and n becomes nmax; returns the rows to use
const float* subsampleRowsDevice(
        GpuResources* res, int device, idx_t& n, int d, idx_t nmax, int64_t seed, const float* xDev,
        GpuMemoryReservation& hold, cudaStream_t stream);

// ------------------------------------------------------------------------------------------
// IndexShards
// ------------------------------------------------------------------------------------------
class DistributedIndexShards;

class IndexShards : public Index {
   public:
    explicit IndexShards(int d, bool threaded = false, bool successive_ids = true);
    ~IndexShards() override;
    bool own_indices = false;
    bool threaded;
    bool successive_ids;

    void add_shard(Index* idx);
    void remove_shard(Index* idx);
    int count() const {
        return (int)shards_.size();
    }
    Index* at(int i) {
        return shards_[i];
    }
    void train(idx_t n, const float* x) override;
    void add(idx_t n, const float* x) override;
    void add_with_ids(idx_t n, const float* x, const idx_t* xids) override;
    void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const override;
    void reset() override;
    void syncWithSubIndexes();
    // which path the last search took: 0 = thread-per-shard + host merge (the reference's), 1 = NCCL fast path
    mutable int lastSearchPath = 0;

   protected:
    template <typename F>
    void runOnIndex(F f) const;
    // fast path: every shard is a GpuIndex on its own device and the shards' resources hold one NCCL clique
    // over exactly those devices -> per-device threads + ncclAllGather + device merge (no host merge)
    bool ncclFastPath_(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const;
    std::vector<Index*> shards_;
    mutable std::vector<std::unique_ptr<DistributedIndexShards>> dist_; // one per device, built on first use
};

// faiss::IndexShardsIVF (faiss/IndexShardsIVF.h, IndexShardsIVF.cpp:100-251): shards are IVF indexes over ONE common
// coarse quantiser (GpuMultipleClonerOptions::common_ivf_quantizer, faiss/gpu/GpuCloner.cpp:418-436): the coarse search
// runs once, every shard scans its part of the probed lists through search_preassigned, results are merged.
class IndexShardsIVF : public IndexShards {
   public:
    IndexShardsIVF(GpuIndexFlat* quantizer, idx_t nlist, bool threaded = false, bool successive_ids = true);
    GpuIndexFlat* quantizer; // shared, not owned
    idx_t nlist;
    void add_shard(Index* idx); // must be a GpuIndexIVF with the same nlist
    void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const override;
};

// ------------------------------------------------------------------------------------------
// IndexShards across NCCL ranks: one shard (a GpuIndex) per rank of the resources' communicator for the
// shard's device.  Same semantics as faiss::IndexShards::search (faiss/IndexShards.cpp:197-264): every query
// goes to every shard, ids are translated by the number of vectors in lower-ranked shards when successive_ids,
// results are merged with the (distance, id) rule of merge_knn_results (faiss/utils/Heap.cpp:166-238) --
// but the exchange is ONE grouped ncclAllGather of the per-shard [n,k] blocks over NVLink and the merge a
// device kernel reading the gathered layout in place.  With Flat shards on the tensor-core path the ranks
// also pool their k-th-score thresholds after every round (one small all-reduce), so per-query work
// (candidate selection, exact re-rank) shrinks with the number of shards instead of being replicated.
// Used by: one process per GPU (every process holds one instance; search() is a collective call), and by
// IndexShards' in-process fast path (one instance per device, driven by one thread per device).
// ------------------------------------------------------------------------------------------
class DistributedIndexShards : public Index {
   public:
    DistributedIndexShards(std::shared_ptr<GpuResources> resources, GpuIndex* local, bool successive_ids = true);
    ~DistributedIndexShards() override;
    bool own_local = false;
    bool successive_ids;

    int rank() const;
    int worldSize() const;
    idx_t idOffset() const {
        return idOffset_;
    }
    GpuIndex* local() {
        return local_;
    }
    // collective: re-reads every shard's ntotal (call after adds)
    void syncWithSubIndexes();
    void train(idx_t n, const float* x) override;           // local shard trains on x
    void add(idx_t n, const float* x) override;              // adds x to the LOCAL shard, then syncWithSubIndexes()
    void add_with_ids(idx_t n, const float* x, const idx_t* xids) override;
    void reset() override;
    // collective; x / distances / labels host or device, identical x on every rank
    void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const override;
    // the collective itself; a rank that does not need the merged result (in-process fast path: only one
    // caller-visible output) skips the merge
    void searchCollective(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels, bool wantResult) const;
    idx_t shardSize(int r) const {
        return sizes_[r];
    }

   private:
    std::shared_ptr<GpuResources> resources_;
    GpuIndex* local_;
    std::shared_ptr<Communicator> comm_;
    std::vector<idx_t> sizes_;
    bool allFlatTc_ = false; // every rank's shard is a tensor-core-capable GpuIndexFlat
    idx_t idOffset_ = 0;
    int64_t maxTiles_ = 0;
    idx_t* dOffsets_ = nullptr; // device [world]
};

// host merge with the reference semantics (faiss/utils/Heap.cpp:166-238)
void merge_knn_results_host(
        idx_t n,
        idx_t k,
        int nshard,
        MetricType metric,
        const float* all_distances,
        const idx_t* all_labels,
        float* distances,
        idx_t* labels);

} // namespace fb200
