// faiss_b200 -- the tensor-core Flat search (flat_tc.cu) and the prepared database it scans.
#pragma once

#include <cuda_fp16.h>

#include "common.h"
#include "flat_tc_schedule.h"
#include "resources.h"

namespace fb200 {

// can the tensor-core path search a database of n rows of dimension d for k results?
bool flatTcSupported(int d, int k, int64_t n);

// Sharded search (one shard per NCCL rank): thresholds are pooled across the ranks after every round
// (one all-reduce of 2 floats per query), so a 1/S-size shard filters as tightly as the whole database would
// and keeps only its share of the global top-k; all ranks must call with the same queries and k.
class Communicator;
struct FlatTcShard {
    const Communicator* comm; // this rank
    int64_t maxTiles;         // max over ranks of ceil(n_r / 256): the common round schedule
};

// The database as the tensor-core search scans it (DESIGN.md 2): the scaled fp16 rows, under L2 sorted by norm (perm:
// stored position -> row id), the bias per stored row, the max / min bias per 256-row tile, the scale and the max norm.
// Rebuilt lazily by prepare() after invalidate(); DeviceVector::resize keeps the allocations, so an index whose rows
// are replaced in place (the k-means loop) re-prepares without reallocating.
class FlatTcDatabase {
   public:
    FlatTcDatabase(GpuResources* res, int device, int d);

    void invalidate() { // the rows changed: the next prepare() rebuilds
        dirty_ = true;
    }
    void clear(); // frees the prepared data
    // rebuilds from the n stored rows (fp32, or __half when yHalf) unless nothing changed since the last call.
    // The rows must stay in place until the next invalidate(): search() reads them.
    void prepare(const void* rows, int64_t n, MetricType metric, int yHalf, cudaStream_t stream);

    // Certified k-NN of nq queries Q [nq][d] (device) over the prepared rows: fp16 wgmma scoring + candidate
    // emission + exact fp32 re-rank, with the exact SIMT kernel as fallback for queries whose certificate fails.
    // shard: a sharded search (see FlatTcShard), or null.  rowMask: null, or [ceil(n/32)] words: only rows whose
    // bit is set can be returned.  outD / outI [nq][k].  Returns the number of queries recomputed exactly.
    int64_t search(const float* Q, int64_t nq, int k, float* outD, idx_t* outI, cudaStream_t stream,
                   const FlatTcShard* shard = nullptr, const uint32_t* rowMask = nullptr) const;

   private:
    // the launch steps of search(), in order
    struct Call;  // one search call
    struct Batch; // one query batch of it
    void prepareQueries(const Call& c, Batch& b) const;
    void runRound(const Call& c, const Batch& b, const tc::FlatTcRound& r, uint2* arena, int* counts, float* contrib,
                  float* outD, idx_t* outI) const;
    void rerank(const Call& c, const Batch& b, float* outD, idx_t* outI) const;
    int recomputeFallbacks(const Call& c, const Batch& b, const uint32_t* rowMask, float* outD, idx_t* outI) const;

    GpuResources* res_;
    int device_;
    int d_, dpad_;
    DeviceVector<__half> y16_;
    DeviceVector<float> bias_;
    DeviceVector<int> perm_; // L2 only
    DeviceVector<float> tileBias_;
    float scale_ = 1.f;
    float maxNorm_ = 0.f;
    bool dirty_ = true;
    // what the last prepare() was built from
    const void* rows_ = nullptr;
    int64_t n_ = 0;
    MetricType metric_ = METRIC_L2;
    int yHalf_ = 0;
};

// debug / unit-test seam: raw fp16 tensor-core score tile  S[nq,n] = Q16 . Y16^T  (fp32 out)
void runFlatTcScoresDebug(const __half* Q16, int64_t nq, const __half* Y16, int64_t n, int dpad, float* S, cudaStream_t stream);

} // namespace fb200
