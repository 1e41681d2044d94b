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

// The database as the tensor-core search scans it (DESIGN.md 2), in one or both of two layouts:
//   fp16: the scaled fp16 rows, under L2 sorted by norm (perm: stored position -> row id), the bias per stored row, the
//         max / min bias per 256-row tile, the scale and the max norm;
//   int8 (L2, 112 < d <= 128): the rows centred on the per-dimension midrange c and quantised with one scale s_y,
//         128 s8 per row, sorted by the centred norm, with their own perm, bias = -|y - c|^2 / 2 and tile bias, and
//         the database constants of the int8 certificate.
// Each layout is built on the first search that needs it after invalidate(); DeviceVector::resize keeps the
// allocations, so an index whose rows are replaced in place (the k-means loop) re-prepares without reallocating.
class FlatTcDatabase {
   public:
    FlatTcDatabase(GpuResources* res, int device, int d);

    void invalidate() { // the rows changed: the next prepare() rebuilds
        dirty_ = true;
    }
    void clear(); // frees the prepared data
    // takes the n stored rows (fp32, or __half when yHalf) as the source of the layouts unless nothing changed since
    // the last call.  The rows must stay in place until the next invalidate(): search() reads them.
    void prepare(const void* rows, int64_t n, MetricType metric, int yHalf, cudaStream_t stream);

    // Certified k-NN of nq queries Q [nq][d] (device) over the prepared rows: fp16 wgmma scoring + candidate
    // emission + exact fp32 re-rank, with the exact SIMT kernel as fallback for queries whose certificate fails.
    // shard: a sharded search (see FlatTcShard), or null.  rowMask: null, or [ceil(n/32)] words: only rows whose
    // bit is set can be returned.  outD / outI [nq][k].  Returns the number of queries recomputed exactly.
    // An unsharded L2 search with 112 < d <= 128 and 2 <= k <= 128 scores on the int8 tensor cores when the database
    // passes the int8 fitness test (prepareInt8); every other search scores in fp16.
    int64_t search(const float* Q, int64_t nq, int k, float* outD, idx_t* outI, cudaStream_t stream,
                   const FlatTcShard* shard = nullptr, const uint32_t* rowMask = nullptr);
    // operand width of the last search's scoring: 8 or 16
    int lastOperandBits() const {
        return lastBits_;
    }

   private:
    // the launch steps of search(), in order
    struct Call;  // one search call
    struct Batch; // one query batch of it
    void prepareQueries(const Call& c, Batch& b) const;
    void runRound(const Call& c, const Batch& b, const tc::FlatTcRound& r, uint2* arena, int* counts, float* contrib,
                  float* outD, idx_t* outI) const;
    void rerank(const Call& c, const Batch& b, float* outD, idx_t* outI) const;
    int recomputeFallbacks(const Call& c, const Batch& b, const uint32_t* rowMask, float* outD, idx_t* outI) const;
    void prepareFp16(cudaStream_t stream);
    void prepareInt8(cudaStream_t stream);
    bool int8Eligible(int k, const FlatTcShard* shard) const;

    GpuResources* res_;
    int device_;
    int d_, dpad_;
    // fp16 layout
    DeviceVector<__half> y16_;
    DeviceVector<float> bias_;
    DeviceVector<int> perm_; // L2 only
    DeviceVector<float> tileBias_;
    float scale_ = 1.f;
    float maxNorm_ = 0.f;
    // int8 layout
    DeviceVector<int8_t> y8_;
    DeviceVector<float> bias8_;
    DeviceVector<int> perm8_;
    DeviceVector<float> tileBias8_;
    DeviceVector<float> center_; // [d]
    float scale8_ = 1.f;         // s_y
    float maxYhat_ = 0.f;        // max |Y8 / s_y|, x 1.0001
    float maxRy_ = 0.f;          // max |(y - c) - Y8 / s_y|, x 1.0001
    float maxYc_ = 0.f;          // max |y - c|, x 1.0001
    bool int8Fit_ = false;       // the int8 certificate is tight enough on this database (prepareInt8)
    bool dirty_ = true;
    bool fp16Ready_ = false, int8Ready_ = false;
    int lastBits_ = 16;
    // what the last prepare() was built from
    const void* rows_ = nullptr;
    int64_t n_ = 0;
    MetricType metric_ = METRIC_L2;
    int yHalf_ = 0;
};

// debug / unit-test seam: raw tensor-core score tile  S[nq,n] = Q . Y^T  (fp32 out).  s8: Q and Y are int8 rows of
// dpad = 128 and S holds the exact int32 dot products; otherwise they are fp16 rows.
void runFlatTcScoresDebug(const void* Q, int64_t nq, const void* Y, int64_t n, int dpad, bool s8, float* S,
                          cudaStream_t stream);

} // namespace fb200
