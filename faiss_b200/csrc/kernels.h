// faiss_b200 -- launcher declarations for the device kernels (L1; the tensor-core Flat search: flat_tc.h).  Host code (index objects,
// C ABI) only sees these; all pointers are DEVICE pointers, all work is enqueued on `stream`.
#pragma once

#include <cuda_fp16.h>

#include "common.h"
#include "resources.h"

namespace fb200 {

// ---------------------------------------------------------------- flat_exact.cu
// ||x||^2 per row (role of runL2Norm, faiss/gpu/impl/L2Norm.cu:176)
void runL2Norms(const float* x, int64_t n, int d, float* norms, cudaStream_t stream);

// Exact fp32 brute-force k-NN (SIMT, direct-form sum (q-y)^2 / sum q*y accumulated in dimension
// order).  This is the always-correct path: small problems, odd dimensions, the fallback of the
// tensor-core path, and the canonical arithmetic the tensor-core re-rank reproduces.  It is also the
// only path of the other metrics (L1, Linf, Lp, Canberra, BrayCurtis, JensenShannon, Jaccard, Gower).
// Role of runDistance<float> / runGeneralDistance (faiss/gpu/impl/Distance.cu:121-405,
// Distance.cuh:223-289) with the k-select fused in.
//   Q [nq,d], Y [n,d] row-major; outD [nq,k], outI [nq,k] (int64, row index + idBase; -1 missing)
//   yHalf: Y holds __half rows (GpuIndexFlatConfig::useFloat16 storage), widened to fp32 on load
//   metricArg: the exponent p of METRIC_Lp (ignored by the other metrics)
//   rowMask: null, or [ceil(n/32)] words: only rows whose bit is set can be returned (SearchParameters::sel)
void runFlatExact(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        const void* Y,
        int64_t n,
        int d,
        int k,
        MetricType metric,
        int64_t idBase,
        float* outD,
        idx_t* outI,
        cudaStream_t stream,
        int yHalf = 0,
        float metricArg = 0.f,
        const uint32_t* rowMask = nullptr);

// k = 1 convenience (assignment): outI int64 [nq], outD optional
void runFlatArgmin(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        const float* Y,
        int64_t n,
        int d,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream);

// All-pairs distances with the arithmetic of runFlatExact (role of allPairwiseDistanceOnDevice,
// faiss/gpu/impl/Distance.cuh:167-292): D[i * ldD + j] = distance(Q[i], Y[j]) for i < nq, j < n, the value the
// k-NN path returns for that pair, bit for bit.  Inner product and Jaccard are the raw similarity; NaN is written
// as computed.  `metric` is what the kernel runs: METRIC_Lp with p = 1 / 2 is mapped by flatKernelMetric first.
void runFlatPairwise(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        const float* Y,
        int64_t n,
        int d,
        MetricType metric,
        float metricArg,
        float* D,
        int64_t ldD,
        cudaStream_t stream);

// the metric the exact kernel runs for (metric, metricArg): METRIC_Lp with p = 1 is L1 and with p = 2 is L2
// (faiss/gpu/impl/Distance.cuh:223-239); the reference GPU's p = -1 -> L2 branch is a test hook, and the CPU sums
// |a-b|^-1 there, as the Lp kernel does
inline MetricType flatKernelMetric(MetricType metric, float metricArg) {
    if (metric == METRIC_Lp && metricArg == 1.f)
        return METRIC_L1;
    if (metric == METRIC_Lp && metricArg == 2.f)
        return METRIC_L2;
    return metric;
}

// Row-wise top-k over candidate lists (role of runBlockSelectPair / merge_knn_results,
// faiss/gpu/utils/BlockSelectFloat.cu:98, faiss/utils/Heap.cpp:166-238).
//   inD/inI: [rows, nlists, kin]; ids == -1 are skipped (any other id, negative ones included, is a stored one);
//   idOffsets (optional, [nlists]) is added to
//   ids of list l (IndexShards successive_ids translation, faiss/IndexShards.cpp:214-220).
//   Keys are user-facing distances (larger is better for is_similarity_metric: IP, Jaccard).
void runMergeTopK(
        const float* inD,
        const idx_t* inI,
        int64_t rows,
        int nlists,
        int kin,
        const idx_t* idOffsets,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream);

// same merge over inputs laid out [nlists][rows][kin] (the layout an all-gather of per-shard results
// produces: no permute copy between the collective and the merge)
void runMergeTopKListMajor(
        const float* inD,
        const idx_t* inI,
        int64_t rows,
        int nlists,
        int kin,
        const idx_t* idOffsets,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream);

// runMergeTopK over inputs already in key space (smaller is better: IP distances negated), without id offsets;
// idBase is added to every id.  Merges the per-CTA partial results of the Flat and IVF scans: an entry is kept by the
// result rule on its key (isResult, select.cuh), whatever its id, so stored ids of -1 or INT64_MAX survive.
void runMergeTopKKeyspace(
        const float* inD,
        const idx_t* inI,
        int64_t rows,
        int nlists,
        int kin,
        int k,
        MetricType metric,
        int64_t idBase,
        float* outD,
        idx_t* outI,
        cudaStream_t stream);

// residual x - c[assign] (NaN if assign = -1) ; role of runCalcResidual (VectorResidual.cu:26-176)
void runCalcResidual(
        const float* x,
        const void* centroids,
        const idx_t* assign,
        int64_t n,
        int d,
        float* out,
        cudaStream_t stream,
        int yHalf = 0);
// gather rows by id (reconstruct_batch) / by range; id < 0 gives a NaN row, or all 0xFF bytes with missingAllOnes (a
// missing search result's reconstruction)
void runGatherRows(
        const void* src, const idx_t* ids, int64_t n, int d, float* out, cudaStream_t stream, int yHalf = 0,
        bool missingAllOnes = false);

// ---------------------------------------------------------------- kmeans.cu
// centroid update (role of compute_centroids, faiss/impl/ClusteringHelpers.cpp:101-172):
// sums[c] += x_i for assign[i]=c, counts[c] += 1 ; then centroids = sums / counts
void runKmeansAccumulate(
        const float* x,
        const idx_t* assign,
        int64_t n,
        int d,
        int64_t k,
        float* sums /*[k,d] zeroed*/,
        float* counts /*[k] zeroed*/,
        cudaStream_t stream);
void runKmeansFinalize(
        const float* sums,
        const float* counts,
        int64_t k,
        int d,
        float* centroids /* in: previous, out: new (unchanged where count==0) */,
        cudaStream_t stream);

// post_process_centroids (faiss/Clustering.cpp:35-45): spherical renormalisation and/or rounding to integers
void runKmeansPostProcess(float* centroids, int64_t k, int d, bool spherical, bool intCentroids, cudaStream_t stream);

// ---------------------------------------------------------------- ivf.cu
// PQ encode: codes[i][m] = argmin_c || r_i[m*dsub:(m+1)*dsub] - pq[m][c] ||^2
//   (role of IVFPQ::appendVectors_ per-subquantizer k=1 search, faiss/gpu/impl/IVFPQ.cu:129-257;
//    arithmetic follows faiss/impl/ProductQuantizer.cpp compute_code: direct L2, first min wins)
void runPQEncode(
        const float* resid,
        int64_t n,
        int d,
        int M,
        int ksub,
        const float* pqCentroids /*[M][ksub][dsub]*/,
        uint8_t* codes /*[n][M]*/,
        cudaStream_t stream);
// codes [n][M] (one byte each, < 2^nbits) -> packed [n][ceil(M*nbits/8)], the CPU's LSB-first bitstring
// (PQEncoderGeneric, faiss/impl/ProductQuantizer-inl.h)
void runPQPack(const uint8_t* codes, int64_t n, int M, int nbits, uint8_t* packed, cudaStream_t stream);

// histogram of list assignments + stable scatter positions (device-side append bookkeeping;
// replaces the host unordered_map pass of IVFBase::addVectorsToLists_, IVFBase.cu:693-905)
void runIvfCountAssign(const idx_t* assign, int64_t n, int64_t nlist, int* counts /*[nlist] += */, cudaStream_t stream);
// offsets[i] = position of vector i inside its list (listLen[assign[i]] before this batch + rank of
// i among batch vectors with the same list, in batch order)
void runIvfAppendOffsets(
        const idx_t* assign,
        int64_t n,
        int64_t nlist,
        const int* listLenBefore /*[nlist]*/,
        int* offsets /*[n]*/,
        int* scratch /*[nlist]*/,
        cudaStream_t stream);
// scatter rows (codeSize bytes each) + ids to list storage: dst = base + listStart[l]*codeSize
void runIvfScatter(
        const uint8_t* rows,
        const idx_t* ids,
        const idx_t* assign,
        const int* offsets,
        int64_t n,
        int codeSize,
        const int64_t* listStart /*[nlist] element offset of each list in the arena*/,
        uint8_t* arenaCodes,
        idx_t* arenaIds,
        cudaStream_t stream);

// ---------------------------------------------------------------- ivf_reconstruct.cu
// What a decoder needs to know about an IVF index's stored lists (all pointers on the device).  Every entry is
// addressed by its arena slot; lists start in ascending list order, so a slot's list is found by bisection.
enum IvfStoredKind { IVF_STORED_FLAT = 0, IVF_STORED_SQ = 1, IVF_STORED_PQ = 2 };
struct IvfStoredLayout {
    int kind = IVF_STORED_FLAT;
    int d = 0;
    int codeSize = 0;         // bytes of one CPU code (fp32 row for IVF-Flat)
    bool interleaved = false; // codes in the interleaved-by-32 layout (8-bit PQ, M in {16, 32}; 4-bit nibble pairs)
    const int64_t* listStart = nullptr;
    const int* listLen = nullptr;
    int64_t nlist = 0;
    int64_t arenaElems = 0;
    const uint8_t* codes = nullptr;
    const idx_t* ids = nullptr;
    const float* centroids = nullptr; // coarse centroid added to every decoded entry of its list, or null
    // SQ: codec of ivf_layout.cuh, decode x = vmin + (c + 0.5) / levels * vdiff per dimension; levels 0: x = c
    int sqCodec = 0;
    float levels = 0.f;
    const float* vmin = nullptr;
    const float* vdiff = nullptr;
    // PQ: codebooks [M][2^nbits][d / M], codes LSB-first bitstrings
    int M = 0, nbits = 8;
    const float* pq = nullptr;
};
// What the list scans read: the stored layout and the tables only the scans use.  They stay out of IvfStoredLayout,
// which the decoder kernels take by value.
struct IvfScanLayout : IvfStoredLayout {
    const float* pqT = nullptr;   // PQ: the codebooks transposed to [2^nbits][M][d / M] (interleaved scan)
    const float* term2 = nullptr; // PQ: the precomputed L2 table [nlist][256][M] of the interleaved 8-bit scan, or null
    const float* sqDecodeMB = nullptr; // SQ: the scan's folded decode x = m + b * c, m[d] | b[d]
};

// out[i] = i: a table of arena slots the list scans read as their id table, so that they return positions
void runIvfIdentitySlots(idx_t* out, int64_t n, cudaStream_t stream);
// runMergeTopKKeyspace over partial results holding arena positions: each position becomes its stored id on the way in
// (same keys, ids and tie order as the plain merge) and is returned in outSlot beside it (-1 with the id -1)
void runIvfMergeTopKSlots(
        const float* inD,
        const idx_t* inPos,
        const idx_t* arenaIds,
        int64_t rows,
        int nlists,
        int kin,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        idx_t* outSlot,
        cudaStream_t stream);
// slots[id - i0] = the largest arena slot storing id, for i0 <= id < i0 + ni; -1 where no entry has that id
void runIvfSlotsOfRange(const IvfStoredLayout& a, idx_t i0, idx_t ni, idx_t* slots, cudaStream_t stream);
// slots[i] = the largest arena slot storing keys[i], or -1; returns false when some key is not stored (synchronises)
bool runIvfSlotsOfKeys(
        GpuResources* res, int device, const IvfStoredLayout& a, const idx_t* keys, int64_t n, idx_t* slots, cudaStream_t stream);
// out[i] = the CPU's reconstruct_from_offset of the entry at slots[i]; slot -1: all 0xFF bytes (fillMissing) or untouched
void runIvfReconstruct(const IvfStoredLayout& a, const idx_t* slots, int64_t n, bool fillMissing, float* out, cudaStream_t stream);
// out[i] = [listno, listnoBytes little-endian bytes][the CPU code bytes] of the entry at slots[i]; slot -1: all 0xFF
void runIvfGatherCodes(const IvfStoredLayout& a, const idx_t* slots, int64_t n, int listnoBytes, uint8_t* out, cudaStream_t stream);

// the slot-keeping variant of a list scan: the scan is handed `identity` as its id table, so its partial results hold
// arena positions, and runIvfScanBatches merges them with runIvfMergeTopKSlots against the real ids
struct IvfSlotOutput {
    const idx_t* identity;
    const idx_t* arenaIds;
    idx_t* outSlot; // [nq][k], beside outD / outI
};

// ---------------------------------------------------------------- ivf.cu: the list scans
// One scan call (device pointers): queries Q [nq][d], their probes [nq][nprobe] (list ids, -1 = skip) and coarse
// distances [nq][nprobe], results outD / outI [nq][k].
struct IvfScanCall {
    const float* Q = nullptr;
    int64_t nq = 0;
    const idx_t* probes = nullptr;
    const float* coarseDis = nullptr;
    int nprobe = 0;
    int k = 0;
    MetricType metric = METRIC_L2;
    float* outD = nullptr;
    idx_t* outI = nullptr;
    cudaStream_t stream = nullptr;
    const uint32_t* mask = nullptr;       // SearchParameters::sel over the arena, or null
    const IvfSlotOutput* slots = nullptr; // the slot-keeping search, or null
};

// Scans the probed lists of `lists` and keeps the top k per query, with the scan of the lists' format:
//   IVF-Flat: fp32 rows (role of runIVFInterleavedScan, faiss/gpu/impl/IVFInterleaved.cu:179);
//   IVF-SQ: the decode folded into per-(query, probe) tables (role of the reference GPU IVFFlatScan with a
//     scalar-quantiser codec); distance forms of faiss/impl/scalar_quantizer/scanners.h:44-135: L2 on the residual
//     q - c_list when the lists hold residuals (centroids set), IP adds the coarse distance then;
//   IVF-PQ: the per-(query, list) LUT built in shared memory, codes streamed, the running top-k on chip (role of
//     runPQScanMultiPassNoPrecomputed + pqCodeDistances, PQScanMultiPassNoPrecomputed-inl.cuh:527,
//     PQCodeDistances-inl.cuh:591), distance form of the CPU scanner (IVFPQ_QueryTables.cpp:126-192): L2
//     sum_m || (q - c_list)_m - pq[m][code_m] ||^2, IP q.c_list + sum_m q_m . pq[m][code_m].  The interleaved layout
//     has its own scan (ivfpq_scan.cu), vector-major codes (8-bit, or packed below 8 bits) the other.
// Kernel timing names: ivfflat_scan, ivfsq_scan, ivfpq_scan, ivfpq_scan_packed (vector-major, nbits < 8).
void runIvfScan(GpuResources* res, int device, const IvfScanLayout& lists, const IvfScanCall& call);

// ---------------------------------------------------------------- ivfsq_scan.cu
// ScalarQuantizer::QuantizerType values (faiss/impl/ScalarQuantizer.h:27-34) the GPU index accepts
enum SqQuantizerType {
    SQ_QT_8bit = 0,
    SQ_QT_4bit = 1,
    SQ_QT_8bit_uniform = 2,
    SQ_QT_4bit_uniform = 3,
    SQ_QT_fp16 = 4,
    SQ_QT_8bit_direct = 5,
    SQ_QT_6bit = 6,
};

// per-dimension min / max over n rows (RS_minmax, faiss/impl/scalar_quantizer/training.cpp:209-383); outputs
// are device arrays [d]
void runSqMinMax(const float* x, int64_t n, int d, float* vminOut, float* vmaxOut, cudaStream_t stream);

// ScalarQuantizer encode (quantizers.h:66-150, codecs.h): codes [n][codeSize], byte-exact with the CPU.
// vmin / vdiff are per dimension (uniform types: the one range repeated); unused for fp16 / 8bit_direct.
void runSqEncode(
        const float* x,
        int64_t n,
        int d,
        int qtype,
        int codeSize,
        const float* vmin,
        const float* vdiff,
        uint8_t* codes,
        cudaStream_t stream);

// shared-memory bytes of the per-(query, probe) decode tables of the IVF-SQ scan
size_t ivfSqScanTableBytes(int d);

// ---- "rotated, interleaved-by-32" PQ code layout (native storage for M % 16 == 0, M <= 32) ----
// List-relative vector v = 32*g + t is stored in group g; byte position j of the vector holds
// code[(j + t) % M] and lives at  g*32*M + (j/16)*512 + t*16 + (j%16).  A warp therefore loads a
// group with fully coalesced 128-bit loads (512 B per instruction), and at step j lane t needs the
// LUT entry of sub-quantiser (j + t) % M: with the LUT laid out [code][slot] (slot = sub-quantiser,
// duplicated up to 64 slots = 256 B per code) lane t reads bank (t + j) % 32 -- conflict-free by
// construction.  copyTo / getListVectorData undo the permutation, so the external format stays the
// CPU ArrayInvertedLists byte layout.
inline bool ivfPqInterleavedSupported(int M) {
    return (M == 16 || M == 32);
}
// flat [n][M] codes -> arena (append): position = listStart[assign[i]] + offsets[i]
void runIvfPqScatterInterleaved(
        const uint8_t* codesFlat,
        const idx_t* ids,
        const idx_t* assign,
        const int* offsets,
        int64_t n,
        int M,
        const int64_t* listStart,
        uint8_t* arenaCodes,
        idx_t* arenaIds,
        cudaStream_t stream);
// one list: flat [len][M] <-> interleaved bytes at `listCodes` (arena + listStart*M)
void runIvfPqListToInterleaved(const uint8_t* flat, int64_t len, int M, uint8_t* listCodes, cudaStream_t stream);
void runIvfPqListFromInterleaved(const uint8_t* listCodes, int64_t len, int M, uint8_t* flat, cudaStream_t stream);

// T2[l][c][m] = ||y_{m,c}||^2 + 2 <centroid_l restricted to sub-space m, y_{m,c}>   (pqT = [256][M][dsub])
void runIvfPqPrecomputeTerm2(
        const float* coarse, const float* pqT, int64_t nlist, int d, int M, float* term2, cudaStream_t stream);

// ---------------------------------------------------------------- cagra_build.cu
// G0[rows[i]] for a batch of rows: the exact fp32 distances of each row's cand [nb][nc] (IVF-PQ ids; -1 skipped), the
// row itself dropped, the best K0 kept by (distance, id) (IP: larger first).  G0 entries past a row's valid candidates
// are 0xFFFFFFFF; valid[i] = the number of valid entries written (<= K0).  nc <= 2048.
void runCagraRefine(
        const float* data, int64_t n, int d, MetricType metric, int64_t row0, int64_t nb, const idx_t* cand, int nc,
        int K0, uint32_t* G0, int* valid, cudaStream_t stream);

// the graph optimisation (DESIGN "GpuIndexCagra"): G0 [n][K0] -> G [n][K] (detour-count prune, reverse edges, merge).
// Every G0 entry must be a row id other than its own row, and no row may hold an id twice.  K <= K0 <= 1024.
void runCagraOptimize(GpuResources* res, int device, const uint32_t* G0, int64_t n, int K0, int K, uint32_t* G, cudaStream_t stream);
// throws when a G0 entry is >= n (a -1 read as uint32) or equals its own row: the checks of b200_cagra_optimize,
// whose caller's G0 comes from outside the build (synchronises the stream; writes nothing of the caller's)
void checkCagraG0(GpuResources* res, int device, const uint32_t* G0, int64_t n, int K0, cudaStream_t stream);

// ---------------------------------------------------------------- cagra_search.cu
// one single-CTA CAGRA search launch over nq queries (device pointers); see cagra_search.cu for the kernel layout
struct CagraSearchArgs {
    const float* queries;  // [nq][d]
    int64_t nq;
    int64_t rowOffset;    // the row of queries[0] in the whole search call (the random entry ids depend on it)
    const float* data;    // [n][d]
    const uint32_t* graph; // [n][graphDegree]; entries >= n (copyFrom's -1) are skipped
    int64_t n;
    int d;
    int graphDegree;
    MetricType metric;    // METRIC_L2 or METRIC_INNER_PRODUCT
    int k;
    int itopk;            // internal top-k (a multiple of 32, <= 512)
    int bufSize;          // next power of two >= itopk
    int searchWidth;
    int candSize;         // next power of two >= max(numInit, searchWidth * graphDegree)
    int numInit;          // num_random_samplings * searchWidth * graphDegree
    int maxIterations;
    int teamSize;         // 4, 8, 16 or 32 lanes per distance
    int blockSize;
    int hashBits;
    int hashLimit;        // insertions allowed before the visited set is refilled from itopk
    uint64_t seed;
    float* outD;          // [nq][k]
    idx_t* outI;          // [nq][k]
    unsigned long long* distanceCount; // += distances computed
};
size_t cagraSearchSmemBytes(const CagraSearchArgs& a);
void runCagraSearch(const CagraSearchArgs& a, cudaStream_t stream);

} // namespace fb200
