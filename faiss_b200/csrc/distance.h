// faiss_b200 -- brute-force distances on externally provided memory: bfKnn, bfKnn_tiling and the all-pairs matrix
// (faiss/gpu/GpuDistance.h:18-181, GpuDistance.cu:61-570).
//
// Every distance is the canonical one of this library (flat_exact.cu): the direct-form chain in dimension order.
// k > 0 runs a transient GpuIndexFlat, so results equal GpuIndexFlat::search bit for bit.  k = -1 writes the full
// [numQueries, numVectors] matrix with the exact kernel (runFlatPairwise): entry [i, I[i][j]] equals the k-NN
// distance D[i][j].  Inputs may be fp32, fp16 or bf16 (widened exactly to fp32 on the device), row- or
// column-major, host or device resident.
#pragma once

#include <memory>

#include "common.h"
#include "resources.h"

namespace fb200 {

// same values as the reference's enums (faiss/gpu/GpuDistance.h:18-29)
enum class DistanceDataType : int { F32 = 1, F16, BF16 };
enum class IndicesDataType : int { I64 = 1, I32 };

// faiss::gpu::GpuDistanceParams (faiss/gpu/GpuDistance.h:32-152) without vectorNorms, ignoreOutDistances and use_cuvs;
// device must be a device ordinal (no -1)
struct GpuDistanceParams {
    MetricType metric = METRIC_L2;
    float metricArg = 0;
    int k = 0; // -1: all pairwise distances, outDistances is [numQueries, numVectors]
    int dims = 0;
    const void* vectors = nullptr; // vectorsRowMajor ? [numVectors][dims] : [dims][numVectors]
    DistanceDataType vectorType = DistanceDataType::F32;
    bool vectorsRowMajor = true;
    idx_t numVectors = 0;
    const void* queries = nullptr; // queriesRowMajor ? [numQueries][dims] : [dims][numQueries]
    DistanceDataType queryType = DistanceDataType::F32;
    bool queriesRowMajor = true;
    idx_t numQueries = 0;
    float* outDistances = nullptr;
    IndicesDataType outIndicesType = IndicesDataType::I64;
    void* outIndices = nullptr; // [numQueries][k]; unused for k = -1
    int device = 0;
};

// A host-resident all-pairs matrix is computed in blocks of at most this many bytes (the role kSearchPageBytes has
// for query pages), double-buffered on the device.
constexpr size_t kPairwisePageBytes = size_t(256) << 20;

// throws on any invalid argument, before any CUDA call
void validateDistanceParams(const GpuDistanceParams& args);

// faiss::gpu::bfKnn.  pairwisePageBytes: the block budget of a host-resident k = -1 output (tests lower it).
void bfKnn(const std::shared_ptr<GpuResources>& res, const GpuDistanceParams& args, size_t pairwisePageBytes = kPairwisePageBytes);

// faiss::gpu::bfKnn_tiling (faiss/gpu/GpuDistance.cu:457-570): host-resident row-major inputs cut into shards of at
// most vectorsMemoryLimit / queriesMemoryLimit bytes (0: no limit); vector shards are merged on the device in id
// order, so the result equals bfKnn's bit for bit
void bfKnn_tiling(
        const std::shared_ptr<GpuResources>& res,
        const GpuDistanceParams& args,
        size_t vectorsMemoryLimit,
        size_t queriesMemoryLimit);

} // namespace fb200
