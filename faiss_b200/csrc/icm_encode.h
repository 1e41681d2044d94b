// faiss_b200 -- GpuIcmEncoder: LocalSearchQuantizer's ICM encoding on the device
// (faiss/gpu/GpuIcmEncoder.h, faiss/impl/LocalSearchQuantizer.cpp:539-795).
//
// encode() runs lsq::IcmEncoder::encode's iterated local search with the perturbation draws given by the caller, so a
// caller that draws them from its std::mt19937 in the CPU's order (m, then k, per row and per perturbation) walks the
// CPU's random trajectory.  With the draws fixed, every row's run is independent of every other row: results do not
// depend on paging, on pointer residency or on how rows are split over devices.
#pragma once

#include <memory>
#include <vector>

#include "common.h"
#include "resources.h"

namespace fb200 {

// The [rows, M*K] inner-product table of one page, plus the page's rows, codes and draws, stay within this budget
// (the role the CPU's LocalSearchQuantizer::chunk_size plays for its [M, n, K] unary table).
constexpr size_t kIcmPageBytes = size_t(256) << 20;

// the largest codebook size the kernel takes: obj[K] lives in registers, K / 32 floats per lane
constexpr int kIcmMaxK = 1024;

class GpuIcmEncoder {
   public:
    // one (resources, device) pair per shard; rows are split into contiguous ranges over them
    GpuIcmEncoder(
            int M,
            int K,
            int d,
            std::vector<std::shared_ptr<GpuResources>> res,
            std::vector<int> devices);
    ~GpuIcmEncoder();
    GpuIcmEncoder(const GpuIcmEncoder&) = delete;
    GpuIcmEncoder& operator=(const GpuIcmEncoder&) = delete;

    // codebooks [M][K][d] (host or device): copied to every device, with their squared norms and the inner products
    // C·Cᵀ [M*K][M*K] from which the binary terms 2·<C_m2[k2], C_m[k]> are read
    void setBinaryTerm(const float* codebooks);

    // codes [n][M] int32 (in: the starting codes, out: the best codes), x [n][d], perturbations
    // [ils_iters][n][nperts] pairs (m, k) as int32; each pointer host or device
    void encode(
            int32_t* codes,
            const float* x,
            idx_t n,
            size_t ils_iters,
            size_t nperts,
            size_t icm_iters,
            const int32_t* perturbations,
            size_t pageBytes = kIcmPageBytes) const;

    const int M, K, d;

   private:
    struct Shard;
    void encodeShard(
            Shard& s,
            int32_t* codes,
            const float* x,
            idx_t n,
            idx_t i0,
            idx_t ni,
            size_t ils_iters,
            size_t nperts,
            size_t icm_iters,
            const int32_t* perturbations,
            size_t pageBytes) const;
    std::vector<std::unique_ptr<Shard>> shards_;
    bool haveBinaryTerm_ = false;
};

} // namespace fb200
