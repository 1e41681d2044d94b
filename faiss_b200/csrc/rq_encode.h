// faiss_b200 -- GpuRqEncoder: ResidualQuantizer's beam-search encoding on the device
// (faiss/impl/ResidualQuantizer.cpp:432-520, faiss/impl/residual_quantizer_encode_steps.cpp).
//
// Both of the CPU's distance modes:
//   refineBeam     use_beam_LUT = 0: each step scores the beam's residuals against codebook m
//                  (‖r‖² + ‖c‖² − 2·⟨r, c⟩) and carries the residuals r − c;
//   refineBeamLUT  use_beam_LUT = 1: each step scores from the tables ‖c‖², x·Cᵀ and the codebook cross products,
//                  no residuals.
// Every row's search is independent of every other row's: results do not depend on paging, on pointer residency or
// on how n is split over calls.  Every pointer may be host or device memory.
#pragma once

#include <memory>
#include <vector>

#include "common.h"
#include "resources.h"

namespace fb200 {

// the per-page buffers (beams, residuals, inner-product tables, packed codes) stay within this budget
constexpr size_t kRqPageBytes = size_t(256) << 20;

// the largest beam (the WarpTopK list of one row holds it) and the largest nbits[m] (ids b·K + k < 2^20)
constexpr int kRqMaxBeam = 256;
constexpr int kRqMaxNbits = 12;

// AdditiveQuantizer::Search_type_t (faiss/impl/AdditiveQuantizer.h:71-86)
enum RqSearchType {
    RQ_ST_decompress = 0,
    RQ_ST_LUT_nonorm = 1,
    RQ_ST_norm_from_LUT = 2,
    RQ_ST_norm_float = 3,
    RQ_ST_norm_qint8 = 4,
    RQ_ST_norm_qint4 = 5,
    RQ_ST_norm_cqint8 = 6,
    RQ_ST_norm_cqint4 = 7,
    RQ_ST_norm_lsq2x4 = 8,
    RQ_ST_norm_rq2x4 = 9,
};

class GpuRqEncoder {
   public:
    // nbits[m] in [1, 12]; codebook m has K_m = 2^nbits[m] rows
    GpuRqEncoder(int d, std::vector<int> nbits, std::shared_ptr<GpuResources> res, int device);
    ~GpuRqEncoder();
    GpuRqEncoder(const GpuRqEncoder&) = delete;
    GpuRqEncoder& operator=(const GpuRqEncoder&) = delete;

    // codebooks [total_K][d] (host or device): a device copy, the centroid norms ‖c‖² and, per step m >= 1, the
    // cross-product block ⟨codebooks[0 : off_m], codebook m⟩ [off_m][K_m] (AdditiveQuantizer::compute_codebook_tables)
    void setCodebooks(const float* codebooks);

    // the beam size after all M steps from beamIn entries with out_beam_size outBeam
    int finalBeam(int beamIn, int outBeam) const;

    // ResidualQuantizer::refine_beam: residuals [n][beamIn][d] -> codes [n][B][M], residualsOut [n][B][d],
    // distances [n][B] with B = finalBeam(beamIn, outBeam); each output may be null
    void refineBeam(
            idx_t n,
            int beamIn,
            const float* residuals,
            int outBeam,
            int32_t* codes,
            float* residualsOut,
            float* distances,
            size_t pageBytes = kRqPageBytes) const;

    // ResidualQuantizer::refine_beam_LUT from x [n][d] instead of the CPU's (query_norms, query_cp): the device makes
    // ‖x‖² and x·Cᵀ itself.  codes [n][B][M], distances [n][B] with B = finalBeam(1, outBeam); each may be null
    void refineBeamLUT(
            idx_t n,
            const float* x,
            int outBeam,
            int32_t* codes,
            float* distances,
            size_t pageBytes = kRqPageBytes) const;

    // ResidualQuantizer::compute_codes_add_centroids: the beam search with out_beam_size maxBeam, entry 0 packed
    // LSB-first with nbits[m] bits per step, then encode_norm(norm) for the ST_norm_* types.  The norm is
    // ‖x − residual‖² in mode 0 without centroids, else ‖decode + centroids‖².  packed [n][codeSize(searchType)];
    // centroids [n][d] or null.  Search types ST_norm_cqint*, ST_norm_lsq2x4 and ST_norm_rq2x4 throw.
    void computeCodes(
            const float* x,
            idx_t n,
            bool useBeamLUT,
            int maxBeam,
            int searchType,
            float normMin,
            float normMax,
            const float* centroids,
            uint8_t* packed,
            size_t pageBytes = kRqPageBytes) const;

    // the same search with the codes left unpacked, codes [n][M] (entry 0 of the beam), for a caller that packs them
    // with a search type the device does not (the CPU computes those norms from the decoded codes)
    void encodeUnpacked(const float* x, idx_t n, bool useBeamLUT, int maxBeam, int32_t* codes, size_t pageBytes = kRqPageBytes) const;

    // bytes of one packed code: (Σ nbits + norm bits) / 8 rounded up
    size_t codeSize(int searchType) const;

    const int d, M;
    const std::vector<int> nbits;

   private:
    struct Pipeline;
    void checkReady() const;
    std::shared_ptr<GpuResources> res_;
    int device_;
    std::vector<int64_t> offsets_; // [M + 1] codebook_offsets
    int64_t totalK_ = 0;
    GpuMemoryReservation codebooks_; // [total_K][d]
    GpuMemoryReservation norms_;     // [total_K]
    GpuMemoryReservation cross_;     // the step blocks [off_m][K_m], m = 1 .. M-1, back to back
    GpuMemoryReservation meta_;      // int32 [M + 1] offsets on the device
    bool haveCodebooks_ = false;
};

} // namespace fb200
