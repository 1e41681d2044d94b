// faiss_b200 -- GpuRqEncoder: ResidualQuantizer's beam search on the device (faiss/impl/ResidualQuantizer.cpp:432-520,
// faiss/impl/residual_quantizer_encode_steps.cpp:46-185, 348-442, 450-793).
//
// Three kernels, one warp per row in each:
//   rq_beam_step_kernel  one step of use_beam_LUT = 0 (beam_search_encode_step without assign_index).  It reads the
//                        [page·B_in, K] inner products runFlatPairwise(METRIC_INNER_PRODUCT) wrote for the residuals
//                        against codebook m and the residual norms of runL2Norms, scores (‖r‖² + ‖c‖²) + (−2·ip) with
//                        one rounding per operation (pairwise_L2sqr's norms, then the sgemm with beta = 1), keeps the
//                        B_out best and writes the children's codes, residuals r − c and distances.
//   rq_beam_lut_kernel   all M steps of use_beam_LUT = 1 (beam_search_encode_step_tab) in one launch.  The parent and
//                        child beams (int16 codes, distances) stay in shared memory; each candidate is scored from the
//                        L2-resident cross-product table as it is generated, so no candidate matrix reaches HBM.
//   rq_pack_kernel       AdditiveQuantizer::pack_codes for entry 0 of the beam, with encode_norm for the ST_norm_*
//                        types and the norm computed where the CPU computes it.
//
// Selection: WarpTopK<int> (select.cuh) over the ids j = b·K + k orders by (value asc, j asc), which is what the CPU's
// heap_addn + heap_reorder with CMax<float, int> keep: the B_out smallest by (value, j).
//
// Mode 1's candidate value, in the order of the reference's AVX2 build (rq_beam_search_tab-inl.h), with
// cd[k] = ‖c_k‖² − 2·qcp[k] and dp = Σ_{m1<m} cross_m[(off[m1] + code_b[m1])·K + k] summed in m1 order, by chunks of 8
// added one after another past m = 8:
//   m = 0                   dist_b + cd[k]
//   1 <= m <= 7, K >= 32    (cd[k] + 2·dp) + dist_b          (accum_and_finalize_tab's fmadd; 2·dp is exact)
//   otherwise               (dist_b + cd[k]) + 2·dp
#include <math_constants.h>

#include <algorithm>
#include <climits>

#include "index.h"
#include "kernels.h"
#include "rq_encode.h"
#include "select.cuh"

namespace fb200 {

namespace {

constexpr int kRqWarps = 4; // rows per CTA
constexpr int kRqBuf = 128; // WarpTopK pending buffer
constexpr size_t kRqSmemLimit = 227 * 1024;

int topkList(int k) {
    return std::max(kRqBuf, next_pow2(k));
}

// ---------------------------------------------------------------- mode 0: one step
__global__ void __launch_bounds__(kRqWarps * 32) rq_beam_step_kernel(
        const float* __restrict__ ip,     // [rows * Bin][K]
        const float* __restrict__ rnorm,  // [rows * Bin]
        const float* __restrict__ cnorm,  // [K]       ‖c‖² of codebook m
        const float* __restrict__ cb,     // [K][d]    codebook m
        const float* __restrict__ resid,  // [rows][Bin][d]
        const int32_t* __restrict__ codes, // [rows][Bin][M], the first m used
        int64_t rows,
        int Bin,
        int logK,
        int Bout,
        int m,
        int M,
        int d,
        int LIST,
        int32_t* __restrict__ codesOut, // [rows][Bout][M]
        float* __restrict__ residOut,   // [rows][Bout][d]
        float* __restrict__ distOut) {  // [rows][Bout]
    extern __shared__ __align__(16) unsigned char rq_step_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kRqWarps + warp;
    if (i >= rows)
        return;
    float* keys = reinterpret_cast<float*>(rq_step_smem + (size_t)warp * (LIST + kRqBuf) * 8);
    int* ids = reinterpret_cast<int*>(keys + LIST + kRqBuf);
    WarpTopK<int> tk;
    tk.init(keys, ids, LIST, kRqBuf, Bout);

    const int K = 1 << logK;
    const int total = Bin << logK;
    const float* ipi = ip + i * Bin * (int64_t)K;
    const float* rni = rnorm + i * Bin;
    for (int j0 = 0; j0 < total; j0 += 32) {
        const int j = j0 + lane;
        const bool valid = j < total;
        float v = 0.f;
        if (valid) {
            const int b = j >> logK, k = j & (K - 1);
            v = __fadd_rn(__fadd_rn(__ldg(rni + b), __ldg(cnorm + k)), -2.f * __ldg(ipi + j));
        }
        tk.add(valid, v, j);
    }
    tk.finish();

    for (int jj = 0; jj < Bout; jj++) {
        const int id = ids[jj];
        const int js = id >> logK, ls = id & (K - 1);
        const int32_t* pc = codes + (i * Bin + js) * M;
        int32_t* cc = codesOut + (i * Bout + jj) * M;
        for (int t = lane; t <= m; t += 32)
            cc[t] = t < m ? pc[t] : ls;
        const float* pr = resid + (i * Bin + js) * d;
        const float* c = cb + (int64_t)ls * d;
        float* rr = residOut + (i * Bout + jj) * d;
        for (int t = lane; t < d; t += 32)
            rr[t] = __fsub_rn(pr[t], __ldg(c + t));
        if (lane == 0)
            distOut[i * Bout + jj] = keys[jj];
    }
}

// ---------------------------------------------------------------- mode 1: all steps
struct LutSmem {
    int LIST, Bmax, M;
    size_t perWarp;
    size_t head; // the CTA's offsets table
    size_t bytes(int warps) const {
        return head + perWarp * warps;
    }
};

LutSmem lutSmem(int M, int Bmax, int outBeam) {
    LutSmem s;
    s.LIST = topkList(outBeam);
    s.Bmax = Bmax;
    s.M = M;
    s.perWarp = round_up((size_t)(s.LIST + kRqBuf) * 8 + (size_t)2 * Bmax * 4 + (size_t)2 * Bmax * M * 2, 16);
    s.head = round_up((size_t)(M + 1) * 4, 16);
    return s;
}

__global__ void __launch_bounds__(kRqWarps * 32) rq_beam_lut_kernel(
        const float* __restrict__ qcp,   // [rows][totalK]  x·Cᵀ
        const float* __restrict__ xnorm, // [rows]          ‖x‖²
        const float* __restrict__ cnorm, // [totalK]        ‖c‖²
        const float* __restrict__ cross, // the step blocks [off_m][K_m], back to back
        const int* __restrict__ offsets, // [M + 1]
        int64_t rows,
        int M,
        int64_t totalK,
        int outBeam,
        int LIST,
        int Bmax,
        int perWarp,
        int head,
        int Bfinal,
        int32_t* __restrict__ codesOut, // [rows][Bfinal][M]
        float* __restrict__ distOut) {  // [rows][Bfinal]
    extern __shared__ __align__(16) unsigned char rq_lut_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int* off = reinterpret_cast<int*>(rq_lut_smem);
    for (int t = threadIdx.x; t <= M; t += blockDim.x)
        off[t] = offsets[t];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (i >= rows)
        return;
    unsigned char* base = rq_lut_smem + head + (size_t)warp * perWarp;
    float* keys = reinterpret_cast<float*>(base);
    int* ids = reinterpret_cast<int*>(keys + LIST + kRqBuf);
    float* distP = reinterpret_cast<float*>(ids + LIST + kRqBuf);
    float* distC = distP + Bmax;
    int16_t* codeP = reinterpret_cast<int16_t*>(distC + Bmax);
    int16_t* codeC = codeP + Bmax * M;

    if (lane == 0)
        distP[0] = __ldg(xnorm + i);
    __syncwarp();
    const float* qi = qcp + i * totalK;
    int Bin = 1;
    int64_t crossOfs = 0;
    WarpTopK<int> tk;
    for (int m = 0; m < M; m++) {
        const int K = off[m + 1] - off[m];
        const int logK = __ffs(K) - 1;
        const int Bout = min(Bin * K, outBeam);
        tk.init(keys, ids, LIST, kRqBuf, Bout);
        const float* qm = qi + off[m];
        const float* nm = cnorm + off[m];
        const float* cr = cross + crossOfs;
        const bool fmaForm = m >= 1 && m <= 7 && K >= 32;
        const int total = Bin * K;
        for (int j0 = 0; j0 < total; j0 += 32) {
            const int j = j0 + lane;
            const bool valid = j < total;
            float v = 0.f;
            if (valid) {
                const int b = j >> logK, k = j & (K - 1);
                const float cd = __fadd_rn(__ldg(nm + k), -2.f * __ldg(qm + k));
                const float db = distP[b];
                if (m == 0) {
                    v = __fadd_rn(db, cd);
                } else {
                    const int16_t* pc = codeP + b * M;
                    float dp = 0.f;
                    for (int c0 = 0; c0 < m; c0 += 8) {
                        const int c1 = min(c0 + 8, m);
                        float s = __ldg(cr + ((int64_t)off[c0] + pc[c0]) * K + k);
                        for (int m1 = c0 + 1; m1 < c1; m1++)
                            s = __fadd_rn(s, __ldg(cr + ((int64_t)off[m1] + pc[m1]) * K + k));
                        dp = c0 == 0 ? s : __fadd_rn(dp, s);
                    }
                    v = fmaForm ? __fadd_rn(__fadd_rn(cd, 2.f * dp), db) : __fadd_rn(__fadd_rn(db, cd), 2.f * dp);
                }
            }
            tk.add(valid, v, j);
        }
        tk.finish();
        for (int jj = lane; jj < Bout; jj += 32) {
            const int id = ids[jj];
            const int js = id >> logK;
            distC[jj] = keys[jj];
            for (int t = 0; t < m; t++)
                codeC[jj * M + t] = codeP[js * M + t];
            codeC[jj * M + m] = (int16_t)(id & (K - 1));
        }
        __syncwarp();
        float* td = distP;
        distP = distC;
        distC = td;
        int16_t* tc = codeP;
        codeP = codeC;
        codeC = tc;
        crossOfs += (int64_t)off[m] * K;
        Bin = Bout;
    }
    if (codesOut)
        for (int e = lane; e < Bfinal * M; e += 32)
            codesOut[i * Bfinal * M + e] = codeP[e];
    if (distOut)
        for (int e = lane; e < Bfinal; e += 32)
            distOut[i * Bfinal + e] = distP[e];
}

// ---------------------------------------------------------------- packing
// encode_qint8 / encode_qint4 (faiss/impl/AdditiveQuantizer.cpp:220-232): int32_t(floor(x1)) as x86 converts it, the
// out-of-range value 0x80000000 for NaN and |x1| >= 2^31 (then clamped to 0)
__device__ __forceinline__ uint32_t rq_encode_qint(float x, float amin, float amax, int levels) {
    const float x1 = __fmul_rn(__fdiv_rn(__fsub_rn(x, amin), __fsub_rn(amax, amin)), (float)levels);
    const float f = floorf(x1);
    const int xi = (f >= -2147483648.f && f < 2147483648.f) ? (int)f : INT_MIN;
    return xi < 0 ? 0u : xi > levels - 1 ? (uint32_t)(levels - 1) : (uint32_t)xi;
}

// normMode: 0 none, 1 ‖x − r‖², 2 ‖decode (+ centroids)‖²
__global__ void __launch_bounds__(kRqWarps * 32) rq_pack_kernel(
        const int32_t* __restrict__ codes, // row i's codes at codes + i * ldc
        int64_t ldc,
        const float* __restrict__ x,     // [rows][d]
        const float* __restrict__ resid, // row i's residual at resid + i * ldr (normMode 1)
        int64_t ldr,
        const float* __restrict__ cb,        // [totalK][d]
        const int* __restrict__ offsets,     // [M + 1]
        const float* __restrict__ centroids, // [rows][d] or null
        int64_t rows,
        int M,
        int d,
        int normMode,
        int searchType,
        float normMin,
        float normMax,
        int codeSize,
        uint8_t* __restrict__ packed) { // [rows][codeSize]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kRqWarps + warp;
    if (i >= rows)
        return;
    const int32_t* ci = codes + i * ldc;
    float norm = 0.f;
    if (normMode != 0) {
        float acc = 0.f;
        for (int c = lane; c < d; c += 32) {
            float r;
            if (normMode == 1) {
                r = __fsub_rn(x[i * d + c], resid[i * ldr + c]);
            } else {
                r = __ldg(cb + ((int64_t)offsets[0] + ci[0]) * d + c);
                for (int m = 1; m < M; m++)
                    r = __fadd_rn(r, __ldg(cb + ((int64_t)offsets[m] + ci[m]) * d + c));
                if (centroids)
                    r = __fadd_rn(r, centroids[i * d + c]);
            }
            acc = __fmaf_rn(r, r, acc);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            acc += __shfl_xor_sync(kFullMask, acc, o);
        norm = __shfl_sync(kFullMask, acc, 0);
    }
    if (lane != 0)
        return;
    // BitstringWriter (faiss/utils/hamming-inl.h): LSB first, the bytes past the last field zero
    uint8_t* out = packed + i * codeSize;
    uint64_t acc = 0;
    int nacc = 0, o = 0;
    auto put = [&](uint32_t v, int nb) {
        acc |= (uint64_t)v << nacc;
        nacc += nb;
        while (nacc >= 8) {
            out[o++] = (uint8_t)acc;
            acc >>= 8;
            nacc -= 8;
        }
    };
    for (int m = 0; m < M; m++)
        put((uint32_t)ci[m], __ffs(offsets[m + 1] - offsets[m]) - 1);
    if (searchType == RQ_ST_norm_float)
        put(__float_as_uint(norm), 32);
    else if (searchType == RQ_ST_norm_qint8)
        put(rq_encode_qint(norm, normMin, normMax, 256), 8);
    else if (searchType == RQ_ST_norm_qint4)
        put(rq_encode_qint(norm, normMin, normMax, 16), 4);
    if (nacc > 0)
        out[o++] = (uint8_t)acc;
    while (o < codeSize)
        out[o++] = 0;
}

int normBits(int searchType) {
    switch (searchType) {
        case RQ_ST_norm_float: return 32;
        case RQ_ST_norm_qint8:
        case RQ_ST_norm_cqint8:
        case RQ_ST_norm_lsq2x4:
        case RQ_ST_norm_rq2x4: return 8;
        case RQ_ST_norm_qint4:
        case RQ_ST_norm_cqint4: return 4;
        default: return 0;
    }
}

bool packedOnDevice(int searchType) {
    return searchType >= RQ_ST_decompress && searchType <= RQ_ST_norm_qint4;
}

bool needsNorm(int searchType) {
    return searchType == RQ_ST_norm_float || searchType == RQ_ST_norm_qint8 || searchType == RQ_ST_norm_qint4;
}

} // namespace

// ------------------------------------------------------------------------------------------
// the page pipeline
// ------------------------------------------------------------------------------------------
struct GpuRqEncoder::Pipeline {
    const GpuRqEncoder& e;
    GpuResources* res;
    cudaStream_t stream;

    // the beam size after each step, from Bin entries
    std::vector<int> beams(int Bin, int outBeam) const {
        std::vector<int> b;
        for (int m = 0; m < e.M; m++) {
            Bin = (int)std::min<int64_t>((int64_t)Bin << e.nbits[m], outBeam);
            b.push_back(Bin);
        }
        return b;
    }

    // mode 0 over one page: `in` holds rp rows of beamIn residuals; on return codes / resid / dist point at the final
    // [rp][Bf][M], [rp][Bf][d], [rp][Bf] buffers (inside the given scratch)
    struct Mode0Bufs {
        GpuMemoryReservation rA, rB, cA, cB, dist, ip, rn;
        const int32_t* codes = nullptr;
        const float* resid = nullptr;
        const float* distances = nullptr;
    };

    // the largest beam after a step, the largest [B_in · K] inner-product block and the largest B_in of mode 0
    struct Mode0Sizes {
        int Bmax = 1, Bip = 1, Brn = 1;
    };
    static Mode0Sizes mode0Sizes(const GpuRqEncoder& e, int beamIn, const std::vector<int>& bs) {
        Mode0Sizes z;
        int Bin = beamIn;
        for (int m = 0; m < e.M; m++) {
            z.Bmax = std::max(z.Bmax, bs[m]);
            z.Bip = std::max<int>(z.Bip, Bin << e.nbits[m]);
            z.Brn = std::max(z.Brn, Bin);
            Bin = bs[m];
        }
        return z;
    }

    static size_t mode0RowBytes(const GpuRqEncoder& e, int beamIn, const std::vector<int>& bs) {
        const Mode0Sizes z = mode0Sizes(e, beamIn, bs);
        return sizeof(float) * ((size_t)beamIn * e.d + 2 * (size_t)z.Bmax * e.d + z.Bmax + z.Bip + z.Brn) +
                sizeof(int32_t) * 2 * (size_t)z.Bmax * e.M;
    }

    void allocMode0(Mode0Bufs& b, int64_t rows, int beamIn, const std::vector<int>& bs) const {
        const Mode0Sizes z = mode0Sizes(e, beamIn, bs);
        b.rA = res->temp(e.device_, sizeof(float) * rows * z.Bmax * e.d);
        b.rB = res->temp(e.device_, sizeof(float) * rows * z.Bmax * e.d);
        b.cA = res->temp(e.device_, sizeof(int32_t) * rows * z.Bmax * e.M);
        b.cB = res->temp(e.device_, sizeof(int32_t) * rows * z.Bmax * e.M);
        b.dist = res->temp(e.device_, sizeof(float) * rows * z.Bmax);
        b.ip = res->temp(e.device_, sizeof(float) * rows * z.Bip);
        b.rn = res->temp(e.device_, sizeof(float) * rows * z.Brn);
    }

    void runMode0(Mode0Bufs& b, const float* in, int64_t rp, int beamIn, const std::vector<int>& bs) const {
        const float* parentR = in;
        const int32_t* parentC = b.cA.as<int32_t>();
        float* childR = b.rA.as<float>();
        int32_t* childC = b.cB.as<int32_t>();
        int Bin = beamIn;
        for (int m = 0; m < e.M; m++) {
            const int K = 1 << e.nbits[m];
            const int Bout = bs[m];
            const float* cbm = e.codebooks_.as<float>() + e.offsets_[m] * e.d;
            KernelTiming::begin("rq_gemm", stream);
            runL2Norms(parentR, rp * Bin, e.d, b.rn.as<float>(), stream);
            runFlatPairwise(res, e.device_, parentR, rp * Bin, cbm, K, e.d, METRIC_INNER_PRODUCT, 0.f, b.ip.as<float>(), K, stream);
            KernelTiming::end("rq_gemm", stream);
            const int LIST = topkList(Bout);
            const size_t smem = (size_t)kRqWarps * (LIST + kRqBuf) * 8; // 12 KB at most (LIST <= 256)
            KernelTiming::begin("rq_step", stream);
            rq_beam_step_kernel<<<(unsigned)ceil_div(rp, kRqWarps), kRqWarps * 32, smem, stream>>>(
                    b.ip.as<float>(), b.rn.as<float>(), e.norms_.as<float>() + e.offsets_[m], cbm, parentR, parentC, rp, Bin,
                    e.nbits[m], Bout, m, e.M, e.d, LIST, childC, childR, b.dist.as<float>());
            CUDA_CHECK_LAST();
            KernelTiming::end("rq_step", stream);
            parentR = childR;
            parentC = childC;
            childR = (childR == b.rA.as<float>()) ? b.rB.as<float>() : b.rA.as<float>();
            childC = (childC == b.cB.as<int32_t>()) ? b.cA.as<int32_t>() : b.cB.as<int32_t>();
            Bin = Bout;
        }
        b.codes = parentC;
        b.resid = parentR;
        b.distances = b.dist.as<float>();
    }

    static size_t mode1RowBytes(const GpuRqEncoder& e, int Bf) {
        return sizeof(float) * ((size_t)e.d + e.totalK_ + 1 + Bf) + sizeof(int32_t) * (size_t)Bf * e.M;
    }

    // mode 1 over one page: x [rp][d] on the device -> codes [rp][Bf][M], dist [rp][Bf]
    void runMode1(const float* x, int64_t rp, int outBeam, const std::vector<int>& bs, float* qcp, float* xn,
                  int32_t* codes, float* dist) const {
        const int Bf = bs.back();
        const int Bmax = *std::max_element(bs.begin(), bs.end());
        KernelTiming::begin("rq_gemm", stream);
        runL2Norms(x, rp, e.d, xn, stream);
        runFlatPairwise(res, e.device_, x, rp, e.codebooks_.as<float>(), e.totalK_, e.d, METRIC_INNER_PRODUCT, 0.f, qcp, e.totalK_, stream);
        KernelTiming::end("rq_gemm", stream);
        const LutSmem s = lutSmem(e.M, std::max(Bmax, 1), outBeam);
        int warps = kRqWarps;
        while (warps > 1 && s.bytes(warps) > kRqSmemLimit)
            warps--;
        const size_t smem = s.bytes(warps);
        if (smem > 48 * 1024)
            CUDA_VERIFY(cudaFuncSetAttribute(rq_beam_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        KernelTiming::begin("rq_lut", stream);
        rq_beam_lut_kernel<<<(unsigned)ceil_div(rp, warps), warps * 32, smem, stream>>>(
                qcp, xn, e.norms_.as<float>(), e.cross_.as<float>(), e.meta_.as<int>(), rp, e.M, e.totalK_, outBeam, s.LIST,
                s.Bmax, (int)s.perWarp, (int)s.head, Bf, codes, dist);
        CUDA_CHECK_LAST();
        KernelTiming::end("rq_lut", stream);
    }

    void pack(const int32_t* codes, int64_t ldc, const float* x, const float* resid, int64_t ldr, const float* centroids,
              int64_t rp, int normMode, int searchType, float normMin, float normMax, uint8_t* packed) const {
        KernelTiming::begin("rq_pack", stream);
        rq_pack_kernel<<<(unsigned)ceil_div(rp, kRqWarps), kRqWarps * 32, 0, stream>>>(
                codes, ldc, x, resid, ldr, e.codebooks_.as<float>(), e.meta_.as<int>(), centroids, rp, e.M, e.d, normMode,
                searchType, normMin, normMax, (int)e.codeSize(searchType), packed);
        CUDA_CHECK_LAST();
        KernelTiming::end("rq_pack", stream);
    }

    static idx_t pageRows(idx_t n, size_t perRow, size_t pageBytes) {
        return std::min<idx_t>(std::max<idx_t>(n, 1), std::max<idx_t>(1, (idx_t)(pageBytes / perRow)));
    }

    // the search of compute_codes over pages; per page, `emit` gets the final codes (entry 0 of row i at codes + i * ldc),
    // the page's x and, in mode 0, the final residuals (entry 0 at resid + i * ldr)
    template <typename Emit>
    void encodePages(const float* x, idx_t n, bool useBeamLUT, int maxBeam, size_t extraPerRow, size_t pageBytes, Emit emit) {
        const int device = e.device_;
        const auto bs = beams(1, maxBeam);
        const int Bf = bs.back();
        const int d = e.d, M = e.M;
        if (useBeamLUT) {
            const idx_t rows = pageRows(n, mode1RowBytes(e, Bf) + extraPerRow, pageBytes);
            GpuMemoryReservation xBuf = res->temp(device, sizeof(float) * rows * d);
            GpuMemoryReservation qcp = res->temp(device, sizeof(float) * rows * e.totalK_);
            GpuMemoryReservation xn = res->temp(device, sizeof(float) * rows);
            GpuMemoryReservation cBuf = res->temp(device, sizeof(int32_t) * rows * Bf * M);
            for (idx_t r0 = 0; r0 < n; r0 += rows) {
                InterruptCallback::check(); // between pages
                const idx_t rp = std::min(rows, n - r0);
                CUDA_VERIFY(cudaMemcpyAsync(xBuf.data, x + r0 * d, sizeof(float) * rp * d, cudaMemcpyDefault, stream));
                runMode1(xBuf.as<float>(), rp, maxBeam, bs, qcp.as<float>(), xn.as<float>(), cBuf.as<int32_t>(), nullptr);
                emit(r0, rp, cBuf.as<int32_t>(), (int64_t)Bf * M, xBuf.as<float>(), nullptr, (int64_t)0);
            }
        } else {
            const idx_t rows = pageRows(n, mode0RowBytes(e, 1, bs) + extraPerRow, pageBytes);
            GpuMemoryReservation xBuf = res->temp(device, sizeof(float) * rows * d);
            Mode0Bufs b;
            allocMode0(b, rows, 1, bs);
            for (idx_t r0 = 0; r0 < n; r0 += rows) {
                InterruptCallback::check(); // between pages
                const idx_t rp = std::min(rows, n - r0);
                CUDA_VERIFY(cudaMemcpyAsync(xBuf.data, x + r0 * d, sizeof(float) * rp * d, cudaMemcpyDefault, stream));
                runMode0(b, xBuf.as<float>(), rp, 1, bs);
                emit(r0, rp, b.codes, (int64_t)Bf * M, xBuf.as<float>(), b.resid, (int64_t)Bf * d);
            }
        }
    }
};

// ------------------------------------------------------------------------------------------
// GpuRqEncoder
// ------------------------------------------------------------------------------------------
GpuRqEncoder::GpuRqEncoder(int d_, std::vector<int> nbits_, std::shared_ptr<GpuResources> res, int device)
        : d(d_), M((int)nbits_.size()), nbits(std::move(nbits_)), res_(std::move(res)), device_(device) {
    FB_THROW_IF_NOT_FMT(d >= 1, "d = %d: GpuRqEncoder needs d >= 1", d);
    FB_THROW_IF_NOT_MSG(M >= 1, "GpuRqEncoder needs at least one codebook");
    FB_THROW_IF_NOT_MSG(res_ != nullptr, "null resources");
    int ndev = 0;
    CUDA_VERIFY(cudaGetDeviceCount(&ndev));
    FB_THROW_IF_NOT_FMT(device >= 0 && device < ndev, "device %d does not exist", device);
    offsets_.assign(M + 1, 0);
    for (int m = 0; m < M; m++) {
        FB_THROW_IF_NOT_FMT(
                nbits[m] >= 1 && nbits[m] <= kRqMaxNbits, "nbits[%d] = %d: GpuRqEncoder takes 1 <= nbits <= 12", m, nbits[m]);
        offsets_[m + 1] = offsets_[m] + (int64_t(1) << nbits[m]);
    }
    totalK_ = offsets_[M];
}

GpuRqEncoder::~GpuRqEncoder() = default;

size_t GpuRqEncoder::codeSize(int searchType) const {
    size_t bits = normBits(searchType);
    for (int b : nbits)
        bits += b;
    return (bits + 7) / 8;
}

int GpuRqEncoder::finalBeam(int beamIn, int outBeam) const {
    int64_t B = beamIn;
    for (int m = 0; m < M; m++)
        B = std::min<int64_t>(B << nbits[m], outBeam);
    return (int)B;
}

void GpuRqEncoder::setCodebooks(const float* codebooks) {
    FB_THROW_IF_NOT_MSG(codebooks != nullptr, "null codebooks");
    haveCodebooks_ = false;
    DeviceScope scope(device_);
    cudaStream_t stream = res_->getDefaultStream(device_);
    int64_t crossSize = 0;
    for (int m = 1; m < M; m++)
        crossSize += offsets_[m] << nbits[m];
    codebooks_ = res_->device_alloc(device_, sizeof(float) * totalK_ * d, AllocType::Other);
    norms_ = res_->device_alloc(device_, sizeof(float) * totalK_, AllocType::Other);
    cross_ = res_->device_alloc(device_, sizeof(float) * std::max<int64_t>(crossSize, 1), AllocType::Other);
    meta_ = res_->device_alloc(device_, sizeof(int) * (M + 1), AllocType::Other);
    std::vector<int> off32(offsets_.begin(), offsets_.end());
    CUDA_VERIFY(cudaMemcpyAsync(meta_.data, off32.data(), sizeof(int) * (M + 1), cudaMemcpyHostToDevice, stream));
    CUDA_VERIFY(cudaMemcpyAsync(codebooks_.data, codebooks, sizeof(float) * totalK_ * d, cudaMemcpyDefault, stream));
    const float* cb = codebooks_.as<float>();
    runL2Norms(cb, totalK_, d, norms_.as<float>(), stream);
    int64_t ofs = 0;
    for (int m = 1; m < M; m++) {
        const int64_t K = int64_t(1) << nbits[m];
        runFlatPairwise(res_.get(), device_, cb, offsets_[m], cb + offsets_[m] * d, K, d, METRIC_INNER_PRODUCT, 0.f,
                        cross_.as<float>() + ofs, K, stream);
        ofs += offsets_[m] * K;
    }
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    haveCodebooks_ = true;
}

void GpuRqEncoder::checkReady() const {
    FB_THROW_IF_NOT_MSG(haveCodebooks_, "setCodebooks must be called before encoding");
}

static void checkBeam(const char* what, int b) {
    FB_THROW_IF_NOT_FMT(b >= 1 && b <= kRqMaxBeam, "%s = %d: GpuRqEncoder takes 1 <= beam <= 256", what, b);
}

void GpuRqEncoder::refineBeam(
        idx_t n,
        int beamIn,
        const float* residuals,
        int outBeam,
        int32_t* codes,
        float* residualsOut,
        float* distances,
        size_t pageBytes) const {
    checkBeam("beam_size", beamIn);
    checkBeam("out_beam_size", outBeam);
    FB_THROW_IF_NOT_FMT(n >= 0, "n = %lld: must be >= 0", (long long)n);
    FB_THROW_IF_NOT_MSG(pageBytes > 0, "page budget must be > 0");
    checkReady();
    if (n == 0)
        return;
    FB_THROW_IF_NOT_MSG(residuals != nullptr, "null residuals");
    DeviceScope scope(device_);
    Pipeline p{*this, res_.get(), res_->getDefaultStream(device_)};
    const auto bs = p.beams(beamIn, outBeam);
    const int Bf = bs.back();
    const idx_t rows = Pipeline::pageRows(n, Pipeline::mode0RowBytes(*this, beamIn, bs), pageBytes);
    GpuMemoryReservation inBuf = res_->temp(device_, sizeof(float) * rows * beamIn * d);
    Pipeline::Mode0Bufs b;
    p.allocMode0(b, rows, beamIn, bs);
    for (idx_t r0 = 0; r0 < n; r0 += rows) {
        InterruptCallback::check(); // between pages
        const idx_t rp = std::min(rows, n - r0);
        CUDA_VERIFY(cudaMemcpyAsync(inBuf.data, residuals + r0 * beamIn * d, sizeof(float) * rp * beamIn * d, cudaMemcpyDefault, p.stream));
        p.runMode0(b, inBuf.as<float>(), rp, beamIn, bs);
        if (codes)
            CUDA_VERIFY(cudaMemcpyAsync(codes + r0 * Bf * M, b.codes, sizeof(int32_t) * rp * Bf * M, cudaMemcpyDefault, p.stream));
        if (residualsOut)
            CUDA_VERIFY(cudaMemcpyAsync(residualsOut + r0 * Bf * d, b.resid, sizeof(float) * rp * Bf * d, cudaMemcpyDefault, p.stream));
        if (distances)
            CUDA_VERIFY(cudaMemcpyAsync(distances + r0 * Bf, b.distances, sizeof(float) * rp * Bf, cudaMemcpyDefault, p.stream));
        CUDA_VERIFY(cudaStreamSynchronize(p.stream));
    }
}

// the LUT kernel's shared memory for (M, the largest beam, outBeam) must fit one warp
static void checkLutFits(const GpuRqEncoder& e, const std::vector<int>& bs, int outBeam) {
    const int Bmax = *std::max_element(bs.begin(), bs.end());
    const LutSmem s = lutSmem(e.M, Bmax, outBeam);
    FB_THROW_IF_NOT_FMT(
            s.bytes(1) <= kRqSmemLimit,
            "M = %d with beam %d: the LUT beam search needs %zu bytes of shared memory per row, more than %zu", e.M, Bmax,
            s.bytes(1), kRqSmemLimit);
}

void GpuRqEncoder::refineBeamLUT(idx_t n, const float* x, int outBeam, int32_t* codes, float* distances, size_t pageBytes) const {
    checkBeam("out_beam_size", outBeam);
    FB_THROW_IF_NOT_FMT(n >= 0, "n = %lld: must be >= 0", (long long)n);
    FB_THROW_IF_NOT_MSG(pageBytes > 0, "page budget must be > 0");
    checkReady();
    DeviceScope scope(device_);
    Pipeline p{*this, res_.get(), res_->getDefaultStream(device_)};
    const auto bs = p.beams(1, outBeam);
    checkLutFits(*this, bs, outBeam);
    if (n == 0)
        return;
    FB_THROW_IF_NOT_MSG(x != nullptr, "null x");
    const int Bf = bs.back();
    const idx_t rows = Pipeline::pageRows(n, Pipeline::mode1RowBytes(*this, Bf), pageBytes);
    GpuMemoryReservation xBuf = res_->temp(device_, sizeof(float) * rows * d);
    GpuMemoryReservation qcp = res_->temp(device_, sizeof(float) * rows * totalK_);
    GpuMemoryReservation xn = res_->temp(device_, sizeof(float) * rows);
    GpuMemoryReservation cBuf = res_->temp(device_, sizeof(int32_t) * rows * Bf * M);
    GpuMemoryReservation dBuf = res_->temp(device_, sizeof(float) * rows * Bf);
    for (idx_t r0 = 0; r0 < n; r0 += rows) {
        InterruptCallback::check(); // between pages
        const idx_t rp = std::min(rows, n - r0);
        CUDA_VERIFY(cudaMemcpyAsync(xBuf.data, x + r0 * d, sizeof(float) * rp * d, cudaMemcpyDefault, p.stream));
        p.runMode1(xBuf.as<float>(), rp, outBeam, bs, qcp.as<float>(), xn.as<float>(), cBuf.as<int32_t>(), dBuf.as<float>());
        if (codes)
            CUDA_VERIFY(cudaMemcpyAsync(codes + r0 * Bf * M, cBuf.data, sizeof(int32_t) * rp * Bf * M, cudaMemcpyDefault, p.stream));
        if (distances)
            CUDA_VERIFY(cudaMemcpyAsync(distances + r0 * Bf, dBuf.data, sizeof(float) * rp * Bf, cudaMemcpyDefault, p.stream));
        CUDA_VERIFY(cudaStreamSynchronize(p.stream));
    }
}

void GpuRqEncoder::computeCodes(
        const float* x,
        idx_t n,
        bool useBeamLUT,
        int maxBeam,
        int searchType,
        float normMin,
        float normMax,
        const float* centroids,
        uint8_t* packed,
        size_t pageBytes) const {
    checkBeam("max_beam_size", maxBeam);
    FB_THROW_IF_NOT_FMT(
            packedOnDevice(searchType),
            "search type %d is not packed on the device (ST_decompress .. ST_norm_qint4 are)", searchType);
    FB_THROW_IF_NOT_FMT(n >= 0, "n = %lld: must be >= 0", (long long)n);
    FB_THROW_IF_NOT_MSG(pageBytes > 0, "page budget must be > 0");
    checkReady();
    DeviceScope scope(device_);
    Pipeline p{*this, res_.get(), res_->getDefaultStream(device_)};
    if (useBeamLUT)
        checkLutFits(*this, p.beams(1, maxBeam), maxBeam);
    if (n == 0)
        return;
    FB_THROW_IF_NOT_MSG(x != nullptr && packed != nullptr, "null x or codes");
    const size_t cs = codeSize(searchType);
    const int normMode = !needsNorm(searchType) ? 0 : (useBeamLUT || centroids) ? 2 : 1;
    const idx_t maxRows = Pipeline::pageRows(n, sizeof(float) * d + cs, pageBytes);
    GpuMemoryReservation pBuf = res_->temp(device_, cs * maxRows);
    GpuMemoryReservation cenBuf = res_->temp(device_, centroids ? sizeof(float) * maxRows * d : 1);
    p.encodePages(x, n, useBeamLUT, maxBeam, sizeof(float) * d + cs, pageBytes,
                [&](idx_t r0, idx_t rp, const int32_t* codes, int64_t ldc, const float* xp, const float* resid, int64_t ldr) {
                    FB_THROW_IF_NOT_MSG(rp <= maxRows, "page larger than its packing buffer");
                    if (centroids)
                        CUDA_VERIFY(cudaMemcpyAsync(cenBuf.data, centroids + r0 * d, sizeof(float) * rp * d, cudaMemcpyDefault, p.stream));
                    p.pack(codes, ldc, xp, resid, ldr, centroids ? cenBuf.as<float>() : nullptr, rp, normMode, searchType,
                           normMin, normMax, pBuf.as<uint8_t>());
                    CUDA_VERIFY(cudaMemcpyAsync(packed + r0 * cs, pBuf.data, cs * rp, cudaMemcpyDefault, p.stream));
                    CUDA_VERIFY(cudaStreamSynchronize(p.stream));
                });
}

void GpuRqEncoder::encodeUnpacked(const float* x, idx_t n, bool useBeamLUT, int maxBeam, int32_t* codes, size_t pageBytes) const {
    checkBeam("max_beam_size", maxBeam);
    FB_THROW_IF_NOT_FMT(n >= 0, "n = %lld: must be >= 0", (long long)n);
    FB_THROW_IF_NOT_MSG(pageBytes > 0, "page budget must be > 0");
    checkReady();
    DeviceScope scope(device_);
    Pipeline p{*this, res_.get(), res_->getDefaultStream(device_)};
    if (useBeamLUT)
        checkLutFits(*this, p.beams(1, maxBeam), maxBeam);
    if (n == 0)
        return;
    FB_THROW_IF_NOT_MSG(x != nullptr && codes != nullptr, "null x or codes");
    p.encodePages(x, n, useBeamLUT, maxBeam, 0, pageBytes,
                  [&](idx_t r0, idx_t rp, const int32_t* pc, int64_t ldc, const float*, const float*, int64_t) {
                      CUDA_VERIFY(cudaMemcpy2DAsync(codes + r0 * M, sizeof(int32_t) * M, pc, sizeof(int32_t) * ldc,
                                                    sizeof(int32_t) * M, rp, cudaMemcpyDefault, p.stream));
                      CUDA_VERIFY(cudaStreamSynchronize(p.stream));
                  });
}

} // namespace fb200
