// faiss_b200 -- IVF scalar quantiser: min/max range training, encoding, and the fused decode-and-scan.
//
// Reference roles: faiss/gpu/impl/IVFFlatScan.cu + GpuScalarQuantizer.cuh (GPU scan with the codec in the
// inner loop).  The arithmetic follows the CPU classes, which are this project's oracle:
// faiss/impl/scalar_quantizer/quantizers.h:66-150 (encode / decode), codecs.h:25-120 (bit layouts),
// training.cpp:209-383 (RS_minmax ranges), scanners.h:44-135 (distance forms).
//
// Lists keep the CPU's vector-major [len][code_size] byte layout (as IVF-Flat and IVF-PQ's flat layout), so
// setList / getListVectorData are plain copies.
#include <cuda_fp16.h>

#include "ivf_layout.cuh"
#include "ivf_scan.cuh"

namespace fb200 {

// ------------------------------------------------------------------------------------------
// RS_minmax training: per-dimension min / max.  Min and max do not depend on the order in which elements
// are visited, so the result is bit-exact with the CPU's sequential loop (training.cpp:221-231, 345-358).
// ------------------------------------------------------------------------------------------
__global__ void sq_minmax_kernel(
        const float* __restrict__ x,
        int64_t n,
        int d,
        int64_t rowsPerBlock,
        unsigned* __restrict__ omin,
        unsigned* __restrict__ omax) {
    const int64_t r0 = (int64_t)blockIdx.x * rowsPerBlock;
    const int64_t r1 = min(n, r0 + rowsPerBlock);
    for (int j = threadIdx.x; j < d; j += blockDim.x) {
        float lo = CUDART_INF_F, hi = -CUDART_INF_F;
        for (int64_t i = r0; i < r1; i++) {
            const float v = x[i * d + j];
            lo = fminf(lo, v);
            hi = fmaxf(hi, v);
        }
        atomicMin(&omin[j], float_to_ordered(lo));
        atomicMax(&omax[j], float_to_ordered(hi));
    }
}

__global__ void sq_ordered_to_float_kernel(const unsigned* __restrict__ in, int n, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        out[i] = ordered_to_float(in[i]);
}

void runSqMinMax(const float* x, int64_t n, int d, float* vminOut, float* vmaxOut, cudaStream_t stream) {
    FB_THROW_IF_NOT(n > 0);
    unsigned* buf;
    CUDA_VERIFY(cudaMallocAsync(&buf, sizeof(unsigned) * 2 * d, stream));
    CUDA_VERIFY(cudaMemsetAsync(buf, 0xff, sizeof(unsigned) * d, stream)); // min: ordered +max
    CUDA_VERIFY(cudaMemsetAsync(buf + d, 0, sizeof(unsigned) * d, stream)); // max: ordered -max
    const int64_t rowsPerBlock = std::max<int64_t>(64, ceil_div(n, 132 * 8));
    sq_minmax_kernel<<<(unsigned)ceil_div(n, rowsPerBlock), 128, 0, stream>>>(x, n, d, rowsPerBlock, buf, buf + d);
    CUDA_CHECK_LAST();
    sq_ordered_to_float_kernel<<<(unsigned)ceil_div(d, 256), 256, 0, stream>>>(buf, d, vminOut);
    sq_ordered_to_float_kernel<<<(unsigned)ceil_div(d, 256), 256, 0, stream>>>(buf + d, d, vmaxOut);
    CUDA_CHECK_LAST();
    CUDA_VERIFY(cudaFreeAsync(buf, stream));
}

// ------------------------------------------------------------------------------------------
// encode: one thread per output byte, so every byte is written exactly once (the CPU zeroes the code and
// ORs components into it, quantizers.h:77-92 + codecs.h).  Byte-exact with the CPU:
//   xi = (x - vmin) / vdiff (IEEE division; 0 when vdiff == 0), clamped to [0, 1];
//   8-bit: (int)(255 * xi), an fp32 product rounded to nearest, then truncated;
//   4-/6-bit: (int)(xi * 15.0) / (int)(xi * 63.0) are double products on the CPU.  xi has 24 significant
//   bits, so the double product is exact, and an fp32 product rounded toward zero truncates to the same
//   integer (an integer is representable, so RZ never crosses it).  A round-to-nearest fp32 product can.
//   fp16: round to nearest even (_mm_cvtps_ph with _MM_FROUND_TO_NEAREST_INT in the avx2 build).
//   8bit_direct: (uint8_t)x, i.e. the low byte of the truncated int.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int sq_level(float x, float vmin, float vdiff, int qtype) {
    float xi = 0.f;
    if (vdiff != 0.f) {
        xi = __fdiv_rn(__fsub_rn(x, vmin), vdiff);
        if (xi < 0.f)
            xi = 0.f;
        if (xi > 1.f)
            xi = 1.f;
    }
    if (qtype == SQ_QT_4bit || qtype == SQ_QT_4bit_uniform)
        return __float2int_rz(__fmul_rz(xi, 15.f));
    if (qtype == SQ_QT_6bit)
        return __float2int_rz(__fmul_rz(xi, 63.f));
    return __float2int_rz(__fmul_rn(255.f, xi));
}

__global__ void sq_encode_kernel(
        const float* __restrict__ x,
        int64_t n,
        int d,
        int qtype,
        int codeSize,
        const float* __restrict__ vmin,
        const float* __restrict__ vdiff,
        uint8_t* __restrict__ codes) {
    const int64_t total = n * codeSize;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = t / codeSize;
        const int j = (int)(t - row * codeSize);
        const float* xr = x + row * d;
        unsigned byte = 0;
        switch (qtype) {
            case SQ_QT_fp16: {
                const unsigned short h = __half_as_ushort(__float2half_rn(xr[j >> 1]));
                byte = (j & 1) ? (h >> 8) : (h & 0xffu);
                break;
            }
            case SQ_QT_8bit_direct:
                byte = (unsigned)__float2int_rz(xr[j]);
                break;
            case SQ_QT_4bit:
            case SQ_QT_4bit_uniform: {
                const int i = 2 * j;
                byte = (unsigned)sq_level(xr[i], vmin[i], vdiff[i], qtype);
                if (i + 1 < d)
                    byte |= (unsigned)sq_level(xr[i + 1], vmin[i + 1], vdiff[i + 1], qtype) << 4;
                break;
            }
            case SQ_QT_6bit: { // codecs.h:64-92: 4 components in 3 bytes
                const int g = j / 3, r = j - 3 * g;
                unsigned b[4];
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int i = 4 * g + c;
                    b[c] = i < d ? (unsigned)sq_level(xr[i], vmin[i], vdiff[i], qtype) : 0u;
                }
                byte = r == 0 ? (b[0] | (b[1] << 6)) : r == 1 ? ((b[1] >> 2) | (b[2] << 4)) : ((b[2] >> 4) | (b[3] << 2));
                break;
            }
            default: // 8bit, 8bit_uniform
                byte = (unsigned)sq_level(xr[j], vmin[j], vdiff[j], qtype);
                break;
        }
        codes[t] = (uint8_t)(byte & 0xffu);
    }
}

void runSqEncode(
        const float* x,
        int64_t n,
        int d,
        int qtype,
        int codeSize,
        const float* vmin,
        const float* vdiff,
        uint8_t* codes,
        cudaStream_t stream) {
    if (n == 0)
        return;
    const int64_t total = n * codeSize;
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(total, 256), 132 * 32);
    sq_encode_kernel<<<blocks, 256, 0, stream>>>(x, n, d, qtype, codeSize, vmin, vdiff, codes);
    CUDA_CHECK_LAST();
}

// ------------------------------------------------------------------------------------------
// scan
//
// Decode folding.  The CPU decodes x_i = vmin_i + vdiff_i * (c_i + 0.5) / s and then forms (r_i - x_i)^2 or
// q_i * x_i.  Here the decode is x_i = m_i + b_i * c_i with b_i = vdiff_i / s and m_i = vmin_i + 0.5 b_i
// (m = 0, b = 1 and c = the stored value for fp16 / 8bit_direct), tabulated once per index.  Per (query,
// probe) the kernel builds, in shared memory,
//   L2:  a_i = r_i - m_i  (r = q - centroid with a residual, else q)   ->  sum_i (a_i - b_i c_i)^2
//   IP:  w_i = q_i b_i,   K = sum_i q_i m_i (+ the coarse distance)   ->  K + sum_i w_i c_i
// so every component costs two FMAs (L2) or one (IP) after the code -> float conversion.  The integer codes
// are turned into floats without I2F: PRMT / LOP3 the code into 0x4B0000cc (= 2^23 + c) and subtract 2^23.
//
// Codecs (template): 0 = one byte per component (8bit, 8bit_uniform, 8bit_direct), 1 = nibbles (4bit,
// 4bit_uniform), 2 = 6-bit (3 bytes per 4 components), 3 = fp16 (ivf_layout.cuh).
// ------------------------------------------------------------------------------------------
template <int CODEC>
struct SqFast {
    // components per 32-bit word, components per 128-byte row chunk, max chunks held in registers
    static constexpr int CPW = CODEC == SQC_BYTE ? 4 : CODEC == SQC_NIBBLE ? 8 : 2;
    static constexpr int PER_CHUNK = 32 * CPW;
    static constexpr int MAXCH = CODEC == SQC_HALF ? 4 : 2; // d <= 256 (8-bit, fp16) or 512 (4-bit)
};

// component j (0 <= j < CPW) of a 32-bit code word
template <int CODEC>
__device__ __forceinline__ float sq_word_comp(unsigned w, int j) {
    if (CODEC == SQC_BYTE) {
        return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540u | (unsigned)j)) - 8388608.f;
    } else if (CODEC == SQC_NIBBLE) {
        return sq_u2f((w >> (4 * j)) & 0xfu);
    } else {
        const __half h = __ushort_as_half((unsigned short)(j ? (w >> 16) : (w & 0xffffu)));
        return __half2float(h);
    }
}

template <int CODEC, bool IS_L2, typename IdT, bool MASKED>
__global__ void __launch_bounds__(kScanWarps * 32) ivfsq_scan_kernel(
        const float* __restrict__ Q,
        int d,
        const idx_t* __restrict__ probes,
        const float* __restrict__ coarseDis, // IP with a residual: added to every distance; else null
        int nprobe,
        int probesPerCta,
        const float* __restrict__ coarse, // L2 with a residual: the centroids; else null
        const float* __restrict__ mb,     // m[d] | b[d]
        const int64_t* __restrict__ listStart,
        const int* __restrict__ listLen,
        const uint8_t* __restrict__ arenaCodes,
        const idx_t* __restrict__ arenaIds,
        int codeSize,
        int fast,
        int k,
        int LIST,
        float* __restrict__ partD, // [nq, chunks, k] keys
        idx_t* __restrict__ partI,
        const uint32_t* __restrict__ slotMask) { // MASKED: the selector's arena mask
    using F = SqFast<CODEC>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int q = blockIdx.y, chunk = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = lane_id();
    float* ta = reinterpret_cast<float*>(smem_raw); // [d]  a (L2) or w (IP)
    float* tb = ta + d;                              // [d]  b (L2)
    float* red = tb + d;                             // [kScanWarps] partial sums of K (IP)
    unsigned char* lists = smem_raw + round_up(sizeof(float) * (2 * d + kScanWarps), 16);
    const size_t perWarp = SmemTopK<IdT>::bytes(LIST, kScanBuf);
    float* oD = partD + ((int64_t)q * gridDim.x + chunk) * k;
    idx_t* oI = partI + ((int64_t)q * gridDim.x + chunk) * k;
    const float* qv = Q + (int64_t)q * d;

    WarpTopK<IdT> w;
    unsigned char* mine = lists + perWarp * warp;
    w.init(reinterpret_cast<float*>(mine), reinterpret_cast<IdT*>(mine + sizeof(float) * (LIST + kScanBuf)), LIST, kScanBuf, k);

    // IP tables and L2 tables without a residual depend on the query only
    const bool perProbe = IS_L2 && coarse != nullptr;
    float K = 0.f;
    if (!perProbe) {
        float part = 0.f;
        for (int i = threadIdx.x; i < d; i += blockDim.x) {
            const float x = qv[i], m = mb[i], b = mb[d + i];
            if (IS_L2) {
                ta[i] = x - m;
                tb[i] = b;
            } else {
                ta[i] = x * b;
                part = fmaf(x, m, part);
            }
        }
        if (!IS_L2) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
                part += __shfl_xor_sync(kFullMask, part, o);
            if (lane == 0)
                red[warp] = part;
        }
        __syncthreads();
        if (!IS_L2) {
#pragma unroll
            for (int ww = 0; ww < kScanWarps; ww++)
                K += red[ww];
        }
    }
    const int pBegin = chunk * probesPerCta, pEnd = min(nprobe, pBegin + probesPerCta);

    for (int p = pBegin; p < pEnd; p++) {
        const idx_t l = probes[(int64_t)q * nprobe + p];
        if (l < 0) // NaN query / missing probe (block-uniform)
            continue;
        if (perProbe) { // a_i = (q_i - c_i) - m_i: the CPU's residual (IndexIVF compute_residual) first
            __syncthreads();
            for (int i = threadIdx.x; i < d; i += blockDim.x) {
                ta[i] = (qv[i] - coarse[l * d + i]) - mb[i];
                tb[i] = mb[d + i];
            }
            __syncthreads();
        }
        const float Kp = IS_L2 ? 0.f : K + (coarseDis ? coarseDis[(int64_t)q * nprobe + p] : 0.f);
        const int len = listLen[l];
        const int64_t ls = listStart[l];
        const uint8_t* base = arenaCodes + ls * codeSize;

        if (CODEC != SQC_SIX && fast) {
            // Fast path (rows of whole 128-byte chunks): lane t owns code word t of every chunk and keeps the
            // tables of its components in registers.  32 vectors per group, issued 16 at a time; the 32
            // per-lane partial sums are reduced with one transposing butterfly (as the IVF-Flat fast path).
            const int nch = codeSize >> 7;
            float ra[F::MAXCH][F::CPW], rb[F::MAXCH][F::CPW];
#pragma unroll
            for (int c = 0; c < F::MAXCH; c++)
#pragma unroll
                for (int j = 0; j < F::CPW; j++) {
                    const int i = c * F::PER_CHUNK + lane * F::CPW + j;
                    ra[c][j] = c < nch ? ta[i] : 0.f;
                    rb[c][j] = (IS_L2 && c < nch) ? tb[i] : 0.f;
                }
            for (int v0 = warp * 32; v0 < len; v0 += kScanWarps * 32) {
                float vals[32];
#pragma unroll
                for (int b16 = 0; b16 < 2; b16++) {
#pragma unroll
                    for (int c = 0; c < F::MAXCH; c++) {
                        if (c < nch) {
                            unsigned y[16];
#pragma unroll
                            for (int j = 0; j < 16; j++) {
                                const int v = min(v0 + b16 * 16 + j, len - 1); // clamped tail, masked at add()
                                y[j] = __ldg(reinterpret_cast<const unsigned*>(base + (int64_t)v * codeSize + c * 128) + lane);
                            }
#pragma unroll
                            for (int j = 0; j < 16; j++) {
                                float acc = c == 0 ? 0.f : vals[b16 * 16 + j];
#pragma unroll
                                for (int e = 0; e < F::CPW; e++) {
                                    const float cv = sq_word_comp<CODEC>(y[j], e);
                                    if (IS_L2) {
                                        const float t = fmaf(-rb[c][e], cv, ra[c][e]);
                                        acc = fmaf(t, t, acc);
                                    } else {
                                        acc = fmaf(ra[c][e], cv, acc);
                                    }
                                }
                                vals[b16 * 16 + j] = acc;
                            }
                        }
                    }
                }
#pragma unroll
                for (int s = 16; s >= 1; s >>= 1) {
#pragma unroll
                    for (int j = 0; j < s; j++) {
                        const bool up = (lane & s) != 0;
                        const float send = up ? vals[j] : vals[j + s];
                        const float keep = up ? vals[j + s] : vals[j];
                        vals[j] = keep + __shfl_xor_sync(kFullMask, send, s);
                    }
                }
                w.add(v0 + lane < len && slotSelected<MASKED>(slotMask, ls + v0), IS_L2 ? vals[0] : -(vals[0] + Kp),
                      (IdT)(ls + v0 + lane));
            }
        } else {
            // generic path: lane = vector, components in order; the table reads are shared-memory broadcasts
            for (int v0 = warp * 32; v0 < len; v0 += kScanWarps * 32) {
                const int v = v0 + lane;
                const bool valid = v < len;
                const uint8_t* cp = base + (int64_t)(valid ? v : len - 1) * codeSize;
                float acc = 0.f;
                for (int i = 0; i < d; i++) {
                    const float cv = sq_row_comp<CODEC>(cp, i);
                    if (IS_L2) {
                        const float t = fmaf(-tb[i], cv, ta[i]);
                        acc = fmaf(t, t, acc);
                    } else {
                        acc = fmaf(ta[i], cv, acc);
                    }
                }
                w.add(valid && slotSelected<MASKED>(slotMask, ls + v0), IS_L2 ? acc : -(acc + Kp), (IdT)(ls + v));
            }
        }
    }
    block_merge_and_write<IdT>(w, warp, lists, perWarp, LIST, k, arenaIds, 0.f, oD, oI);
}

size_t ivfSqScanTableBytes(int d) {
    return round_up(sizeof(float) * (2 * d + kScanWarps), 16);
}

void runIvfSqScan(GpuResources* res, int device, const IvfScanLayout& a, const IvfScanCall& c) {
    const int d = a.d, k = c.k, nprobe = c.nprobe, codeSize = a.codeSize, codec = a.sqCodec;
    const int bits = codec == SQC_BYTE ? 8 : codec == SQC_NIBBLE ? 4 : codec == SQC_SIX ? 6 : 16;
    const int maxch = codec == SQC_HALF ? SqFast<SQC_HALF>::MAXCH : SqFast<SQC_BYTE>::MAXCH;
    const int fast = codec != SQC_SIX && (codeSize & 127) == 0 && (int64_t)d * bits == (int64_t)codeSize * 8 &&
            (codeSize >> 7) <= maxch;
    const int LIST = std::max(64, next_pow2(k));
    const bool wide = ivfScanWideIds(a);
    const size_t listBytes = wide ? SmemTopK<long long>::bytes(LIST, kScanBuf) : SmemTopK<int>::bytes(LIST, kScanBuf);
    const size_t smem = ivfSqScanTableBytes(d) + listBytes * kScanWarps;
    FB_THROW_IF_NOT_MSG(smem <= 220 * 1024, "k / d too large for the IVF-SQ scan kernel");
    // lists of residuals (centroids set): L2 scans q - c_list, IP adds the coarse distance
    const bool l2 = c.metric == METRIC_L2;
    const float* coarse = l2 ? a.centroids : nullptr;
    const float* cdis = (!l2 && a.centroids) ? c.coarseDis : nullptr;
    runIvfScanBatches(res, device, c, false, "ivfsq_scan", [&](const IvfScanBatch& b) {
        withInt<SQC_BYTE, SQC_NIBBLE, SQC_SIX, SQC_HALF>(codec, [&](auto cc) {
            withBool(l2, [&](auto isL2) {
                withBool(wide, [&](auto wideIds) {
                    withBool(c.mask != nullptr, [&](auto masked) {
                        auto kern = ivfsq_scan_kernel<cc, isL2, ScanIdT<decltype(wideIds)>, masked>;
                        CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                        kern<<<b.grid, kScanWarps * 32, smem, c.stream>>>(
                                c.Q + b.q0 * d, d, c.probes + b.q0 * nprobe, cdis ? cdis + b.q0 * nprobe : nullptr,
                                nprobe, b.probesPerCta, coarse, a.sqDecodeMB, a.listStart, a.listLen, a.codes, a.ids,
                                codeSize, fast, k, LIST, b.partD, b.partI, c.mask);
                    });
                });
            });
        });
    });
}

} // namespace fb200
