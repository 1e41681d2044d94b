// faiss_b200 -- IVF-PQ scan over the rotated, interleaved-by-32 code layout (see kernels.h).
//
// What it replaces: pqCodeDistances (LUT [nq,nprobe,M,256] written to HBM,
// faiss/gpu/impl/PQCodeDistances-inl.cuh:34-285) + pqScanNoPrecomputedMultiPass (per-thread 32-byte
// strided code loads, every distance written to HBM, PQScanMultiPassNoPrecomputed-inl.cuh:174-270,
// PQCodeLoad.cuh:439-454) + pass1/pass2SelectLists (IVFUtilsSelect1/2.cu).
//
// Bound: HBM (codes: M bytes per scanned vector), co-limited by shared-memory gathers (M lookups per
// vector).  Both limits are attacked by the layout:
//   * a warp reads a 32-vector group as M/16 fully coalesced 512-byte loads;
//   * per lookup the inner loop is PRMT (byte -> LUT row address | lane slot) + LDS + FADD, and the
//     LUT access is bank-conflict-free by construction (lane t reads bank (t + j) % 32).
// LUT and distances never touch HBM; the running top-k stays in shared memory (select.cuh).
#include <cfloat>
#include <type_traits>

#include "ivf_layout.cuh"
#include "ivf_scan.cuh"
#include "kernels.h"
#include "select.cuh"

namespace fb200 {
namespace {

constexpr int kLutSlots = 64; // 256 B per code value
constexpr int kIlvScanWarps = 16;  // warps per scan CTA (ivf_scan.cuh's kScanWarps is the 4-warp scans')
constexpr int kScanMinCtas = 2; // CTAs per SM the scan kernel's register budget is set for (64 registers)

__global__ void pq_scatter_interleaved_kernel(
        const uint8_t* __restrict__ flat,
        const idx_t* __restrict__ ids,
        const idx_t* __restrict__ assign,
        const int* __restrict__ offsets,
        int64_t n,
        int M,
        const int64_t* __restrict__ listStart,
        uint8_t* __restrict__ arenaCodes,
        idx_t* __restrict__ arenaIds) {
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n)
        return;
    const int off = offsets[i];
    if (off < 0)
        return;
    const int64_t ls = listStart[assign[i]];
    uint8_t* base = arenaCodes + ls * M;
    for (int b = lane_id(); b < M; b += 32)
        base[ivfInterleavedByte(off, b, M)] = flat[i * M + b];
    if (lane_id() == 0)
        arenaIds[ls + off] = ids[i];
}

__global__ void pq_list_to_interleaved_kernel(const uint8_t* __restrict__ flat, int64_t len, int M, uint8_t* __restrict__ dst) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= len * M)
        return;
    const int64_t v = e / M;
    const int b = (int)(e - v * M);
    dst[ivfInterleavedByte(v, b, M)] = flat[e];
}

__global__ void pq_list_from_interleaved_kernel(const uint8_t* __restrict__ src, int64_t len, int M, uint8_t* __restrict__ flat) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= len * M)
        return;
    const int64_t v = e / M;
    const int b = (int)(e - v * M);
    flat[e] = src[ivfInterleavedByte(v, b, M)];
}

// PRMT with the generic-mode selector (PTX prmt.b32): nibble n picks byte (n & 7) of {a (0-3), b (4-7)};
// bit 3 of the nibble replicates that byte's sign bit instead (used below to produce zero bytes)
template <unsigned SEL>
__device__ __forceinline__ unsigned prmt(unsigned a, unsigned b) {
    unsigned d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "n"(SEL));
    return d;
}

// ld.shared with a compile-time byte offset: LDS R, [Raddr + imm]
template <int IMM>
__device__ __forceinline__ float lds_f32(unsigned addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(IMM));
    return v;
}

// One CTA = one query x one chunk of its probes, kIlvScanWarps warps.
//
//   * ONE top-k list per CTA (CtaTopK, select.cuh): every warp filters against the CTA-wide k-th key,
//     survivors go to a small per-warp buffer, only the final half-merge runs under a CTA lock.  The list
//     and its threshold live across all probes of the chunk.
//   * LUT = [256 codes][2 buffers][32 slots] fp32 (64 KB): lane t looks byte j of its vector up in slot
//     j ^ t (conflict-free: a permutation of the banks for every j), so a row is 128 B and TWO lookup tables
//     fit where the rotated layout needed one.  L2 probes are therefore processed in PAIRS: barrier, build
//     both tables, barrier, then the 16 warps walk the two lists as one stream of work units (units dealt
//     round-robin across list boundaries) -- one barrier per probe instead of three, and the tail imbalance
//     of a list is amortised over two.  IP (and any list-independent table) needs no barrier at all.
//   * inner loop per lookup: PRMT (code byte -> row, packed per-lane slot byte -> column) + LDS + FADD.
// Keys: L2 -> sum of LUT entries (+ ||x - c||^2 with precomputed tables); IP -> -(q.centroid) - sum.
// SBASE: shared-window address of the dynamic shared memory (0x400 on sm_90: the first KB of the window is
// reserved), folded into the LDS immediate so that the PRMT result IS the address; -1 = unknown (one extra
// IADD per lookup).
// NIB (table-build policy): 4-bit PQ with MQ = 2M sub-quantisers whose nibble pairs are the M code bytes.  The
// 16 x MQ direct entries are built first (into `dir`), then each of the 256 x M table entries is the sum of two
// of them, T'[j][b] = T[2j][b & 15] + T[2j+1][b >> 4]; everything after the build is the 8-bit kernel's.
template <int M, bool IS_L2, bool PRECOMP, typename IdT, int SBASE, bool NIB, bool MASKED>
__global__ void __launch_bounds__(kIlvScanWarps * 32, kScanMinCtas) ivfpq_scan_interleaved_kernel(
        const float* __restrict__ Q,
        int d,
        const idx_t* __restrict__ probes,
        const float* __restrict__ coarseDis,
        int nprobe,
        int probesPerCta,
        const float* __restrict__ coarse,
        const float* __restrict__ pqT, // [256][M][dsub]
        const float* __restrict__ term2, // PRECOMP: [nlist][256][M]
        const int64_t* __restrict__ listStart,
        const int* __restrict__ listLen,
        const uint8_t* __restrict__ arenaCodes,
        const idx_t* __restrict__ arenaIds,
        int k,
        int LIST,
        float* __restrict__ partD,
        idx_t* __restrict__ partI,
        const uint32_t* __restrict__ slotMask) { // MASKED: the selector's arena mask
    static_assert(!PRECOMP || IS_L2, "precomputed tables are an L2 decomposition");
    static_assert(!PRECOMP || !NIB, "no precomputed tables for 4-bit codes");
    static_assert((kIlvScanWarps & (kIlvScanWarps - 1)) == 0, "kIlvScanWarps must be a power of two");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int kThreads = kIlvScanWarps * 32;
    constexpr int kU = M == 32 ? 4 : 8;      // groups of 32 vectors per work unit: 4 KB of codes in flight per warp
    constexpr int H = M / 16;                // 16-byte words per lane and group
    constexpr int kEntriesPerThread = 256 * M / kThreads;
    constexpr int MQ = NIB ? 2 * M : M; // sub-quantisers
    static_assert(256 * M % kThreads == 0, "LUT entries must divide evenly among the threads");
    const int q = blockIdx.y, chunk = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int dsub = d / MQ;
    float* lut = reinterpret_cast<float*>(smem_raw);                 // [256][2][32]
    float* rs = lut + 256 * 64;                                      // [2][d] residuals of the probe pair / [d] query
    float* dir = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(rs) + round_up(sizeof(float) * 2 * d, 16)); // NIB: [2][16][MQ]
    int* ctl = reinterpret_cast<int*>(reinterpret_cast<unsigned char*>(dir) + (NIB ? sizeof(float) * 2 * 16 * MQ : 0));
    float* t1s = reinterpret_cast<float*>(ctl + 2);                  // [2] ||x - c||^2 of the pair (PRECOMP)
    unsigned char* listMem = reinterpret_cast<unsigned char*>(ctl) + 16;
    float* oD = partD + ((int64_t)q * gridDim.x + chunk) * k;
    idx_t* oI = partI + ((int64_t)q * gridDim.x + chunk) * k;

    CtaTopK<IdT> top;
    top.init(listMem, ctl, LIST, k, kIlvScanWarps);
    const unsigned sbase = (unsigned)__cvta_generic_to_shared(lut);
    if (SBASE >= 0 && sbase != (unsigned)SBASE)
        __trap(); // compiled for another shared-window base: refuse to read the wrong addresses
    // per-lane column byte of lookup j: X_j = ((lane ^ j) << 2) | (table << 7).  Three of them travel in one
    // register (byte 3 stays zero and supplies the address's two high bytes), derived per triple with ONE
    // LOP3 from Pbase = X_0 replicated: P_i = Pbase ^ {12i << 2, (12i + 4) ..} -- constants.
    const unsigned t4 = (unsigned)lane << 2;
    // direct LUT entry e = c*M + m from a vector r[d] in shared memory:
    //   L2: ||r|m - y||^2 (r = query - list centroid);  IP / PRECOMP term 3: <r|m, y> (r = query)
    auto entry = [&](const float* r, int e, bool l2form) {
        const int c = e / MQ, m = e - c * MQ;
        const float* cp = pqT + (size_t)e * dsub;
        const float* rp = r + m * dsub;
        float acc = 0.f;
        if ((dsub & 3) == 0) {
            for (int j = 0; j < dsub; j += 4) {
                const float4 cv = __ldg(reinterpret_cast<const float4*>(cp + j));
                const float4 rv = *reinterpret_cast<const float4*>(rp + j);
                if (l2form) {
                    float d0 = rv.x - cv.x, d1 = rv.y - cv.y, d2 = rv.z - cv.z, d3 = rv.w - cv.w;
                    acc = fmaf(d0, d0, acc);
                    acc = fmaf(d1, d1, acc);
                    acc = fmaf(d2, d2, acc);
                    acc = fmaf(d3, d3, acc);
                } else {
                    acc = fmaf(rv.x, cv.x, acc);
                    acc = fmaf(rv.y, cv.y, acc);
                    acc = fmaf(rv.z, cv.z, acc);
                    acc = fmaf(rv.w, cv.w, acc);
                }
            }
        } else {
            for (int j = 0; j < dsub; j++) {
                if (l2form) {
                    float df = rp[j] - __ldg(cp + j);
                    acc = fmaf(df, df, acc);
                } else {
                    acc = fmaf(rp[j], __ldg(cp + j), acc);
                }
            }
        }
        return acc;
    };
    // entry (c, m) of table `buf` -> slots m, m+M, ... (< 32) of the half-row
    auto store = [&](int buf, int e, float val) {
        const int c = e / M, m = e - c * M;
#pragma unroll
        for (int s = 0; s < 32; s += M)
            lut[c * 64 + buf * 32 + s + m] = val;
    };
    // NIB: the 16 x MQ direct entries of table `buf` from r (IP: negated, as the 8-bit tables) ...
    auto directBuild = [&](int buf, const float* r, bool l2form) {
        for (int e = threadIdx.x; e < 16 * MQ; e += kThreads) {
            const float v = entry(r, e, l2form);
            dir[buf * 16 * MQ + e] = l2form ? v : -v;
        }
    };
    // ... and, after a barrier, the 256 x M pair sums
    auto pairBuild = [&](int buf) {
        const float* t = dir + buf * 16 * MQ;
        for (int e = threadIdx.x; e < 256 * M; e += kThreads) {
            const int c = e / M, j = e - c * M;
            store(buf, e, t[(c & 15) * MQ + 2 * j] + t[(c >> 4) * MQ + 2 * j + 1]);
        }
    };

    // 32 vectors (one group, this lane's vector): sum of its M table entries in table `buf` (0 / 1: a runtime
    // value folded into the column bytes, so there is ONE copy of the lookup code in the instruction cache)
    auto groupSum = [&](const uint4 (&c)[H], unsigned Pbase) {
        float a0 = 0.f, a1 = 0.f;
        unsigned P = 0;
#pragma unroll
        for (int j = 0; j < M; j++) {
            const unsigned word = j / 4 % 4 == 0 ? c[j / 16].x : j / 4 % 4 == 1 ? c[j / 16].y : j / 4 % 4 == 2 ? c[j / 16].z : c[j / 16].w;
            if (j % 3 == 0) { // column bytes of lookups j, j+1, j+2
                const unsigned C = ((unsigned)(j) << 2) | (((unsigned)(j + 1) << 2) << 8) | (((unsigned)(j + 2) << 2) << 16);
                P = Pbase ^ (C & 0x007c7c7cu);
            }
            // R = (code byte << 8) | column byte; bytes 2, 3 = byte 3 of P = 0
            unsigned R;
            switch ((j % 4) * 4 + j % 3) {
                case 0: R = prmt<0x7704>(word, P); break;
                case 1: R = prmt<0x7705>(word, P); break;
                case 2: R = prmt<0x7706>(word, P); break;
                case 4: R = prmt<0x7714>(word, P); break;
                case 5: R = prmt<0x7715>(word, P); break;
                case 6: R = prmt<0x7716>(word, P); break;
                case 8: R = prmt<0x7724>(word, P); break;
                case 9: R = prmt<0x7725>(word, P); break;
                case 10: R = prmt<0x7726>(word, P); break;
                case 12: R = prmt<0x7734>(word, P); break;
                case 13: R = prmt<0x7735>(word, P); break;
                default: R = prmt<0x7736>(word, P); break;
            }
            float v;
            if (SBASE >= 0)
                v = lds_f32<(SBASE >= 0 ? SBASE : 0)>(R);
            else
                v = lds_f32<0>(R + sbase);
            if (j < 2) { // start the two chains without adding to zero
                if (j == 0)
                    a0 = v;
                else
                    a1 = v;
            } else if (j & 1) {
                a1 += v;
            } else {
                a0 += v;
            }
        }
        return a0 + a1;
    };
    auto loadGroup = [&](const uint8_t* codes, int g, uint4 (&dst)[H]) {
        const uint4* gp = reinterpret_cast<const uint4*>(codes + (int64_t)g * 32 * M) + lane;
#pragma unroll
        for (int h = 0; h < H; h++)
            dst[h] = __ldg(gp + h * 32);
    };

    // one work unit: kU groups of 32 vectors of one list, looked up in table `buf`
    auto scanUnit = [&](int buf, const uint8_t* codes, int ngroups, int g0, int len, int64_t ls, float add) {
        uint4 cur[kU][H];
#pragma unroll
        for (int u = 0; u < kU; u++)
            loadGroup(codes, min(g0 + u, ngroups - 1), cur[u]); // clamped: tail groups re-read the last one (masked below)
        top.refresh();
        const unsigned Pbase = (t4 | ((unsigned)buf << 7)) * 0x010101u;
#pragma unroll
        for (int u = 0; u < kU; u++) {
            const float sum = groupSum(cur[u], Pbase);
            const int v = (g0 + u) * 32 + lane;
            const float key = (IS_L2 && !PRECOMP) ? sum : sum + add;
            top.add(g0 + u < ngroups && v < len && slotSelected<MASKED>(slotMask, ls + (int64_t)(g0 + u) * 32), key,
                    (IdT)(ls + v));
        }
    };

    // Query-only part, once per CTA.  IP: the whole table (-<x|m, y> does not depend on the list), buffer 0.
    // PRECOMP: term 3 = -2 <x|m, y> for this thread's entries, kept in registers across the probes.
    float t3[PRECOMP ? kEntriesPerThread : 1];
    if (!IS_L2 || PRECOMP) {
        for (int i = threadIdx.x; i < d; i += kThreads)
            rs[i] = Q[(int64_t)q * d + i];
        __syncthreads();
        if (NIB) {
            directBuild(0, rs, false);
            __syncthreads();
            pairBuild(0);
        } else {
#pragma unroll
            for (int i = 0; i < kEntriesPerThread; i++) {
                const int e = threadIdx.x + i * kThreads;
                const float dot = entry(rs, e, false);
                if (PRECOMP)
                    t3[i] = -2.f * dot;
                else
                    store(0, e, -dot);
            }
        }
    }
    __syncthreads(); // list initialised (and the IP table built)

    const int pBegin = chunk * probesPerCta;
    const int pEnd = min(nprobe, pBegin + probesPerCta);
    int base = 0; // work units dealt so far (identical in every warp): unit i belongs to warp i % kIlvScanWarps
    if (IS_L2) {
        for (int p0 = pBegin; p0 < pEnd; p0 += 2) {
            idx_t l[2];
            int len[2];
            int64_t ls[2];
#pragma unroll
            for (int s = 0; s < 2; s++) {
                l[s] = p0 + s < pEnd ? probes[(int64_t)q * nprobe + p0 + s] : -1;
                len[s] = l[s] >= 0 ? listLen[l[s]] : 0;
                ls[s] = l[s] >= 0 ? listStart[l[s]] : 0;
            }
            if (len[0] == 0 && len[1] == 0)
                continue; // block-uniform
            if (!PRECOMP) {
                // only the table build reads rs, and the previous build finished before its closing barrier
                for (int i = threadIdx.x; i < 2 * d; i += kThreads) {
                    const int s = i >= d ? 1 : 0, j = i - s * d;
                    const idx_t ll = s ? l[1] : l[0];
                    rs[i] = ll >= 0 ? Q[(int64_t)q * d + j] - __ldg(coarse + ll * d + j) : 0.f;
                }
            }
            __syncthreads(); // every warp is done with the previous pair's tables; residuals visible
            if (NIB) {
#pragma unroll
                for (int s = 0; s < 2; s++)
                    if (len[s] != 0)
                        directBuild(s, rs + s * d, true);
                __syncthreads();
#pragma unroll
                for (int s = 0; s < 2; s++)
                    if (len[s] != 0)
                        pairBuild(s);
            }
#pragma unroll
            for (int s = 0; s < 2 && !NIB; s++) {
                if (len[s] == 0)
                    continue;
                if (PRECOMP) {
                    // table = T2[list] + term 3 (one coalesced load and one add per entry); term 1 = ||x - c||^2
                    // is recomputed here, so the result does not depend on the caller's coarse distances
                    // (search == search_preassigned bit for bit)
                    const float* t2 = term2 + (size_t)l[s] * 256 * M;
                    float v2[kEntriesPerThread];
#pragma unroll
                    for (int i = 0; i < kEntriesPerThread; i++)
                        v2[i] = __ldg(t2 + threadIdx.x + i * kThreads);
                    if (warp == s) {
                        float part = 0.f;
                        for (int i = lane; i < d; i += 32) {
                            const float df = rs[i] - __ldg(coarse + l[s] * d + i);
                            part = fmaf(df, df, part);
                        }
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1)
                            part += __shfl_xor_sync(kFullMask, part, o);
                        if (lane == 0)
                            t1s[s] = part;
                    }
#pragma unroll
                    for (int i = 0; i < kEntriesPerThread; i++)
                        store(s, threadIdx.x + i * kThreads, v2[i] + t3[i]);
                } else if (dsub == 4) {
                    // every entry of this thread belongs to sub-quantiser m = tid % M (kThreads % M == 0): its slice
                    // of the residual is read from shared memory ONCE per probe, not once per entry
                    const float4 rv = *reinterpret_cast<const float4*>(rs + s * d + (threadIdx.x % M) * 4);
#pragma unroll 8
                    for (int e = threadIdx.x; e < 256 * M; e += kThreads) {
                        const float4 cv = __ldg(reinterpret_cast<const float4*>(pqT + (size_t)e * 4));
                        const float d0 = rv.x - cv.x, d1 = rv.y - cv.y, d2 = rv.z - cv.z, d3 = rv.w - cv.w;
                        float acc = d0 * d0; // same association as entry(): fma chain from 0
                        acc = fmaf(d1, d1, acc);
                        acc = fmaf(d2, d2, acc);
                        acc = fmaf(d3, d3, acc);
                        store(s, e, acc);
                    }
                } else {
#pragma unroll 8
                    for (int e = threadIdx.x; e < 256 * M; e += kThreads)
                        store(s, e, entry(rs + s * d, e, true));
                }
            }
            __syncthreads();
#pragma unroll 1
            for (int s = 0; s < 2; s++) {
                if (len[s] == 0)
                    continue;
                const uint8_t* codes = arenaCodes + ls[s] * (int64_t)M;
                const int ngroups = (len[s] + 31) >> 5;
                const int units = (ngroups + kU - 1) / kU;
                const float add = PRECOMP ? t1s[s] : 0.f;
                for (int u = (warp - base) & (kIlvScanWarps - 1); u < units; u += kIlvScanWarps)
                    scanUnit(s, codes, ngroups, u * kU, len[s], ls[s], add);
                base += units;
            }
        }
    } else {
        for (int p = pBegin; p < pEnd; p++) {
            const idx_t l = probes[(int64_t)q * nprobe + p];
            if (l < 0)
                continue;
            const int len = listLen[l];
            if (len == 0)
                continue;
            const int64_t ls = listStart[l];
            const uint8_t* codes = arenaCodes + ls * (int64_t)M;
            const int ngroups = (len + 31) >> 5;
            const int units = (ngroups + kU - 1) / kU;
            const float add = -coarseDis[(int64_t)q * nprobe + p];
            for (int u = (warp - base) & (kIlvScanWarps - 1); u < units; u += kIlvScanWarps)
                scanUnit(0, codes, ngroups, u * kU, len, ls, add);
            base += units;
        }
    }
    top.finish();
    __syncthreads();
    // the CTA's list -> partial result; list ids are arena positions, user labels only for the k survivors
    for (int j = threadIdx.x; j < k; j += kThreads) {
        const IdT id = top.q.ids[j];
        const bool ok = id != IdLimits<IdT>::max();
        oD[j] = ok ? top.q.keys[j] : CUDART_INF_F;
        oI[j] = ok ? arenaIds[id] : -1;
    }
}

// T2[l][e] (e = c*M + m) = ||y_e||^2 + 2 <centroid_l | m, y_e>
__global__ void ivfpq_term2_kernel(
        const float* __restrict__ coarse, const float* __restrict__ pqT, int64_t nlist, int d, int M, float* __restrict__ term2) {
    const int64_t l = blockIdx.y;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 256 * M)
        return;
    const int dsub = d / M;
    const int m = e % M;
    const float* y = pqT + (size_t)e * dsub;
    const float* c = coarse + l * d + m * dsub;
    float acc = 0.f;
    for (int j = 0; j < dsub; j++) {
        const float yj = y[j];
        acc = fmaf(yj, yj, acc);
        acc = fmaf(2.f * c[j], yj, acc);
    }
    term2[(size_t)l * 256 * M + e] = acc;
}

} // namespace

void runIvfPqPrecomputeTerm2(
        const float* coarse, const float* pqT, int64_t nlist, int d, int M, float* term2, cudaStream_t stream) {
    if (nlist == 0)
        return;
    FB_THROW_IF_NOT_MSG(nlist <= 65535 * 32, "nlist too large for the term-2 precompute grid");
    // grid.y is limited to 65535: fold the lists into (x = entries, y = lists) with y chunks
    for (int64_t l0 = 0; l0 < nlist; l0 += 65535) {
        const int64_t nl = std::min<int64_t>(65535, nlist - l0);
        dim3 grid((unsigned)ceil_div(256 * M, 256), (unsigned)nl);
        ivfpq_term2_kernel<<<grid, 256, 0, stream>>>(coarse + l0 * d, pqT, nl, d, M, term2 + (size_t)l0 * 256 * M);
        CUDA_CHECK_LAST();
    }
}

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
        cudaStream_t stream) {
    if (n == 0)
        return;
    int warps = 8;
    pq_scatter_interleaved_kernel<<<(unsigned)ceil_div(n, warps), warps * 32, 0, stream>>>(
            codesFlat, ids, assign, offsets, n, M, listStart, arenaCodes, arenaIds);
    CUDA_CHECK_LAST();
}

void runIvfPqListToInterleaved(const uint8_t* flat, int64_t len, int M, uint8_t* listCodes, cudaStream_t stream) {
    if (len == 0)
        return;
    pq_list_to_interleaved_kernel<<<(unsigned)ceil_div(len * M, 256), 256, 0, stream>>>(flat, len, M, listCodes);
    CUDA_CHECK_LAST();
}

void runIvfPqListFromInterleaved(const uint8_t* listCodes, int64_t len, int M, uint8_t* flat, cudaStream_t stream) {
    if (len == 0)
        return;
    pq_list_from_interleaved_kernel<<<(unsigned)ceil_div(len * M, 256), 256, 0, stream>>>(listCodes, len, M, flat);
    CUDA_CHECK_LAST();
}

__global__ void smem_base_probe_kernel(unsigned* out) {
    extern __shared__ __align__(16) unsigned char probe_raw[];
    if (threadIdx.x == 0)
        *out = (unsigned)__cvta_generic_to_shared(probe_raw);
}

// shared-window address of dynamic shared memory on this device (probed once)
constexpr int kExpectedSmemBase = 1024;
static int probedSmemBase(int device, cudaStream_t stream) {
    static int cache[64];
    static bool have[64] = {};
    if (device >= 0 && device < 64 && have[device])
        return cache[device];
    unsigned* out = nullptr;
    unsigned h = 0xffffffffu;
    CUDA_VERIFY(cudaMalloc(&out, sizeof(unsigned)));
    CUDA_VERIFY(cudaFuncSetAttribute(smem_base_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    smem_base_probe_kernel<<<1, 32, 100 * 1024, stream>>>(out);
    CUDA_CHECK_LAST();
    CUDA_VERIFY(cudaMemcpyAsync(&h, out, sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    CUDA_VERIFY(cudaFree(out));
    if (device >= 0 && device < 64) {
        cache[device] = (int)h;
        have[device] = true;
    }
    return (int)h;
}

void runIvfPqScanInterleaved(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        int d,
        const idx_t* probes,
        const float* coarseDis,
        int nprobe,
        const float* coarseCentroids,
        const float* pqCentroidsT,
        const float* term2,
        int M,
        bool nibble,
        const int64_t* listStart,
        const int* listLen,
        const uint8_t* arenaCodes,
        const idx_t* arenaIds,
        int64_t arenaElems,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream,
        const uint32_t* slotMask,
        const IvfSlotOutput* slots) {
    if (nq == 0)
        return;
    FB_THROW_IF_NOT(ivfPqInterleavedSupported(M));
    FB_THROW_IF_NOT(!nibble || term2 == nullptr);
    const int LIST = std::max(CtaTopK<int>::BUF, next_pow2(k)); // a sorted buffer (<= BUF entries) is merged into the list
    const bool wide = arenaElems >= (int64_t(1) << 31) - 1; // arena positions need 64-bit list ids
    const int smemBase = probedSmemBase(device, stream);
    const size_t listBytes = wide ? CtaTopK<long long>::bytes(LIST, kIlvScanWarps) : CtaTopK<int>::bytes(LIST, kIlvScanWarps);
    size_t smem = sizeof(float) * 256 * kLutSlots + round_up(sizeof(float) * 2 * d, 16) + 16 + listBytes +
            (nibble ? sizeof(float) * 2 * 16 * 2 * M : 0);
    FB_THROW_IF_NOT_MSG(smem <= 220 * 1024, "LUT + top-k lists do not fit shared memory");
    const bool l2 = metric == METRIC_L2;
    const bool pre = l2 && term2 != nullptr;
    runIvfScanBatches(res, device, nq, nprobe, k, metric, false, "ivfpq_scan", outD, outI, stream, [&](const IvfScanBatch& b) {
        withInt<16, 32>(M, [&](auto m) {
            withBool(nibble, [&](auto nib) {
                withBool(l2, [&](auto isL2) {
                    withBool(pre, [&](auto precomp) {
                        withBool(wide, [&](auto wideIds) {
                            withBool(slotMask != nullptr, [&](auto masked) {
                                // precomputed tables are an L2 decomposition of 8-bit codes (pre implies l2 and !nibble)
                                if constexpr (!precomp || (isL2 && !nib)) {
                                    using IdT = ScanIdT<decltype(wideIds)>;
                                    // any other shared-window base than the expected one: generic addressing
                                    auto kern = smemBase == kExpectedSmemBase
                                            ? ivfpq_scan_interleaved_kernel<m, isL2, precomp, IdT, kExpectedSmemBase, nib, masked>
                                            : ivfpq_scan_interleaved_kernel<m, isL2, precomp, IdT, -1, nib, masked>;
                                    CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                                    kern<<<b.grid, kIlvScanWarps * 32, smem, stream>>>(
                                            Q + b.q0 * d, d, probes + b.q0 * nprobe, coarseDis + b.q0 * nprobe, nprobe,
                                            b.probesPerCta, coarseCentroids, pqCentroidsT, term2, listStart, listLen,
                                            arenaCodes, arenaIds, k, LIST, b.partD, b.partI, slotMask);
                                }
                            });
                        });
                    });
                });
            });
        });
    }, slots);
}

} // namespace fb200
