// faiss_b200 -- the wgmma Flat scoring + filter kernel (included by flat_tc.cu).
//
// Roles in one persistent CTA (one CTA per SM).  A work unit is one 128-query tile.
//   Two-warpgroup layout (2 consumer warpgroups + 1 producer warp = 288 threads): warpgroup g owns query rows
//               64 g .. 64 g + 63.  For every database tile it issues wgmma.m64n256k16 (fp16 operands straight from
//               the 128B-swizzled shared-memory stages, fp32 accumulators in registers: 128 per thread), waits for
//               them, hands the stage back and filters its own accumulator fragment (below).  Nine warps put three on
//               one scheduler, which caps a thread at 168 registers: the 128 accumulators plus the filter state fit.
//   QUAD layout, 112 < d <= 128 (4 consumer warpgroups + 1 producer warp = 544 threads): warpgroup (g, h) owns query
//               rows 64 g .. 64 g + 63 and columns 128 h .. 128 h + 127 of every database tile.  Ring stages hold
//               128-row halves of a tile; stage s holds half s % 2 and is read by the two warpgroups with h = s % 2.
//               A warpgroup runs one wgmma.m64n128k16 chain per tile (64 accumulators per thread), waits for it,
//               hands the stage back and filters.  While one warpgroup filters, three others have chains to run:
//               the warp schedulers interleave tensor and filter work with no software pipelining.  Seventeen warps
//               put five on one scheduler, which caps a thread at 96 registers: 64 accumulators plus the filter state.
//   The consumer warpgroups share the ring without synchronising with each other.  Survivors (rare) are written to
//   their candidate segment; scores never reach HBM.
//   Last warp: TMA producer -- the unit's query tile once, then database tiles (256 rows x dpad fp16, QUAD: two
//   128-row halves of one, 128B-swizzled K-major) through an mbarrier ring.
//
// A thread's fragment holds two query rows (r and r + 8) and, of each, the columns 8 j + 2 (lane % 4) + {0, 1} of
// the tile: the four lanes of a quad split a row's 256 columns, which is why a query row has kParts = 4 candidate
// segments.  In the two-warpgroup layout one thread writes a segment (plain stores, thread-private count).  In the
// QUAD layout the segment's columns are split between warpgroups (g, 0) and (g, 1), so the two writers take slots
// from a 16-bit shared-memory counter per segment; the candidate SET of a segment is the same, only its order is not.
#pragma once

#include <cuda_fp16.h>

#include <type_traits>

#include "flat_tc_schedule.h" // kUnitM, kTileN, kParts, kSegsPerUnit
#include "select.cuh"
#include "tc_ptx.cuh"

namespace fb200 {
namespace tc {

constexpr int kTileM = kUnitM;    // queries per work unit (the query tile)
constexpr int kWgM = 64;          // query rows per consumer warpgroup (wgmma M)
constexpr int kHalfN = kTileN / 2; // QUAD: database rows per ring stage and per MMA chain
constexpr int kKBlock = 64;       // fp16 elements per 128-byte swizzle row
constexpr int kMaxYStages = 6;
// S8 (int8 operands, QUAD only): a 128-byte swizzle row holds 128 s8, so the query tile and a half-tile stage are 16 KB
// each and twelve stages fit beside them
constexpr int kS8Stages = 12;
// S8 search: the fp32 biases of a stage's 128 rows are copied with its codes, on its y_full barrier, so the filter's
// exact test reads them from shared memory (a bias read from global memory is an HBM round trip the whole warpgroup
// waits on).  The stage's n-th fill (pass n over the ring, yphase = n % 2) puts them in bias slot stage + kS8Stages *
// yphase: twice as many slots as stages, so a warp can hand its stage back before its filter, as without the slots.
// The fill that next writes a slot is two passes later, and it waits for the release of the fill one pass later,
// which every reader of the slot gives only after the MMAs of that fill, which come after its filter of this one.
constexpr int kS8BiasSlotBytes = kHalfN * 4;
constexpr int kS8BiasSlots = 2 * kS8Stages;
// QUAD: one 16-bit candidate count per segment of the unit.  A writer stops counting at its first slot >= cap, so a
// count never exceeds cap + 2 (two writers): caps up to kQuadMaxCap keep it in 16 bits.
constexpr int kQuadCountBytes = kSegsPerUnit * 2;
constexpr int kQuadMaxCap = 65533;

// consumer warps of a layout: two or four warpgroups; the producer warp comes after them
__host__ __device__ constexpr int tc_consumer_warps(bool quad) {
    return quad ? 16 : 8;
}
__host__ __device__ constexpr int tc_threads(bool quad) {
    return 32 * tc_consumer_warps(quad) + 32;
}

struct TcParams {
    int numUnits;
    int slices;
    int qPairs;         // number of query units; unit u = slice * qPairs + qunit: neighbouring CTAs stream the SAME database tiles (L2 reuse)
    int tileBegin;      // permuted position range of this round
    int tileEnd;
    int tilesPerSlice;
    unsigned long long permA, permB, numTiles;
    int permStep;       // permA % numTiles: the tile id step between consecutive positions
    int KB;             // dpad / 64
    int kSteps;         // ceil(d / 16): 16-wide MMA K-steps that hold data; the zero padding up to dpad is never issued
    int ksplit;         // 1: a ring stage holds ONE 64-wide K-block of a database tile (128 < d <= 256), else a whole tile
    int yStages;
    const float* invScalePtr; // device scalar: 1 / (qScale * yScale)
    const float* bias;  // [numTiles*256], -inf padded (read on the slow path only; S8 search: staged, 16-byte aligned)
    const float* tileMaxBias; // [numTiles] max bias of the tile's rows (rows are stored sorted by norm)
    const float* tileMinBias; // [numTiles] min bias of the tile's rows (SELF mode: a lower bound of the chunk's best score)
    const float* thr;   // [nq]  pass if score > thr
    const float* eps;   // [nq]  SELF mode (k = 1 streaming): a passing score v raises the thread's threshold to v - 2 eps
    uint2* cand;        // [numUnits*512][cap] (score bits, row)
    int cap;
    int* candCount;     // [numUnits*512]
    float* dump;        // debug: raw accumulators [nq][dumpLd]
    long long dumpLd;
    int nq;
    const float* invQ;  // S8: [nq] per-query 1 / (s_q * s_y)
};

// The QUAD layout runs exactly 8 K-steps over one 2-K-block half-tile stage: 112 < d <= 128.  The K-step count is a
// compile-time constant there, so the chain is fully unrolled.
__host__ __device__ constexpr bool tc_quad(int KB, int kSteps) {
    return KB == 2 && kSteps == 2 * kKBlock / 16;
}

__device__ __forceinline__ int perm_tile(const TcParams& p, int pos) {
    return (int)(((unsigned long long)pos * p.permA + p.permB) % p.numTiles);
}

// column of element e of a 32-element chunk, relative to the chunk's first column (fragment layout above)
__device__ __forceinline__ int chunk_col(int e) {
    return 8 * (e >> 1) + (e & 1);
}

// Appends the survivors of one candidate segment (one query row, one part) of the unit.
// Everything but cnt is recomputed from kernel-wide values where it is used (survivors are rare): the QUAD consumer
// has 96 registers per thread.
template <bool QUAD>
struct SegmentWriter {
    const TcParams& p;
    const int& unit;
    uint32_t sCounts; // QUAD: shared-memory address of the unit's 16-bit segment counts
    int local;        // the segment within the unit: query row * kParts + part
    int cnt = 0;      // two-warpgroup layout: the segment's count; QUAD: 1 once this writer has met the cap

    __device__ __forceinline__ long long seg() const {
        return (long long)unit * kSegsPerUnit + local;
    }
    // QUAD: the address of the segment's 16-bit count
    __device__ __forceinline__ uint32_t countAddr() const {
        return sCounts + 2u * (uint32_t)local;
    }
    __device__ __forceinline__ void operator()(float v, unsigned col) {
        uint2* buf = p.cand + seg() * p.cap;
        const uint2 c = make_uint2(__float_as_uint(v), col);
        if constexpr (QUAD) {
            if (cnt == 0) {
                const uint32_t a = countAddr();
                const uint32_t sh = 8u * (a & 2u); // the count's half of its 32-bit word
                uint32_t old;
                asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(a & ~3u), "r"(1u << sh) : "memory");
                const int slot = (int)((old >> sh) & 0xffffu);
                if (slot < p.cap)
                    buf[slot] = c;
                else
                    cnt = 1; // a count above cap already flags the segment; stop before the 16 bits could wrap
            }
        } else {
            if (cnt < p.cap)
                buf[cnt] = c;
            cnt++;
        }
    }
    // the segment's count for candCount; QUAD, once every writer is done: also clears the counter for the next unit
    __device__ __forceinline__ int take() {
        if constexpr (QUAD) {
            const uint32_t a = countAddr();
            uint16_t n;
            asm volatile("ld.shared.u16 %0, [%1];" : "=h"(n) : "r"(a) : "memory");
            asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((uint16_t)0) : "memory");
            return n;
        }
        return cnt;
    }
};

// Filter of one query row against 32 of its columns (database rows).  T is the accumulator type: float (fp16 operands)
// or int (s8 operands, where the fast path is an integer max tree and one exact int -> float conversion: |acc| < 2^24).
//
// The exact test is  score = fma(acc, inv, bias[row]) > thr.  The database tiles hold rows SORTED BY
// NORM, so the biases of a tile are nearly equal and  bound = fma(max acc, inv, max bias of the tile)
// is a tight upper bound of every score in a group (inv > 0 and rounding are monotonic: no false
// negatives, bit for bit).  The fast path is therefore a pure max tree over raw accumulators --
// no bias loads, no per-element FMA -- plus one FMA per 32 columns; the rare group whose bound beats
// the threshold evaluates the exact test with biases read through L1/L2 (SMEM_BIAS: from the bias slot at shared
// address sBias, which holds the 128 rows from colBase rounded down to a multiple of 128) and hands every survivor
// (score, global row) to emit.
__device__ __forceinline__ float tc_max(float a, float b) {
    return fmaxf(a, b);
}
__device__ __forceinline__ int tc_max(int a, int b) {
    return max(a, b);
}

template <bool DUMP, bool SELF, bool SMEM_BIAS = false, typename T, typename Emit>
__device__ __forceinline__ void epi_filter32(
        const TcParams& p,
        const T (&r)[32],
        int q,
        long long colBase, // global (sorted) row index of element 0 of this chunk
        float inv,
        float& thr,  // SELF: tightened in place (running maximum minus the slack)
        float slack, // SELF: 2 * eps of this query
        float maxb,
        float minb,  // SELF: min bias of the tile
        Emit&& emit,
        uint32_t sBias = 0) {
    if (DUMP) {
        if (q < p.nq) {
            float* dst = p.dump + (long long)q * p.dumpLd + colBase;
#pragma unroll
            for (int j = 0; j < 32; j++)
                dst[chunk_col(j)] = (float)r[j];
        }
        return;
    }
    T mg[4];
#pragma unroll
    for (int g = 0; g < 4; g++) {
        const int o = 8 * g;
        const T a = tc_max(tc_max(r[o + 0], r[o + 1]), tc_max(r[o + 2], r[o + 3]));
        const T c = tc_max(tc_max(r[o + 4], r[o + 5]), tc_max(r[o + 6], r[o + 7]));
        mg[g] = tc_max(a, c);
    }
    const float m = (float)tc_max(tc_max(mg[0], mg[1]), tc_max(mg[2], mg[3]));
    if (SELF) {
        // the chunk's best row scores at least fma(m, inv, min bias of the tile) (monotone rounding, bias >= minb):
        // the running "best - 2 eps" threshold can be raised BEFORE any per-element work, so the slow path below
        // only looks at the groups that can still hold the new best or its near-ties
        thr = fmaxf(thr, nextafterf(fmaf(m, inv, minb) - slack, -CUDART_INF_F));
    }
    if (fmaf(m, inv, maxb) > thr) {
        const float* bias = p.bias + colBase;
        const unsigned rowBase = (unsigned)colBase;
#pragma unroll
        for (int g = 0; g < 4; g++) {
            if (fmaf((float)mg[g], inv, maxb) > thr) {
                // SMEM_BIAS: elements j, j + 1 (neighbouring columns) take their biases as one pair
                const uint32_t slotCol0 = sBias + 4u * (rowBase % kHalfN);
                float2 pair;
#pragma unroll
                for (int j = 8 * g; j < 8 * g + 8; j++) {
                    float b;
                    if constexpr (SMEM_BIAS) {
                        if ((j & 1) == 0)
                            pair = ptx::lds64f(slotCol0 + 4u * (uint32_t)chunk_col(j));
                        b = (j & 1) ? pair.y : pair.x;
                    } else {
                        b = __ldg(bias + chunk_col(j));
                    }
                    const float v = fmaf((float)r[j], inv, b);
                    if (v > thr) {
                        emit(v, rowBase + chunk_col(j));
                        if (SELF) // k = 1: nothing scoring <= v - 2 eps can be the exact argmin any more
                            thr = fmaxf(thr, nextafterf(v - slack, -CUDART_INF_F));
                    }
                }
            }
        }
    }
}

// SELF (k = 1 streaming mode, used for k-means assignment): one pass over all tiles, every consumer thread keeps
// a running "best approximate score minus 2 eps" threshold for its two queries over its own columns and emits only
// the candidates that beat it -- about ln(columns per thread) plus the near-ties of the maximum.
// QUAD: tc_quad(p.KB, p.kSteps) holds, mapY's box is kHalfN rows, p.yStages == kMaxYStages and every ring stage holds one
// half of a tile; the dynamic shared memory ends with kQuadCountBytes of segment counters.
// S8 (QUAD, not SELF): int8 operands, 128 per swizzle row (one K-block: d <= 128), kS8Stages stages of 16 KB, four
// m64n128k32 K-steps per half-tile, exact int32 accumulators, a per-query p.invQ in place of p.invScalePtr.  The search
// (not DUMP) copies each half-tile's 128 biases into the bias ring, kS8BiasSlots slots of kS8BiasSlotBytes behind the
// segment counters at the end of the dynamic shared memory.
template <bool DUMP, bool SELF = false, bool QUAD = false, bool S8 = false>
__global__ void __launch_bounds__(tc_threads(QUAD), 1) flat_tc_kernel(
        const __grid_constant__ CUtensorMap mapQ,
        const __grid_constant__ CUtensorMap mapY,
        const TcParams p) {
    constexpr int kConsumerWarps = tc_consumer_warps(QUAD);
    extern __shared__ unsigned char smem_dyn[];
    // 1024-byte aligned carve-up (SWIZZLE_128B atoms need it)
    unsigned char* smem = reinterpret_cast<unsigned char*>(
            (reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
    // QUAD runs at KB = 2 with kMaxYStages stages: compile-time sizes spare the consumers registers
    static_assert(!S8 || (QUAD && !SELF), "int8 scoring runs the QUAD layout outside streaming mode");
    constexpr int kStages = S8 ? kS8Stages : kMaxYStages; // barrier slots
    const int KB = S8 ? 1 : QUAD ? 2 : p.KB;
    const int yStages = QUAD ? kStages : p.yStages;
    const int qBytes = KB * kTileM * kKBlock * 2; // the query tile (128 rows; S8: 128 rows x 128 s8)
    // one ring stage: a whole database tile (256 rows x dpad), or -- K-split mode, dpad > 128, where the query tile
    // plus several whole-tile stages no longer fit 227 KB -- one 64-wide K-block of it; QUAD: one 128-row half of a
    // tile, laid out [kblock][128 rows][64] like a whole tile (the K-block stride is 16 KB)
    const int stageBytes = QUAD ? KB * kHalfN * kKBlock * 2 : (p.ksplit ? 1 : KB) * kTileN * kKBlock * 2;
    unsigned char* sQ = smem;
    unsigned char* sY = smem + qBytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sY + (size_t)yStages * stageBytes);
    uint64_t* q_full = bars + 0;
    uint64_t* q_empty = bars + 1;
    uint64_t* y_full = bars + 2;
    uint64_t* y_empty = y_full + kStages;
    // QUAD: 16-bit candidate counts of the unit's segments, behind the 512 bytes of barriers
    uint32_t* segCount = reinterpret_cast<uint32_t*>(reinterpret_cast<unsigned char*>(bars) + 512);
    const uint32_t sCounts = ptx::smem_u32(segCount);
    // S8 search: the bias ring behind the counts (the raw-score dump reads no biases)
    constexpr bool kStageBias = S8 && !DUMP;
    unsigned char* sBias = reinterpret_cast<unsigned char*>(segCount) + kQuadCountBytes;

    // warp index as a provably warp-uniform value: ptxas then knows every warpgroup reaches its wgmma converged
    // (otherwise it serialises the wgmma chain)
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;

    if (warp == kConsumerWarps && lane == 0) {
        ptx::prefetch_tensormap(&mapQ);
        ptx::prefetch_tensormap(&mapY);
        ptx::mbar_init(q_full, 1);
        ptx::mbar_init(q_empty, kConsumerWarps);
        for (int i = 0; i < yStages; i++) {
            ptx::mbar_init(&y_full[i], 1);
            ptx::mbar_init(&y_empty[i], 8); // the eight warps (two warpgroups) that read a stage
        }
        ptx::fence_barrier_init();
    }
    if (QUAD && !DUMP)
        for (int i = threadIdx.x; i < kQuadCountBytes / 4; i += blockDim.x)
            segCount[i] = 0;
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ================================ TMA producer ================================
        if (lane == 0) {
            int ys = 0;
            uint32_t yphase = 0;
            int it = 0;
            for (int u = blockIdx.x; u < p.numUnits; u += gridDim.x, it++) {
                const int qunit = u % p.qPairs;
                const int sl = u / p.qPairs;
                ptx::mbar_wait(q_empty, (it & 1) ^ 1);
                ptx::mbar_arrive_expect_tx(q_full, (uint32_t)qBytes);
                ptx::tma_load_3d(sQ, &mapQ, q_full, 0, qunit * kUnitM, 0);
                const int pb = p.tileBegin + sl * p.tilesPerSlice;
                const int pe = min(p.tileEnd, pb + p.tilesPerSlice);
                for (int pp = pb; pp < pe; pp++) {
                    const int t = perm_tile(p, pp);
                    // K-split: mapY's box is one K-block; QUAD: it is one half of the tile's rows (the second half of
                    // the last tile may lie wholly past N: TMA zero-fills it and still counts the full box)
                    const int loads = QUAD ? 2 : p.ksplit ? KB : 1;
                    for (int l = 0; l < loads; l++) {
                        ptx::mbar_wait(&y_empty[ys], yphase ^ 1);
                        ptx::mbar_arrive_expect_tx(&y_full[ys], (uint32_t)(stageBytes + (kStageBias ? kS8BiasSlotBytes : 0)));
                        if (QUAD)
                            ptx::tma_load_3d(sY + (size_t)ys * stageBytes, &mapY, &y_full[ys], 0, t * kTileN + l * kHalfN, 0);
                        else
                            ptx::tma_load_3d(sY + (size_t)ys * stageBytes, &mapY, &y_full[ys], 0, t * kTileN, l);
                        if constexpr (kStageBias)
                            ptx::bulk_load_1d(sBias + (ys + kS8Stages * yphase) * kS8BiasSlotBytes,
                                              p.bias + (size_t)t * kTileN + l * kHalfN, kS8BiasSlotBytes, &y_full[ys]);
                        if (++ys == yStages) {
                            ys = 0;
                            yphase ^= 1;
                        }
                    }
                }
            }
        }
        return;
    }

    // ================================ consumers ================================
    const int wg = warp >> 2;
    const int g = QUAD ? (wg & 1) : wg; // query half
    const int h = QUAD ? (wg >> 1) : 0; // QUAD: column half of every tile (and of the ring)
    const int part = lane & 3;
    const int row = g * kWgM + (warp & 3) * 16 + (lane >> 2); // first of the thread's two rows; the second is row + 8
    const float inv = S8 ? 0.f : *p.invScalePtr;
    const uint32_t sQaddr = ptx::smem_u32(sQ) + (uint32_t)(g * kWgM * kKBlock * 2); // this warpgroup's 64 rows
    const uint32_t sYaddr = ptx::smem_u32(sY);
    const int qkb = kTileM * kKBlock * 2; // bytes per K-block of the query tile
    const int ykb = kTileN * kKBlock * 2; // bytes per K-block of a database tile
    const int hkb = kHalfN * kKBlock * 2; // QUAD: bytes per K-block of a half-tile stage
    constexpr int kAcc = QUAD ? 64 : 128;
    using Acc = std::conditional_t<S8, int, float>;
    Acc acc[kAcc];
#pragma unroll
    for (int i = 0; i < kAcc; i++)
        acc[i] = 0;
    // QUAD: this warpgroup's sub-ring is stages h, h + 2, h + 4, ...
    int ys = h;
    uint32_t yphase = 0;
    int it = 0;
    for (int u = blockIdx.x; u < p.numUnits; u += gridDim.x, it++) {
        const int qunit = u % p.qPairs;
        const int sl = u / p.qPairs;
        // per-thread filter state for its two queries
        const int q0 = qunit * kUnitM + row;
        const int q1 = q0 + 8;
        float thr0 = (!DUMP && q0 < p.nq) ? p.thr[q0] : CUDART_INF_F;
        float thr1 = (!DUMP && q1 < p.nq) ? p.thr[q1] : CUDART_INF_F;
        const float slack0 = (SELF && q0 < p.nq) ? 2.f * p.eps[q0] : 0.f;
        const float slack1 = (SELF && q1 < p.nq) ? 2.f * p.eps[q1] : 0.f;
        const float inv0 = S8 ? (!DUMP && q0 < p.nq ? p.invQ[q0] : 0.f) : inv;
        const float inv1 = S8 ? (!DUMP && q1 < p.nq ? p.invQ[q1] : 0.f) : inv;
        SegmentWriter<QUAD> w0{p, u, sCounts, row * kParts + part};
        SegmentWriter<QUAD> w1{p, u, sCounts, (row + 8) * kParts + part};
        const int pb = p.tileBegin + sl * p.tilesPerSlice;
        const int pe = min(p.tileEnd, pb + p.tilesPerSlice);

        // tile ids follow the producer's affine permutation incrementally; the tile's bias bound is
        // fetched one tile ahead (its L2 latency would otherwise sit on the filter's critical path)
        int t = pb < pe ? perm_tile(p, pb) : 0;
        float maxbNext = (!DUMP && pb < pe) ? __ldg(p.tileMaxBias + t) : 0.f;
        float minbNext = (SELF && pb < pe) ? __ldg(p.tileMinBias + t) : 0.f;
        ptx::mbar_wait(q_full, it & 1);

        // the tile being filtered and its bias bounds
        int tile = 0;
        float maxb = 0.f, minb = 0.f;
        auto nextTile = [&](int pp) {
            tile = t;
            maxb = maxbNext;
            minb = minbNext;
            t += p.permStep;
            if (t >= (int)p.numTiles)
                t -= (int)p.numTiles;
            if (!DUMP && pp + 1 < pe)
                maxbNext = __ldg(p.tileMaxBias + t);
            if (SELF && pp + 1 < pe)
                minbNext = __ldg(p.tileMinBias + t);
        };
        // filter of the 128 columns held in acc[64 c .. 64 c + 63] for both of the thread's rows; kStageBias: their
        // biases are in the bias slot at shared address sb
        auto filterHalf = [&](int c, uint32_t sb) {
            // this thread's first column of them
            const long long colBase = (long long)tile * kTileN + kHalfN * (h + c) + 2 * part;
#pragma unroll
            for (int hr = 0; hr < 2; hr++) {
                Acc r[32];
#pragma unroll
                for (int e = 0; e < 32; e++)
                    r[e] = acc[4 * (16 * c + (e >> 1)) + 2 * hr + (e & 1)];
                if (hr)
                    epi_filter32<DUMP, SELF, kStageBias>(p, r, q1, colBase, inv1, thr1, slack1, maxb, minb, w1, sb);
                else
                    epi_filter32<DUMP, SELF, kStageBias>(p, r, q0, colBase, inv0, thr0, slack0, maxb, minb, w0, sb);
            }
        };

        if constexpr (QUAD) {
            // the bias bounds are loaded for the tile at hand: the stage wait and the MMA chain hide their latency,
            // and a bound fetched a tile ahead would cost registers the 96-register budget does not have
            tile = t;
            for (int left = pe - pb; left > 0; left--) {
                maxb = DUMP ? 0.f : __ldg(p.tileMaxBias + tile);
                minb = SELF ? __ldg(p.tileMinBias + tile) : 0.f;
                ptx::mbar_wait(&y_full[ys], yphase);
                const uint32_t yaddr = sYaddr + (uint32_t)ys * (uint32_t)stageBytes;
                ptx::wgmma_fence_operands<64>(acc);
                ptx::wgmma_fence(); // the accumulators were last read by the filter
                if constexpr (S8) {
#pragma unroll
                    for (int ks = 0; ks < 4; ks++) { // 4 x k32 over the 128-byte row
                        const uint64_t da = ptx::make_smem_desc_sw128(sQaddr + ks * 32);
                        const uint64_t db = ptx::make_smem_desc_sw128(yaddr + ks * 32);
                        ptx::wgmma_m64n128k32_s8_ss(acc, da, db, ks != 0 ? 1u : 0u);
                    }
                } else {
#pragma unroll
                    for (int ks = 0; ks < 2 * kKBlock / 16; ks++) {
                        const int kb = ks >> 2, k4 = ks & 3;
                        const uint64_t da = ptx::make_smem_desc_sw128(sQaddr + kb * qkb + k4 * 32);
                        const uint64_t db = ptx::make_smem_desc_sw128(yaddr + kb * hkb + k4 * 32);
                        ptx::wgmma_m64n128k16_f16_ss(acc, da, db, ks != 0 ? 1u : 0u);
                    }
                }
                ptx::wgmma_commit();
                ptx::wgmma_wait_all();
                ptx::wgmma_fence_operands<64>(acc);
                const uint32_t sb = kStageBias ? ptx::smem_u32(sBias) + (uint32_t)((ys + kS8Stages * yphase) * kS8BiasSlotBytes) : 0u;
                __syncwarp();
                if (lane == 0) // this warp's share of the stage has been read
                    ptx::mbar_arrive(&y_empty[ys]);
                ys += 2;
                if (ys >= yStages) {
                    ys -= yStages;
                    yphase ^= 1;
                }
                filterHalf(0, sb);
                tile += p.permStep;
                if (tile >= (int)p.numTiles)
                    tile -= (int)p.numTiles;
            }
        } else {
            for (int pp = pb; pp < pe; pp++) {
                nextTile(pp);
                // ---- scores of the tile: acc = Q[64 rows] . Y[256 rows]^T
                const int stagesPerTile = p.ksplit ? p.KB : 1;
#pragma unroll 1
                for (int kb0 = 0; kb0 < stagesPerTile; kb0++) {
                    ptx::mbar_wait(&y_full[ys], yphase);
                    const uint32_t yaddr = sYaddr + (uint32_t)ys * (uint32_t)stageBytes;
                    // K-steps of this stage (d = 96: 6 of the 8 K-steps of the padded tile -- a quarter of the tensor
                    // work is zeros otherwise)
                    const int ks0 = p.ksplit ? 4 * kb0 : 0;
                    const int ks1 = p.ksplit ? min(p.kSteps, ks0 + 4) : p.kSteps;
                    ptx::wgmma_fence();
#pragma unroll 1
                    for (int ks = ks0; ks < ks1; ks++) {
                        const int kb = ks >> 2, k4 = ks & 3;
                        const uint64_t da = ptx::make_smem_desc_sw128(sQaddr + kb * qkb + k4 * 32);
                        const uint64_t db = ptx::make_smem_desc_sw128(yaddr + (p.ksplit ? 0 : kb * ykb) + k4 * 32);
                        ptx::wgmma_m64n256k16_f16_ss(acc, da, db, ks != 0 ? 1u : 0u);
                    }
                    ptx::wgmma_commit();
                    ptx::wgmma_wait_all();
                    __syncwarp();
                    if (lane == 0) // this warp's share of the stage has been read
                        ptx::mbar_arrive(&y_empty[ys]);
                    if (++ys == p.yStages) {
                        ys = 0;
                        yphase ^= 1;
                    }
                }
                filterHalf(0, 0u);
                filterHalf(1, 0u);
            }
        }
        if (QUAD && !DUMP) {
            // both writers of this query half's segments are done: warpgroup (g, 0) publishes the counts and clears
            // the counters.  Warpgroup (g, 1) counts again only after the next query tile arrives, which needs this
            // warp's q_empty arrival below.
            asm volatile("bar.sync %0, 256;" ::"r"(1 + g) : "memory");
            if (h == 0) {
                p.candCount[w0.seg()] = w0.take();
                p.candCount[w1.seg()] = w1.take();
            }
        }
        __syncwarp();
        if (lane == 0) // the query tile may be overwritten
            ptx::mbar_arrive(q_empty);
        if (!QUAD && !DUMP) {
            p.candCount[w0.seg()] = w0.take();
            p.candCount[w1.seg()] = w1.take();
        }
    }
}

} // namespace tc
} // namespace fb200
