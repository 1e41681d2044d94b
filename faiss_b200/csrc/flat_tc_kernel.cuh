// faiss_b200 -- the wgmma Flat scoring + filter kernel (included by flat_tc.cu).
//
// Roles in one persistent CTA (2 consumer warpgroups + 1 producer warp = 288 threads, one CTA per SM):
//   warps 0-7 : two consumer warpgroups.  A work unit is one 128-query tile; warpgroup g owns its query rows
//               64 g .. 64 g + 63.  For every database tile it issues wgmma.m64n256k16 (fp16 operands straight
//               from the 128B-swizzled shared-memory stages, fp32 accumulators in registers: 128 per thread),
//               waits for them, hands the stage back and filters its own accumulator fragment (below).  At
//               112 < d <= 128 (PIPE) a tile runs as two N = 128 chains, A (columns 0-127) and B (128-255), each
//               reading its own half-tile stage, and the warpgroup is software-pipelined: it filters A(t) while
//               B(t) runs and B(t) while A(t + 1) runs, so it always has MMAs of its own in flight.  Otherwise a
//               warpgroup's own MMAs and filter do not overlap.  The two warpgroups share the ring without
//               synchronising with each other, so one's tensor work can also overlap the other's filter.  Survivors
//               (rare) are appended with plain stores to a thread-private candidate segment; scores never reach HBM.
//   warp 8    : TMA producer -- the unit's query tile once, then database tiles (256 rows x dpad fp16, or PIPE: two
//               128-row halves of one, 128B-swizzled K-major) through an mbarrier ring.
// Nine warps put three on one scheduler, which caps a thread at 168 registers: the 128 accumulators plus the filter
// state fit without spills.
//
// A thread's fragment holds two query rows (r and r + 8) and, of each, the 64 columns 8 j + 2 (lane % 4) + {0, 1}:
// the four lanes of a quad split a row's 256 columns, which is why a query row has kParts = 4 candidate segments.
#pragma once

#include <cuda_fp16.h>

#include "flat_tc_schedule.h" // kUnitM, kTileN, kParts, kSegsPerUnit
#include "select.cuh"
#include "tc_ptx.cuh"

namespace fb200 {
namespace tc {

constexpr int kTileM = kUnitM;    // queries per work unit (the query tile)
constexpr int kWgM = 64;          // query rows per consumer warpgroup (wgmma M)
constexpr int kHalfN = kTileN / 2; // PIPE: database rows per ring stage and per MMA chain
constexpr int kKBlock = 64;       // fp16 elements per 128-byte swizzle row
constexpr int kConsumerWarps = 8; // two warpgroups
constexpr int kTcThreads = 32 * kConsumerWarps + 32;
constexpr int kMaxYStages = 6;

struct TcParams {
    int numUnits;
    int slices;
    int qPairs;         // number of query units; unit u = slice * qPairs + qunit: neighbouring CTAs stream the SAME database tiles (L2 reuse)
    int tileBegin;      // permuted position range of this round
    int tileEnd;
    int tilesPerSlice;
    unsigned long long permA, permB, numTiles;
    int KB;             // dpad / 64
    int kSteps;         // ceil(d / 16): 16-wide MMA K-steps that hold data; the zero padding up to dpad is never issued
    int ksplit;         // 1: a ring stage holds ONE 64-wide K-block of a database tile (128 < d <= 256), else a whole tile
    int yStages;
    const float* invScalePtr; // device scalar: 1 / (qScale * yScale)
    const float* bias;  // [numTiles*256], -inf padded (read on the slow path only)
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
};

// The pipelined consumer (PIPE) needs exactly 8 K-steps in one 2-K-block stage: 112 < d <= 128.  Its K-step count must
// be a compile-time constant: with a run-time count ptxas cannot tell which wgmma group is in flight and serialises
// every MMA.
__host__ __device__ constexpr bool tc_pipelined(int KB, int kSteps) {
    return KB == 2 && kSteps == 2 * kKBlock / 16;
}

__device__ __forceinline__ int perm_tile(const TcParams& p, int pos) {
    return (int)(((unsigned long long)pos * p.permA + p.permB) % p.numTiles);
}

// column of element e of a 32-element chunk, relative to the chunk's first column (fragment layout above)
__device__ __forceinline__ int chunk_col(int e) {
    return 8 * (e >> 1) + (e & 1);
}

// Filter of one query row against 32 of its columns (database rows).
//
// The exact test is  score = fma(acc, inv, bias[row]) > thr.  The database tiles hold rows SORTED BY
// NORM, so the biases of a tile are nearly equal and  bound = fma(max acc, inv, max bias of the tile)
// is a tight upper bound of every score in a group (inv > 0 and rounding are monotonic: no false
// negatives, bit for bit).  The fast path is therefore a pure max tree over raw accumulators --
// no bias loads, no per-element FMA -- plus one FMA per 32 columns; the rare group whose bound beats
// the threshold evaluates the exact test with biases read through L1/L2.
template <bool DUMP, bool SELF>
__device__ __forceinline__ void epi_filter32(
        const TcParams& p,
        const float (&r)[32],
        int q,
        long long colBase, // global (sorted) row index of element 0 of this chunk
        float inv,
        float& thr,  // SELF: tightened in place (running maximum minus the slack)
        float slack, // SELF: 2 * eps of this query
        float maxb,
        uint2* buf,
        int& cnt,
        float minb = 0.f) { // SELF: min bias of the tile
    if (DUMP) {
        if (q < p.nq) {
            float* dst = p.dump + (long long)q * p.dumpLd + colBase;
#pragma unroll
            for (int j = 0; j < 32; j++)
                dst[chunk_col(j)] = r[j];
        }
        return;
    }
    float mg[4];
#pragma unroll
    for (int g = 0; g < 4; g++) {
        const int o = 8 * g;
        const float a = fmaxf(fmaxf(r[o + 0], r[o + 1]), fmaxf(r[o + 2], r[o + 3]));
        const float c = fmaxf(fmaxf(r[o + 4], r[o + 5]), fmaxf(r[o + 6], r[o + 7]));
        mg[g] = fmaxf(a, c);
    }
    const float m = fmaxf(fmaxf(mg[0], mg[1]), fmaxf(mg[2], mg[3]));
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
            if (fmaf(mg[g], inv, maxb) > thr) {
#pragma unroll
                for (int j = 8 * g; j < 8 * g + 8; j++) {
                    const float v = fmaf(r[j], inv, __ldg(bias + chunk_col(j)));
                    if (v > thr) {
                        if (cnt < p.cap)
                            buf[cnt] = make_uint2(__float_as_uint(v), rowBase + chunk_col(j));
                        cnt++;
                        if (SELF) // k = 1: nothing scoring <= v - 2 eps can be the exact argmin any more
                            thr = fmaxf(thr, nextafterf(v - slack, -CUDART_INF_F));
                    }
                }
            }
        }
    }
}

// SELF (k = 1 streaming mode, used for k-means assignment): one pass over all tiles, every consumer thread keeps
// a running "best approximate score minus 2 eps" threshold for its two queries and emits only the candidates
// that beat it -- about ln(columns per thread) plus the near-ties of the maximum.
// PIPE: tc_pipelined(p.KB, p.kSteps) holds, mapY's box is kHalfN rows and every ring stage holds one half of a tile.
template <bool DUMP, bool SELF = false, bool PIPE = false>
__global__ void __launch_bounds__(kTcThreads, 1) flat_tc_kernel(
        const __grid_constant__ CUtensorMap mapQ,
        const __grid_constant__ CUtensorMap mapY,
        const TcParams p) {
    extern __shared__ unsigned char smem_dyn[];
    // 1024-byte aligned carve-up (SWIZZLE_128B atoms need it)
    unsigned char* smem = reinterpret_cast<unsigned char*>(
            (reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
    const int qBytes = p.KB * kTileM * kKBlock * 2; // the query tile (128 rows)
    // one ring stage: a whole database tile (256 rows x dpad), or -- K-split mode, dpad > 128, where the query tile
    // plus several whole-tile stages no longer fit 227 KB -- one 64-wide K-block of it; PIPE: one 128-row half of a
    // tile, laid out [kblock][128 rows][64] like a whole tile (the K-block stride is 16 KB)
    const int stageBytes = PIPE ? p.KB * kHalfN * kKBlock * 2 : (p.ksplit ? 1 : p.KB) * kTileN * kKBlock * 2;
    unsigned char* sQ = smem;
    unsigned char* sY = smem + qBytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sY + (size_t)p.yStages * stageBytes);
    uint64_t* q_full = bars + 0;
    uint64_t* q_empty = bars + 1;
    uint64_t* y_full = bars + 2;
    uint64_t* y_empty = y_full + kMaxYStages;

    // warp index as a provably warp-uniform value: ptxas then knows every warpgroup reaches its wgmma converged
    // (otherwise it serialises the wgmma chain)
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;

    if (warp == kConsumerWarps && lane == 0) {
        ptx::prefetch_tensormap(&mapQ);
        ptx::prefetch_tensormap(&mapY);
        ptx::mbar_init(q_full, 1);
        ptx::mbar_init(q_empty, kConsumerWarps);
        for (int i = 0; i < p.yStages; i++) {
            ptx::mbar_init(&y_full[i], 1);
            ptx::mbar_init(&y_empty[i], kConsumerWarps);
        }
        ptx::fence_barrier_init();
    }
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
                    // K-split: mapY's box is one K-block; PIPE: it is one half of the tile's rows (the second half of
                    // the last tile may lie wholly past N: TMA zero-fills it and still counts the full box).  Both
                    // warpgroups consume every stage.
                    const int loads = PIPE ? 2 : p.ksplit ? p.KB : 1;
                    for (int l = 0; l < loads; l++) {
                        ptx::mbar_wait(&y_empty[ys], yphase ^ 1);
                        ptx::mbar_arrive_expect_tx(&y_full[ys], (uint32_t)stageBytes);
                        if (PIPE)
                            ptx::tma_load_3d(sY + (size_t)ys * stageBytes, &mapY, &y_full[ys], 0, t * kTileN + l * kHalfN, 0);
                        else
                            ptx::tma_load_3d(sY + (size_t)ys * stageBytes, &mapY, &y_full[ys], 0, t * kTileN, l);
                        if (++ys == p.yStages) {
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
    const int part = lane & 3;
    const int row = wg * kWgM + (warp & 3) * 16 + (lane >> 2); // first of the thread's two rows; the second is row + 8
    const float inv = *p.invScalePtr;
    const uint32_t sQaddr = ptx::smem_u32(sQ) + (uint32_t)(wg * kWgM * kKBlock * 2); // this warpgroup's 64 rows
    const uint32_t sYaddr = ptx::smem_u32(sY);
    const int qkb = kTileM * kKBlock * 2; // bytes per K-block of the query tile
    const int ykb = kTileN * kKBlock * 2; // bytes per K-block of a database tile
    const int hkb = kHalfN * kKBlock * 2; // PIPE: bytes per K-block of a half-tile stage
    const int permStep = (int)(p.permA % p.numTiles);
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; i++)
        acc[i] = 0.f;
    int ys = 0;
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
        const long long seg0 = ((long long)u * kUnitM + row) * kParts + part;
        const long long seg1 = ((long long)u * kUnitM + row + 8) * kParts + part;
        uint2* buf0 = DUMP ? nullptr : p.cand + seg0 * p.cap;
        uint2* buf1 = DUMP ? nullptr : p.cand + seg1 * p.cap;
        int cnt0 = 0, cnt1 = 0;
        const int pb = p.tileBegin + sl * p.tilesPerSlice;
        const int pe = min(p.tileEnd, pb + p.tilesPerSlice);

        // tile ids follow the producer's affine permutation incrementally; the tile's bias bound is
        // fetched one tile ahead (its L2 latency would otherwise sit on the filter's critical path)
        int t = pb < pe ? perm_tile(p, pb) : 0;
        float maxbNext = (!DUMP && pb < pe) ? __ldg(p.tileMaxBias + t) : 0.f;
        float minbNext = (SELF && pb < pe) ? __ldg(p.tileMinBias + t) : 0.f;
        ptx::mbar_wait(q_full, it & 1);

        // the tile being filtered: this thread's first column of it and its bias bounds
        long long colBase = 0;
        float maxb = 0.f, minb = 0.f;
        auto nextTile = [&](int pp) {
            colBase = (long long)t * kTileN + 2 * part;
            maxb = maxbNext;
            minb = minbNext;
            t += permStep;
            if (t >= (int)p.numTiles)
                t -= (int)p.numTiles;
            if (!DUMP && pp + 1 < pe)
                maxbNext = __ldg(p.tileMaxBias + t);
            if (SELF && pp + 1 < pe)
                minbNext = __ldg(p.tileMinBias + t);
        };
        // filter of the tile's columns 128 c .. 128 c + 127 (acc[64 c .. 64 c + 63]) for both of the thread's rows
        auto filterHalf = [&](int c) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                float r[32];
#pragma unroll
                for (int e = 0; e < 32; e++)
                    r[e] = acc[4 * (16 * c + (e >> 1)) + 2 * h + (e & 1)];
                if (h)
                    epi_filter32<DUMP, SELF>(p, r, q1, colBase + 128 * c, inv, thr1, slack1, maxb, buf1, cnt1, minb);
                else
                    epi_filter32<DUMP, SELF>(p, r, q0, colBase + 128 * c, inv, thr0, slack0, maxb, buf0, cnt0, minb);
            }
        };

        if constexpr (PIPE) {
            // ring stages are taken and handed back one half-tile at a time
            auto acquireStage = [&]() {
                ptx::mbar_wait(&y_full[ys], yphase);
                const int s = ys;
                if (++ys == p.yStages) {
                    ys = 0;
                    yphase ^= 1;
                }
                return s;
            };
            auto releaseStage = [&](int s) {
                __syncwarp();
                if (lane == 0) // this warp's share of the stage has been read
                    ptx::mbar_arrive(&y_empty[s]);
            };
            // chain c: columns 128 c .. 128 c + 127 of the tile (the half in stage s) into acc[64 c .. 64 c + 63],
            // committed as one wgmma group.  c must be a compile-time constant at every call.
            auto issueHalf = [&](int c, int s) {
                const uint32_t yaddr = sYaddr + (uint32_t)s * (uint32_t)stageBytes;
                ptx::wgmma_fence_operands<64>(acc + 64 * c);
                ptx::wgmma_fence(); // the accumulators were last read by the filter
#pragma unroll
                for (int ks = 0; ks < 2 * kKBlock / 16; ks++) {
                    const int kb = ks >> 2, k4 = ks & 3;
                    const uint64_t da = ptx::make_smem_desc_sw128(sQaddr + kb * qkb + k4 * 32);
                    const uint64_t db = ptx::make_smem_desc_sw128(yaddr + kb * hkb + k4 * 32);
                    ptx::wgmma_m64n128k16_f16_ss(acc + 64 * c, da, db, ks != 0 ? 1u : 0u);
                }
                ptx::wgmma_commit();
                ptx::wgmma_fence_operands<64>(acc + 64 * c);
            };
            // Iteration pp issues A(pp), filters B(pp - 1) while A(pp) runs, then issues B(pp) and filters A(pp) while
            // B(pp) runs.  Nothing is in flight across the back-edge: ptxas cannot follow a group that is still in
            // flight there and would serialise every MMA, so B(pp) is waited for at the end of the iteration and
            // filtered at the start of the next (the unit's last one after the loop).  A half-stage goes back to the
            // producer as soon as its chain retires.  The filter order per thread -- tile by tile, columns 0-127
            // first -- is that of the unpipelined loop.
            for (int pp = pb; pp < pe; pp++) {
                const int sA = acquireStage();
                issueHalf(0, sA);
                // only A(pp) is in flight, so this returns at once; without it ptxas cannot tell that B(pp - 1) has
                // retired and waits for A(pp) before the filter below
                ptx::wgmma_wait_all_but_one();
                if (pp > pb)
                    filterHalf(1); // B(pp - 1)
                nextTile(pp);
                const int sB = acquireStage();
                issueHalf(1, sB);
                ptx::wgmma_wait_all_but_one(); // A(pp) retired
                ptx::wgmma_fence_operands<64>(acc);
                releaseStage(sA);
                filterHalf(0);
                ptx::wgmma_wait_all(); // B(pp) retired
                ptx::wgmma_fence_operands<64>(acc + 64);
                releaseStage(sB);
            }
            if (pb < pe)
                filterHalf(1); // B of the unit's last tile
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
                filterHalf(0);
                filterHalf(1);
            }
        }
        __syncwarp();
        if (lane == 0) // the query tile may be overwritten
            ptx::mbar_arrive(q_empty);
        if (!DUMP) {
            p.candCount[seg0] = cnt0;
            p.candCount[seg1] = cnt1;
        }
    }
}

} // namespace tc
} // namespace fb200
