// faiss_b200 -- Flat L2/IP k-NN on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// Replaces, for the Flat path, the reference chain
//   runDistance<float> (faiss/gpu/impl/Distance.cu:121-405) = cuBLAS SGEMM -> fp32 tile in HBM ->
//   l2SelectMinK (faiss/gpu/impl/L2Select.cu:137-187) -> blockSelectPair second level.
//
// Design (see DESIGN.md "Flat"):
//   * Scoring.  score(q,y) = q.y - ||y||^2/2 (L2; maximise) or q.y (IP).  q and y are rounded to
//     fp16 after a power-of-two scaling; the dot product runs on wgmma.mma_async (fp16 inputs,
//     fp32 accumulate in registers).  |approx - exact| <= eps_q, a rigorous bound from the fp16 rounding
//     model (10 mantissa bits) and the fp32 accumulation.
//   * Fused filter (flat_tc_kernel.cuh).  A persistent warp-specialised kernel: one TMA producer warp
//     (the unit's 128-query tile once per work unit, 256-row database tiles through an mbarrier ring) and
//     two consumer warpgroups that each run 64x256xK wgmma tiles into register accumulators and filter
//     them in place: each thread holds two query rows and 64 of a tile's 256 columns of each, folds the
//     RAW accumulators with a max tree and compares one bound per 32 of them against the query's
//     threshold held in a register -- the fp16 copy
//     is stored sorted by norm, so the tile's maximum bias bounds every row's bias tightly.  Scores
//     never reach HBM; only the rare survivors are appended (plain stores, no atomics) to a
//     thread-private candidate segment.
//   * Thresholds come from geometric rounds over a pseudo-randomly permuted tile order: round 0
//     scans ~40 k rows, round r 3x the rows seen so far; after each round a small kernel folds the new candidates into
//     a per-query sorted base list and sets threshold = (k-th best approx score) - 2*eps_q, which
//     provably keeps every true top-k member.
//   * Certified exact result.  The final kernel re-ranks the base list with the library's canonical
//     fp32 arithmetic (same expression and order as flat_exact.cu) and sorts by (distance, id).
//     Queries whose certificate fails (candidate segment or base list overflow) are recomputed by
//     the exact SIMT kernel -- correctness never depends on the data distribution.
#include <cuda_fp16.h>

#include <cfloat>
#include <cmath>
#include <cub/cub.cuh>
#include <mutex>
#include <vector>

#include "comm.h"
#include "kernels.h"
#include "select.cuh"
#include "tc_ptx.cuh"
#include "flat_tc_kernel.cuh"

namespace fb200 {

void runMergeTopKKeyspace(
        const float*, const idx_t*, int64_t, int, int, int, MetricType, int64_t, float*, idx_t*, cudaStream_t);

namespace {

using namespace tc;

// ------------------------------------------------------------------------------------------
// small helper kernels
// ------------------------------------------------------------------------------------------
// database rows as stored: fp32, or fp16 under GpuIndexFlatConfig::useFloat16 (widened on load; every kernel below
// then runs the same fp32 arithmetic on the widened values)
template <bool YH>
__device__ __forceinline__ float row_load1(const void* base, int64_t idx) {
    if (YH)
        return __half2float(reinterpret_cast<const __half*>(base)[idx]);
    return __ldg(reinterpret_cast<const float*>(base) + idx);
}
template <bool YH>
__device__ __forceinline__ float4 row_load4(const void* base, int64_t idx) { // idx % 4 == 0, row start 8 / 16 B aligned
    if (YH) {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(base) + idx));
        const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
        const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        return make_float4(lo.x, lo.y, hi.x, hi.y);
    }
    return __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + idx));
}

__global__ void absmax_kernel(const void* __restrict__ x, int yHalf, int64_t count, float* out) {
    float m = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        float v = fabsf(yHalf ? row_load1<true>(x, i) : reinterpret_cast<const float*>(x)[i]);
        if (v == v && v <= FLT_MAX) // ignore NaN / inf for the scale
            m = fmaxf(m, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        m = fmaxf(m, __shfl_xor_sync(kFullMask, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f)
        atomicMax(reinterpret_cast<int*>(out), __float_as_int(m)); // non-negative floats order as ints
}

// rows -> fp16 (scaled, zero padded to dpad) + bias + norms ; one warp per row
__global__ void tc_prepare_rows_kernel(
        const void* __restrict__ Y,
        int yHalf,
        int64_t n,
        int d,
        int dpad,
        float scale,
        int isL2,
        const int* __restrict__ perm, // stored position -> source row (null: identity)
        __half* __restrict__ Y16,
        float* __restrict__ bias,
        float* __restrict__ norms) {
    int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n)
        return;
    const int64_t src = (perm ? (int64_t)perm[row] : row) * d;
    __half* dst = Y16 + row * dpad;
    float acc = 0.f;
    for (int i = lane_id(); i < dpad; i += 32) {
        float v = i < d ? (yHalf ? row_load1<true>(Y, src + i) : reinterpret_cast<const float*>(Y)[src + i]) : 0.f;
        acc = fmaf(v, v, acc);
        if (Y16)
            dst[i] = __float2half_rn(v * scale);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        acc += __shfl_xor_sync(kFullMask, acc, o);
    if (lane_id() == 0) {
        if (norms)
            norms[row] = acc;
        if (bias)
            bias[row] = isL2 ? -0.5f * acc : 0.f;
    }
}

__global__ void tc_iota_kernel(int* v, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        v[i] = (int)i;
}

// max bias per 256-row tile (NaN and the -inf padding never win: fmaxf drops NaN, a real row beats -inf), and
// -- at tileMax[numTiles + 1 + t] -- the MIN bias of the tile (-inf for a tile with padding rows or NaN: it then
// simply yields no lower bound), used by the k = 1 streaming mode
__global__ void tc_tile_max_bias_kernel(const float* __restrict__ bias, int64_t numTiles, float* __restrict__ tileMax) {
    int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= numTiles)
        return;
    float m = -CUDART_INF_F, mn = CUDART_INF_F;
    for (int i = lane_id(); i < kTileN; i += 32) {
        const float b = bias[t * kTileN + i];
        m = fmaxf(m, b);
        mn = (b == b) ? fminf(mn, b) : -CUDART_INF_F;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        m = fmaxf(m, __shfl_xor_sync(kFullMask, m, o));
        mn = fminf(mn, __shfl_xor_sync(kFullMask, mn, o));
    }
    if (lane_id() == 0) {
        tileMax[t] = m;
        tileMax[numTiles + 1 + t] = mn;
    }
}

// per-batch query preparation: power-of-two scale from absmax, fp16 conversion, eps, 1/(sq*sy)
__global__ void tc_query_scale_kernel(const float* absmax, float yScale, float* qScaleOut, float* invOut) {
    float m = *absmax;
    float s = 1.f;
    if (m > 0.f) {
        int e;
        frexpf(m, &e);           // m = f * 2^e, f in [0.5,1)
        s = ldexpf(1.f, 14 - e); // m*s in [2^13, 2^14)
    }
    *qScaleOut = s;
    *invOut = 1.f / (s * yScale);
}

__global__ void tc_prepare_queries_kernel(
        const float* __restrict__ Q,
        int64_t nq,
        int d,
        int dpad,
        const float* __restrict__ qScale,
        float c1,
        float c2,
        float yMaxNorm,
        __half* __restrict__ Q16,
        float* __restrict__ eps,
        float* __restrict__ thr) {
    int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= nq)
        return;
    const float scale = *qScale;
    const float* src = Q + row * d;
    __half* dst = Q16 + row * dpad;
    float acc = 0.f;
    for (int i = lane_id(); i < dpad; i += 32) {
        float v = i < d ? src[i] : 0.f;
        acc = fmaf(v, v, acc);
        dst[i] = __float2half_rn(v * scale);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        acc += __shfl_xor_sync(kFullMask, acc, o);
    if (lane_id() == 0) {
        float qn = sqrtf(acc) * 1.0001f;
        // |approx score - score implied by the exact kernel's fp32 distance| <= c1*|q||y| + c2*(|q|+|y|)^2
        // (see DESIGN.md, error model): c1 = fp16 input rounding + fp32 accumulation of q.y, c2 = fp32
        // rounding of the bias (norms), of the final FMA and of the exact kernel's own sum (d terms)
        const float qy = qn + yMaxNorm;
        eps[row] = c1 * qn * yMaxNorm + c2 * qy * qy;
        thr[row] = -CUDART_INF_F;
    }
}

// pending-candidate buffer of the select kernel: a round brings ~(growth-1)*k candidates per query, and
// the cost of a flush is dominated by the merge into the 2k-entry list -- fewer, larger flushes
constexpr int kSelectBuf = 128;

// Fold this round's candidate segments into the per-query base list; set the new threshold.
//   base lists hold (key = -score, id = row) sorted ascending; sentinel = (+inf, INT_MAX)
__global__ void tc_select_kernel(
        int nq,
        int k,
        int LIST,
        int slices,
        int parts,
        const uint2* __restrict__ cand,
        int cap,
        const int* __restrict__ candCount,
        const float* __restrict__ eps,
        float* __restrict__ baseKey, // [nq][LIST]
        int* __restrict__ baseId,    // [nq][LIST]
        float* __restrict__ thr,
        int* __restrict__ flags,
        float* __restrict__ contrib, // sharded search: [2][nq] certified lower bounds for the cross-rank threshold (or null)
        int kFrac) {                 // ceil(k / number of shards)
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = lane_id();
    const int q = blockIdx.x * (blockDim.x >> 5) + warp;
    if (q >= nq)
        return;
    constexpr int BUF = kSelectBuf;
    unsigned char* base = smem_raw + SmemTopK<int>::bytes(LIST, BUF) * warp;
    WarpTopK<int> w;
    w.init(reinterpret_cast<float*>(base), reinterpret_cast<int*>(base + sizeof(float) * (LIST + BUF)), LIST, BUF, LIST);
    // note: selection keeps the LIST best (k = LIST for the queue threshold)
    const float* bk = baseKey + (int64_t)q * LIST;
    const int* bi = baseId + (int64_t)q * LIST;
    // the base list is already sorted (sentinels last): adopt it as the queue's list.  The threshold may
    // have been raised since the list was written (cross-rank pooling): entries it now excludes form a
    // suffix of the sorted list and are dropped here.
    const float thrNow = thr[q];
    for (int e0 = 0; e0 < LIST; e0 += 32) {
        const float kk = bk[e0 + lane];
        const bool keep = -kk > thrNow;
        w.q.keys[e0 + lane] = keep ? kk : CUDART_INF_F;
        w.q.ids[e0 + lane] = keep ? bi[e0 + lane] : IdLimits<int>::max();
    }
    __syncwarp();
    w.thr = w.q.threshold();
    int overflow = 0;
    const int pair = q / kUnitM, prow = q % kUnitM; // row within the unit's 128 query rows
    const int qPairs = (nq + kUnitM - 1) / kUnitM;
    // segment counts are fetched 32 at a time (one per lane): the loop over a query's slices x parts
    // segments would otherwise serialise one L2 round trip per segment, and most segments are empty
    const int nseg = slices * parts;
    for (int s0 = 0; s0 < nseg; s0 += 32) {
        const int si = s0 + lane;
        long long mySeg = 0;
        int myCount = 0;
        if (si < nseg) {
            const int s = si / parts, h = si - s * parts;
            mySeg = ((long long)(s * qPairs + pair) * kUnitM + prow) * parts + h;
            myCount = candCount[mySeg];
        }
        unsigned pending = __ballot_sync(kFullMask, myCount > 0);
        while (pending) {
            const int src = __ffs(pending) - 1;
            pending &= pending - 1;
            int c = __shfl_sync(kFullMask, myCount, src);
            const long long seg = __shfl_sync(kFullMask, mySeg, src);
            if (c > cap) {
                overflow = 1;
                c = cap;
            }
            const uint2* sp = cand + seg * cap;
            for (int e0 = 0; e0 < c; e0 += 32) {
                int e = e0 + lane;
                uint2 v = e < c ? sp[e] : make_uint2(0, 0);
                w.add(e < c, -__uint_as_float(v.x), (int)v.y);
            }
        }
    }
    w.finish();
    // k-th best approximate score -> threshold
    float kthKey = w.q.keys[k - 1];
    int kthId = w.q.ids[k - 1];
    float t = -CUDART_INF_F;
    if (kthId != IdLimits<int>::max()) {
        float s = -kthKey - 2.f * eps[q];
        t = nextafterf(s, -CUDART_INF_F);
    }
    // saturated list: an entry we could not keep might have been >= t
    float lastKey = w.q.keys[LIST - 1];
    int lastId = w.q.ids[LIST - 1];
    if (lastId != IdLimits<int>::max() && -lastKey > t)
        overflow = 1;
    float* ok = baseKey + (int64_t)q * LIST;
    int* oi = baseId + (int64_t)q * LIST;
    for (int j = lane; j < LIST; j += 32) {
        float key = w.q.keys[j];
        int id = w.q.ids[j];
        bool keep = id != IdLimits<int>::max() && (-key > t);
        ok[j] = keep ? key : CUDART_INF_F;
        oi[j] = keep ? id : IdLimits<int>::max();
    }
    if (lane == 0) {
        thr[q] = fmaxf(t, thrNow);
        if (overflow)
            flags[q] = 1;
        if (contrib) {
            // certified lower bounds of true scores: >= k rows of this shard score at least c0, >= kFrac rows at
            // least c1.  Across S shards: max_r c0 and min_r c1 (S * kFrac >= k rows) both bound the global k-th.
            const float e = eps[q];
            const float c0 = kthId != IdLimits<int>::max() ? -kthKey - e : -CUDART_INF_F;
            const int fid = w.q.ids[kFrac - 1];
            const float c1 = fid != IdLimits<int>::max() ? -w.q.keys[kFrac - 1] - e : -CUDART_INF_F;
            contrib[q] = c0;
            contrib[nq + q] = -c1; // max-reduced: -min_r c1 (+inf if any shard cannot vouch for kFrac rows)
        }
    }
}

// ---- threshold selection WITHOUT sorting (k <= 128): the round only needs (a) the k-th best approximate score seen
// so far and (b) the set of entries above the new threshold -- not an ordered list.  One warp per query: the surviving
// base-list entries and the round's candidates are gathered into a per-warp shared-memory array (ballot compaction),
// their order-preserving integer keys are pulled into registers (kSelPerLane per lane), the k-th largest key is found
// by a 32-step bitwise bisection (one compare per register and step + one warp reduction), and the entries above the
// new threshold are written back compacted (unsorted; the exact re-rank orders them).  ~2-3 k instructions per query
// and round instead of the ~15 k of the bitonic list maintenance, and no bank conflicts.
constexpr int kSelCap = 1536;
constexpr int kSelPerLane = kSelCap / 32;
constexpr int kSelWarps = 4;

__global__ void __launch_bounds__(kSelWarps * 32) tc_select_bisect_kernel(
        int nq,
        int k,
        int LIST,
        int slices,
        int parts,
        const uint2* __restrict__ cand,
        int cap,
        const int* __restrict__ candCount,
        const float* __restrict__ eps,
        float* __restrict__ baseKey, // [nq][LIST]  (-score), valid entries first, unsorted
        int* __restrict__ baseId,    // [nq][LIST]
        float* __restrict__ thr,
        int* __restrict__ flags,
        float* __restrict__ contrib,
        int kFrac) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = lane_id();
    const int q = blockIdx.x * kSelWarps + warp;
    if (q >= nq)
        return;
    uint2* buf = reinterpret_cast<uint2*>(smem_raw) + (size_t)warp * kSelCap;
    const float thrNow = thr[q];
    const unsigned lt = (1u << lane) - 1u;
    int E = 0;
    int overflow = 0;
    // (1) the base list: valid entries are packed at the front.  All LIST/32 loads are independent (no early exit)
    // so they overlap; entries a raised threshold excludes are dropped by the final compaction, not here.
    float* bk = baseKey + (int64_t)q * LIST;
    int* bi = baseId + (int64_t)q * LIST;
    {
        constexpr int kMaxListIter = 8; // LIST <= 256
        int ids[kMaxListIter];
        float scs[kMaxListIter];
#pragma unroll
        for (int it = 0; it < kMaxListIter; it++) {
            const int e = it * 32 + lane;
            ids[it] = e < LIST ? bi[e] : IdLimits<int>::max();
            scs[it] = e < LIST ? -bk[e] : 0.f;
        }
#pragma unroll
        for (int it = 0; it < kMaxListIter; it++) {
            const bool valid = ids[it] != IdLimits<int>::max();
            const unsigned m = __ballot_sync(kFullMask, valid);
            if (valid)
                buf[E + __popc(m & lt)] = make_uint2(__float_as_uint(scs[it]), (unsigned)ids[it]);
            E += __popc(m);
        }
    }
    // (2) this round's candidates.  32 segments at a time: a warp scan of their counts gives every lane the offset
    // of ITS segment, then the lanes copy their segments in parallel (one memory round trip per batch of 32
    // segments instead of one per segment -- the gather is latency-bound, not bandwidth-bound).
    const int pair = q / kUnitM, prow = q % kUnitM;
    const int qPairs = (nq + kUnitM - 1) / kUnitM;
    const int nseg = slices * parts;
    for (int s0 = 0; s0 < nseg; s0 += 32) {
        const int si = s0 + lane;
        long long mySeg = 0;
        int myCount = 0;
        if (si < nseg) {
            const int s = si / parts, h = si - s * parts;
            mySeg = ((long long)(s * qPairs + pair) * kUnitM + prow) * parts + h;
            myCount = candCount[mySeg];
            if (myCount > cap) {
                overflow = 1;
                myCount = cap;
            }
        }
        int incl = myCount;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(kFullMask, incl, o);
            if (lane >= o)
                incl += v;
        }
        const int total = __shfl_sync(kFullMask, incl, 31);
        if (total == 0)
            continue;
        if (E + total > kSelCap) { // cannot hold more: certificate lost for this query
            overflow = 1;
            break;
        }
        const uint2* sp = cand + mySeg * cap;
        uint2* dst = buf + E + incl - myCount;
        for (int j = 0; j < myCount; j++)
            dst[j] = sp[j];
        E += total;
    }
    overflow = __any_sync(kFullMask, overflow) ? 1 : 0;
    __syncwarp();
    // (3) order-preserving keys into registers (0 sorts below every float, including -inf)
    unsigned key[kSelPerLane];
#pragma unroll
    for (int i = 0; i < kSelPerLane; i++) {
        const int idx = i * 32 + lane;
        key[i] = idx < E ? float_to_ordered(__uint_as_float(buf[idx].x)) : 0u;
    }
    const int nIter = (E + 31) >> 5;
    // k-th largest key (0 if fewer than kk entries)
    auto kthLargest = [&](int kk) -> unsigned {
        if (E < kk)
            return 0u;
        unsigned T = 0;
#pragma unroll 1
        for (int bit = 31; bit >= 0; bit--) {
            const unsigned c = T | (1u << bit);
            int cnt = 0;
#pragma unroll
            for (int i = 0; i < kSelPerLane; i++)
                if (i < nIter)
                    cnt += key[i] >= c ? 1 : 0;
            cnt = __reduce_add_sync(kFullMask, cnt);
            if (cnt >= kk)
                T = c;
        }
        return T;
    };
    const float e2 = eps[q];
    const unsigned Tk = kthLargest(k);
    float t = -CUDART_INF_F;
    float kthScore = -CUDART_INF_F;
    if (Tk != 0u) {
        kthScore = ordered_to_float(Tk);
        t = nextafterf(kthScore - 2.f * e2, -CUDART_INF_F);
    }
    const float tNew = fmaxf(t, thrNow);
    // (4) survivors -> base list (compacted, unsorted), sentinels behind them
    int W = 0;
#pragma unroll 1
    for (int i = 0; i < nIter; i++) {
        const int idx = i * 32 + lane;
        const uint2 v = idx < E ? buf[idx] : make_uint2(0, 0);
        const bool keep = idx < E && __uint_as_float(v.x) > tNew;
        const unsigned m = __ballot_sync(kFullMask, keep);
        const int pos = W + __popc(m & lt);
        if (keep && pos < LIST) {
            bk[pos] = -__uint_as_float(v.x);
            bi[pos] = (int)v.y;
        }
        W += __popc(m);
    }
    if (W > LIST) {
        overflow = 1; // more entries above the threshold than the list holds: masses of near-ties
        W = LIST;
    }
    for (int j = W + lane; j < LIST; j += 32) {
        bk[j] = CUDART_INF_F;
        bi[j] = IdLimits<int>::max();
    }
    if (contrib) {
        const unsigned Tf = kFrac == k ? Tk : kthLargest(kFrac);
        if (lane == 0) {
            contrib[q] = Tk != 0u ? kthScore - e2 : -CUDART_INF_F;
            contrib[nq + q] = Tf != 0u ? -(ordered_to_float(Tf) - e2) : CUDART_INF_F;
        }
    }
    if (lane == 0) {
        thr[q] = tNew;
        if (overflow)
            flags[q] = 1;
    }
}

// sharded search: fold the all-reduced (max) contributions into the local threshold
__global__ void tc_pooled_thr_kernel(int nq, const float* __restrict__ contrib, const float* __restrict__ eps, float* __restrict__ thr) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq)
        return;
    const float T = fmaxf(contrib[q], -contrib[nq + q]);
    if (T > -CUDART_INF_F) {
        const float t = nextafterf(T - eps[q], -CUDART_INF_F);
        thr[q] = fmaxf(thr[q], t);
    }
}

// exact re-rank of the base list with the canonical fp32 arithmetic; output sorted by (dist, id)
template <bool IS_L2, bool YH>
__global__ void tc_rerank_kernel(
        int nq,
        int d,
        int k,
        int LIST,
        int KL, // output list size (pow2 >= k, >= 64)
        const float* __restrict__ Q,
        const void* __restrict__ Y,
        const int* __restrict__ perm, // stored (norm-sorted) position -> row id; null: identity
        const int* __restrict__ baseId,
        const float* __restrict__ baseKey, // with thr: entries whose approximate score is <= thr[q] are skipped
        const float* __restrict__ thr,     // (the threshold may have been raised after the list was written); or null
        float* __restrict__ outD,
        idx_t* __restrict__ outI) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = lane_id();
    const int q = blockIdx.x * (blockDim.x >> 5) + warp;
    if (q >= nq)
        return;
    constexpr int BUF = 64;
    unsigned char* base = smem_raw + SmemTopK<int>::bytes(KL, BUF) * warp;
    WarpTopK<int> w;
    w.init(reinterpret_cast<float*>(base), reinterpret_cast<int*>(base + sizeof(float) * (KL + BUF)), KL, BUF, k);
    const float* qp = Q + (int64_t)q * d;
    const int* bi = baseId + (int64_t)q * LIST;
    const float tq = thr ? thr[q] : -CUDART_INF_F;
    for (int e0 = 0; e0 < LIST; e0 += 32) {
        int id = bi[e0 + lane];
        const bool present = id != IdLimits<int>::max();
        bool valid = present;
        if (valid && thr)
            valid = -baseKey[(int64_t)q * LIST + e0 + lane] > tq;
        if (valid && perm)
            id = perm[id];
        float acc = 0.f;
        if (valid) {
            const int64_t yo = (int64_t)id * d;
            // canonical order: sequential FMA over the dimension (loads vectorised, math not reordered)
            int i = 0;
            if ((d & 3) == 0) {
                // unrolled: 8 independent 16-byte row loads in flight per lane (the FMA chain stays sequential)
#pragma unroll 8
                for (; i < d; i += 4) {
                    const float4 a4 = *reinterpret_cast<const float4*>(qp + i);
                    const float4 b4 = row_load4<YH>(Y, yo + i);
                    const float aa[4] = {a4.x, a4.y, a4.z, a4.w};
                    const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        if (IS_L2) {
                            float df = aa[u] - bb[u];
                            acc = fmaf(df, df, acc);
                        } else {
                            acc = fmaf(aa[u], bb[u], acc);
                        }
                    }
                }
            }
            for (; i < d; i++) {
                float a = qp[i], b = row_load1<YH>(Y, yo + i);
                if (IS_L2) {
                    float df = a - b;
                    acc = fmaf(df, df, acc);
                } else {
                    acc = fmaf(a, b, acc);
                }
            }
            if (!IS_L2)
                acc = -acc;
        }
        // valid entries are packed at the front of the base list, sentinels behind them.  The list is NOT ordered by
        // score (bisection select), so entries the pooled threshold excludes can sit anywhere: only a group made of
        // sentinels ends the walk.
        if (!__any_sync(kFullMask, present))
            break;
        w.add(valid, acc, id);
    }
    w.finish();
    for (int j = lane; j < k; j += 32) {
        int id = w.q.ids[j];
        bool ok = id != IdLimits<int>::max();
        float key = w.q.keys[j];
        outD[(int64_t)q * k + j] = ok ? (IS_L2 ? key : -key) : (IS_L2 ? FLT_MAX : -FLT_MAX);
        outI[(int64_t)q * k + j] = ok ? (idx_t)id : -1;
    }
}

__global__ void tc_init_base_kernel(float* baseKey, int* baseId, int64_t count) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) {
        baseKey[i] = CUDART_INF_F;
        baseId[i] = IdLimits<int>::max();
    }
}

// k = 1 streaming mode: select + exact re-rank in one pass.  One warp per query: (1) the maximum approximate
// score m over the query's candidate segments, (2) every candidate scoring >= m - 2 eps (typically one to three)
// gets its canonical fp32 distance -- one lane per candidate, sequential FMA over the dimension exactly like
// flat_exact.cu -- (3) the (distance, id) minimum is the answer.  A segment that overflowed flags the query for
// the exact kernel.
template <bool IS_L2, bool YH>
__global__ void tc_argmin_finish_kernel(
        int nq,
        int d,
        int slices,
        int parts,
        const uint2* __restrict__ cand,
        int cap,
        const int* __restrict__ candCount,
        const float* __restrict__ eps,
        const float* __restrict__ Q,
        const void* __restrict__ Y,
        const int* __restrict__ perm,
        float* __restrict__ outD,
        idx_t* __restrict__ outI,
        int* __restrict__ flags) {
    const int warp = threadIdx.x >> 5;
    const int lane = lane_id();
    const int q = blockIdx.x * (blockDim.x >> 5) + warp;
    if (q >= nq)
        return;
    const int pair = q / kUnitM, prow = q % kUnitM;
    const int qPairs = (nq + kUnitM - 1) / kUnitM;
    const int nseg = slices * parts;
    // pass 1: maximum approximate score
    float m = -CUDART_INF_F;
    int overflow = 0;
    for (int si = 0; si < nseg; si++) {
        const int s = si / parts, h = si - s * parts;
        const long long seg = ((long long)(s * qPairs + pair) * kUnitM + prow) * parts + h;
        int c = candCount[seg];
        if (c > cap) {
            overflow = 1;
            c = cap;
        }
        const uint2* sp = cand + seg * cap;
        for (int e = lane; e < c; e += 32)
            m = fmaxf(m, __uint_as_float(sp[e].x));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        m = fmaxf(m, __shfl_xor_sync(kFullMask, m, o));
    const float t = nextafterf(m - 2.f * eps[q], -CUDART_INF_F);
    // pass 2: exact distances of the survivors, best (distance, id)
    float bestD = CUDART_INF_F;
    int bestI = IdLimits<int>::max();
    const float* qp = Q + (int64_t)q * d;
    for (int si = 0; si < nseg; si++) {
        const int s = si / parts, h = si - s * parts;
        const long long seg = ((long long)(s * qPairs + pair) * kUnitM + prow) * parts + h;
        const int c = min(candCount[seg], cap);
        const uint2* sp = cand + seg * cap;
        for (int e0 = 0; e0 < c; e0 += 32) {
            const int e = e0 + lane;
            const uint2 v = e < c ? sp[e] : make_uint2(0, 0);
            if (e < c && __uint_as_float(v.x) > t) {
                int id = (int)v.y;
                if (perm)
                    id = perm[id];
                const int64_t yo = (int64_t)id * d;
                float acc = 0.f;
                for (int i = 0; i < d; i++) {
                    const float a = qp[i], b = row_load1<YH>(Y, yo + i);
                    if (IS_L2) {
                        const float df = a - b;
                        acc = fmaf(df, df, acc);
                    } else {
                        acc = fmaf(a, b, acc);
                    }
                }
                if (!IS_L2)
                    acc = -acc;
                if (acc < bestD || (acc == bestD && id < bestI)) {
                    bestD = acc;
                    bestI = id;
                }
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(kFullMask, bestD, o);
        const int oi = __shfl_xor_sync(kFullMask, bestI, o);
        if (od < bestD || (od == bestD && oi < bestI)) {
            bestD = od;
            bestI = oi;
        }
    }
    if (lane == 0) {
        const bool ok = bestI != IdLimits<int>::max();
        outD[q] = ok ? (IS_L2 ? bestD : -bestD) : (IS_L2 ? FLT_MAX : -FLT_MAX);
        outI[q] = ok ? (idx_t)bestI : -1;
        if (overflow || !ok)
            flags[q] = 1;
    }
}

// compact flagged query indices: list[0..count)
__global__ void tc_collect_flags_kernel(const int* flags, int nq, int* list, int* count) {
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < nq && flags[q]) {
        int pos = atomicAdd(count, 1);
        list[pos] = q;
    }
}
__global__ void tc_gather_queries_kernel(const float* Q, const int* list, int d, float* out) {
    int i = blockIdx.x;
    int q = list[i];
    for (int j = threadIdx.x; j < d; j += blockDim.x)
        out[(int64_t)i * d + j] = Q[(int64_t)q * d + j];
}
__global__ void tc_scatter_results_kernel(
        const float* D,
        const idx_t* I,
        const int* list,
        int k,
        float* outD,
        idx_t* outI) {
    int i = blockIdx.x;
    int q = list[i];
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        outD[(int64_t)q * k + j] = D[(int64_t)i * k + j];
        outI[(int64_t)q * k + j] = I[(int64_t)i * k + j];
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(
        CUtensorMap*,
        CUtensorMapDataType,
        cuuint32_t,
        void*,
        const cuuint64_t*,
        const cuuint64_t*,
        const cuuint32_t*,
        const cuuint32_t*,
        CUtensorMapInterleave,
        CUtensorMapSwizzle,
        CUtensorMapL2promotion,
        CUtensorMapFloatOOBfill);

PFN_encodeTiled getEncodeTiled() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (err == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    FB_THROW_IF_NOT_MSG(fn != nullptr, "cuTensorMapEncodeTiled not available from the driver");
    return fn;
}

// fp16 matrix [rows][dpad] viewed as (64, rows, dpad/64); one box = (64, 128, dpad/64) = a full
// K-extent tile laid out [kblock][row][64] with the 128-byte swizzle the UMMA descriptors expect.
// boxK = 0: the box spans every K-block (a whole tile); boxK = 1: one K-block per copy (K-split database stages).
CUtensorMap makeTileMap(const __half* base, int64_t rows, int dpad, int boxRows, int boxK = 0) {
    CUtensorMap m;
    cuuint64_t dims[3] = {(cuuint64_t)kKBlock, (cuuint64_t)rows, (cuuint64_t)(dpad / kKBlock)};
    cuuint64_t strides[2] = {(cuuint64_t)dpad * 2, (cuuint64_t)kKBlock * 2};
    cuuint32_t box[3] = {(cuuint32_t)kKBlock, (cuuint32_t)boxRows, (cuuint32_t)(boxK > 0 ? boxK : dpad / kKBlock)};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = getEncodeTiled()(
            &m,
            CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
            3,
            const_cast<__half*>(base),
            dims,
            strides,
            box,
            estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B,
            CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    FB_THROW_IF_NOT_FMT(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with %d", (int)r);
    return m;
}

unsigned long long gcd64(unsigned long long a, unsigned long long b) {
    while (b) {
        unsigned long long t = a % b;
        a = b;
        b = t;
    }
    return a;
}

struct SmemPlan {
    int yStages;
    size_t bytes;
    int ksplit; // ring stages hold single K-blocks (see flat_tc_kernel)
};

constexpr int kMaxKB = 4; // d <= 256: the query tile (16 KB per K-block) + at least three 32 KB K-block stages in 227 KB

// d <= 128: whole-tile stages (64 KB at d = 128: three of them); beyond, K-block stages (see flat_tc_kernel)
SmemPlan planSmem(int KB) {
    FB_THROW_IF_NOT_MSG(KB <= kMaxKB, "dimension too large for the tensor-core Flat kernel");
    const int ksplit = KB > 2 ? 1 : 0;
    const size_t qtile = (size_t)KB * kTileM * kKBlock * 2;
    const size_t fixed = 1024 /*align slack*/ + 512 /*barriers*/ + qtile;
    const size_t stage = (size_t)(ksplit ? 1 : KB) * kTileN * kKBlock * 2;
    const size_t budget = 226 * 1024; // 232448 B is the opt-in limit per CTA
    int ys = (int)std::min<size_t>(kMaxYStages, (budget - fixed) / stage);
    FB_THROW_IF_NOT(ys >= 3);
    return {ys, fixed + ys * stage, ksplit};
}

template <bool DUMP>
void launchTc(const CUtensorMap& mq, const CUtensorMap& my, const TcParams& p, int grid, size_t smem, cudaStream_t stream, bool self = false) {
    auto kern = flat_tc_kernel<DUMP>;
    if (self && !DUMP) // k = 1 streaming mode (self-tightening thresholds)
        kern = flat_tc_kernel<false, true>;
    CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTiming::begin("flat_tc", stream);
    kern<<<grid, kTcThreads, smem, stream>>>(mq, my, p);
    KernelTiming::end("flat_tc", stream);
    CUDA_CHECK_LAST();
}

} // namespace

// ------------------------------------------------------------------------------------------
// public launchers
// ------------------------------------------------------------------------------------------
void runAbsMax(const void* x, int64_t count, float* out, cudaStream_t stream, int yHalf) {
    if (count == 0)
        return;
    int blocks = (int)std::min<int64_t>(1184, ceil_div(count, 256));
    absmax_kernel<<<blocks, 256, 0, stream>>>(x, yHalf, count, out);
    CUDA_CHECK_LAST();
}

void runMaxOf(const float* x, int64_t count, float* out, cudaStream_t stream) {
    runAbsMax(x, count, out, stream, 0);
}

void runFlatTcPrepareRows(
        GpuResources* res,
        int device,
        const void* Y,
        int64_t n,
        int d,
        int dpad,
        float scale,
        MetricType metric,
        __half* Y16,
        float* bias,
        int* perm,
        float* tileMaxBias,
        float* norms,
        cudaStream_t stream,
        int yHalf) {
    if (n == 0)
        return;
    const int warps = 8;
    const unsigned rowBlocks = (unsigned)ceil_div(n, warps);
    const int isL2 = metric == METRIC_L2 ? 1 : 0;
    // squared norms in row order (also feeds the caller's max-norm reduction)
    tc_prepare_rows_kernel<<<rowBlocks, warps * 32, 0, stream>>>(Y, yHalf, n, d, dpad, scale, isL2, nullptr, nullptr, nullptr, norms);
    CUDA_CHECK_LAST();
    if (perm) {
        // stored order = rows sorted by squared norm: the biases of a 256-row tile are then nearly
        // equal, which is what makes the kernel's per-tile score bound tight (flat_tc_kernel.cuh)
        auto keysOut = res->temp(device, sizeof(float) * n);
        auto valsIn = res->temp(device, sizeof(int) * n);
        tc_iota_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(valsIn.as<int>(), n);
        CUDA_CHECK_LAST();
        size_t tmpBytes = 0;
        CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(
                nullptr, tmpBytes, norms, keysOut.as<float>(), valsIn.as<int>(), perm, (int)n, 0, 32, stream));
        auto tmp = res->temp(device, tmpBytes);
        CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(
                tmp.data, tmpBytes, norms, keysOut.as<float>(), valsIn.as<int>(), perm, (int)n, 0, 32, stream));
    }
    tc_prepare_rows_kernel<<<rowBlocks, warps * 32, 0, stream>>>(Y, yHalf, n, d, dpad, scale, isL2, perm, Y16, bias, nullptr);
    CUDA_CHECK_LAST();
    const int64_t numTiles = ceil_div(n, kTileN);
    tc_tile_max_bias_kernel<<<(unsigned)ceil_div(numTiles, warps), warps * 32, 0, stream>>>(bias, numTiles, tileMaxBias);
    CUDA_CHECK_LAST();
}

bool flatTcSupported(int d, int k, int64_t n) {
    int dpad = (int)round_up(d, kKBlock);
    // k = 1 takes the streaming mode, which pays off from a few tiles on (coarse assignment against nlist >= 2048
    // centroids during add / k-means); the round-based path needs a database worth several rounds
    return dpad <= kMaxKB * kKBlock && k >= 1 && k <= 2048 && n >= (k == 1 ? 2048 : 32768) && n < (int64_t(1) << 31) - 512;
}

void runFlatTcScoresDebug(
        const __half* Q16,
        int64_t nq,
        const __half* Y16,
        int64_t n,
        int dpad,
        float* S,
        cudaStream_t stream) {
    FB_THROW_IF_NOT(dpad % kKBlock == 0 && dpad <= kMaxKB * kKBlock);
    const int KB = dpad / kKBlock;
    SmemPlan sp = planSmem(KB);
    CUtensorMap my = makeTileMap(Y16, n, dpad, kTileN, sp.ksplit);
    const int64_t numTiles = ceil_div(n, kTileN);
    const int64_t qPairs = ceil_div(nq, kUnitM);
    // the kernel reads whole 128-row query tiles: zero-padded private copy
    __half* qpad = nullptr;
    CUDA_VERIFY(cudaMallocAsync(&qpad, sizeof(__half) * qPairs * kUnitM * dpad, stream));
    CUDA_VERIFY(cudaMemsetAsync(qpad, 0, sizeof(__half) * qPairs * kUnitM * dpad, stream));
    CUDA_VERIFY(cudaMemcpyAsync(qpad, Q16, sizeof(__half) * nq * dpad, cudaMemcpyDeviceToDevice, stream));
    // scale (1.0) for the debug run; the dump path never reads biases
    float* one = nullptr;
    CUDA_VERIFY(cudaMallocAsync(&one, sizeof(float), stream));
    float h1 = 1.f;
    CUDA_VERIFY(cudaMemcpyAsync(one, &h1, sizeof(float), cudaMemcpyHostToDevice, stream));
    TcParams p{};
    p.slices = 1;
    p.qPairs = (int)qPairs;
    p.numUnits = (int)qPairs;
    CUtensorMap mq = makeTileMap(qpad, qPairs * kUnitM, dpad, kTileM);
    p.tileBegin = 0;
    p.tileEnd = (int)numTiles;
    p.tilesPerSlice = (int)numTiles;
    p.permA = 1;
    p.permB = 0;
    p.numTiles = (unsigned long long)numTiles;
    p.KB = KB;
    p.ksplit = sp.ksplit;
    p.kSteps = dpad / 16; // debug seam: operands arrive padded
    p.yStages = sp.yStages;
    p.invScalePtr = one;
    p.bias = nullptr;
    p.tileMaxBias = nullptr;
    p.thr = nullptr;
    p.cand = nullptr;
    p.cap = 0;
    p.candCount = nullptr;
    p.dump = S;
    p.dumpLd = numTiles * kTileN; // S must be [nq][numTiles*128]
    p.nq = (int)nq;
    int dev = 0, sms = 0;
    CUDA_VERIFY(cudaGetDevice(&dev));
    CUDA_VERIFY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    launchTc<true>(mq, my, p, (int)std::min<int64_t>(p.numUnits, sms), sp.bytes, stream);
    CUDA_VERIFY(cudaFreeAsync(qpad, stream));
    CUDA_VERIFY(cudaFreeAsync(one, stream));
}

void runFlatTcSearch(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nqAll,
        const void* Y,
        const __half* Y16,
        const float* bias,
        const int* perm,
        const float* tileMaxBias,
        float yScale,
        float yMaxNorm,
        int64_t n,
        int d,
        int dpad,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream,
        const FlatTcShard* shard,
        int yHalf) {
    if (nqAll == 0)
        return;
    FB_THROW_IF_NOT(flatTcSupported(d, k, n));
    const int KB = dpad / kKBlock;
    const SmemPlan sp = planSmem(KB);
    const int sms = res->numSMs(device);
    const int64_t T = ceil_div(n, kTileN);
    // Sharded search: every rank runs the SAME number of rounds (one all-reduce per round), so the schedule
    // is laid out over the largest shard's tile count and clamped to this shard's.  Thresholds are pooled
    // across ranks after every round, i.e. a round over t local tiles is worth S*t tiles of evidence: the first
    // round shrinks by S and the rounds grow faster (fewer launches for a 1/S-size shard).
    const int nShards = shard ? shard->comm->size() : 1;
    const int64_t Tsched = shard ? std::max<int64_t>(T, shard->maxTiles) : T;
    const int kFrac = (k + nShards - 1) / nShards;
    const int LIST = std::max(128, next_pow2(2 * k));
    const int KL = std::max(64, next_pow2(k));

    // tile permutation: multiplicative hash with a multiplier coprime to T
    unsigned long long A = (unsigned long long)((double)T * 0.6180339887498949);
    if (A < 1)
        A = 1;
    while (gcd64(A, (unsigned long long)T) != 1)
        A++;
    const unsigned long long B = (unsigned long long)(T / 3);

    // error model constants (DESIGN.md): fp16 rounding of both operands + fp32 accumulation slack
    const float c1 = 1.01f * (ldexpf(1.f, -10) + (float)dpad * ldexpf(1.f, -22));
    const float c2 = (float)(dpad + 16) * ldexpf(1.f, -24);

    CUtensorMap mapY = makeTileMap(Y16, n, dpad, kTileN, sp.ksplit);

    // first round: ~40 k rows (16 tiles at k = 100).  Every score of round 0 becomes a candidate, so a
    // fixed 16 tiles would make small-k searches (k-means assignment: k = 1, millions of queries) pay 4096
    // candidates per query for nothing.
    int r0Tiles = std::max(std::max(1, (40 * k + kTileN - 1) / kTileN), (k + 127) / 128 * 2);
    if (nShards > 1) // pooled evidence: nShards * r0Tiles tiles; a shard must still be able to vouch for kFrac rows
        r0Tiles = std::max<int>((r0Tiles + nShards - 1) / nShards, std::max(2, (2 * kFrac + kTileN - 1) / kTileN));
    // threshold selection by bisection (no sorted lists) holds kSelCap entries per query and round: the all-pass first
    // round is sized to 3/4 of that
    const bool useBisect = LIST <= 256;
    if (useBisect)
        r0Tiles = std::min(r0Tiles, std::max(2, kSelCap * 3 / 4 / kTileN));
    // queries per pass: bounds the candidate arena, whose largest user is the all-pass round 0
    // (2 KB per query and tile) -- 16384 queries at k = 100, up to 131072 for small k
    // k = 1 (k-means assignment, the coarse quantiser of an add): streaming mode -- one pass over all tiles with
    // self-tightening per-thread thresholds (flat_tc_kernel SELF) and a fused select + exact re-rank
    // (tc_argmin_finish_kernel); no rounds, no all-pass first round, no per-query sorted lists.
    const bool streaming = k == 1 && !shard;
    // streaming: a batch is a whole number of waves of the persistent grid (one 128-query unit per CTA and wave)
    // (large k: the all-pass round covers 40 k rows, so the floor drops to keep the arena near 1 GiB)
    const int64_t kQFloor = r0Tiles > 64 ? 2048 : 16384;
    const int64_t kQBatch = streaming ? (int64_t)sms * kUnitM * 4
                                      : std::min<int64_t>(131072, std::max<int64_t>(kQFloor, (int64_t)262144 / r0Tiles));
    for (int64_t qb = 0; qb < nqAll; qb += kQBatch) {
        const int64_t nq = std::min(kQBatch, nqAll - qb);
        const float* Qb = Q + qb * d;
        const int64_t qPairs = ceil_div(nq, kUnitM);

        auto q16 = res->temp(device, sizeof(__half) * qPairs * kUnitM * dpad);
        auto scal = res->temp(device, sizeof(float) * 4); // [absmax, qScale, inv, -]
        auto eps = res->temp(device, sizeof(float) * nq);
        auto thr = res->temp(device, sizeof(float) * nq);
        auto flags = res->temp(device, sizeof(int) * (nq + 1));
        auto baseKey = res->temp(device, streaming ? sizeof(float) : sizeof(float) * nq * LIST);
        auto baseId = res->temp(device, streaming ? sizeof(int) : sizeof(int) * nq * LIST);

        CUDA_VERIFY(cudaMemsetAsync(scal.data, 0, sizeof(float) * 4, stream));
        CUDA_VERIFY(cudaMemsetAsync(flags.data, 0, sizeof(int) * (nq + 1), stream));
        CUDA_VERIFY(cudaMemsetAsync(q16.data, 0, sizeof(__half) * qPairs * kUnitM * dpad, stream));
        float* sc = scal.as<float>();
        runAbsMax(Qb, nq * d, sc + 0, stream);
        tc_query_scale_kernel<<<1, 1, 0, stream>>>(sc + 0, yScale, sc + 1, sc + 2);
        CUDA_CHECK_LAST();
        tc_prepare_queries_kernel<<<(unsigned)ceil_div(nq, 8), 256, 0, stream>>>(
                Qb, nq, d, dpad, sc + 1, c1, c2, yMaxNorm, q16.as<__half>(), eps.as<float>(), thr.as<float>());
        CUDA_CHECK_LAST();
        if (!streaming) {
            int64_t cnt = nq * LIST;
            tc_init_base_kernel<<<(unsigned)ceil_div(cnt, 256), 256, 0, stream>>>(
                    baseKey.as<float>(), baseId.as<int>(), cnt);
            CUDA_CHECK_LAST();
        }

        // ---- geometric rounds over the permuted tile order
        struct Round {
            int begin, end, slices, tilesPerSlice, cap;
        };
        const int parts = kParts;
        std::vector<Round> rounds;
        {
            const double g = nShards > 1 ? std::max(4.0, std::min(8.0, 2.0 * nShards)) : 4.0; // growth per round
            int64_t seen = 0;
            while (seen < Tsched) {
                int64_t end = seen == 0 ? std::min<int64_t>(Tsched, r0Tiles)
                                        : std::min<int64_t>(Tsched, (int64_t)(seen * g));
                if (Tsched - end < end / 4)
                    end = Tsched; // do not leave a sliver for an extra round
                if (streaming)
                    end = Tsched; // k = 1: ONE pass, thresholds tighten themselves inside the kernel
                int64_t tiles = end - seen;
                // choose the slice count minimising (waves x tiles per slice)
                int bestS = 1;
                double bestCost = 1e300;
                int64_t maxS = std::max<int64_t>(1, std::min<int64_t>(512, tiles / 8));
                for (int64_t S = 1; S <= maxS; S++) {
                    int64_t tps = ceil_div(tiles, S);
                    int64_t units = qPairs * ceil_div(tiles, tps);
                    int64_t waves = ceil_div(units, sms);
                    double cost = (double)waves * (double)(tps + 6); // +6: per-unit fixed overhead
                    if (cost < bestCost * 0.999) {
                        bestCost = cost;
                        bestS = (int)S;
                    }
                }
                int64_t tps = ceil_div(tiles, bestS);
                int S = (int)ceil_div(tiles, tps);
                int cap;
                if (streaming) {
                    // a thread emits ~ln(columns it sees) running maxima plus the near-ties of the maximum
                    cap = 64;
                } else if (seen == 0) {
                    cap = (int)(tps * (kTileN / parts)); // everything passes in round 0
                } else {
                    double expect = 1.5 * k * ((double)tps / (double)seen) / parts;
                    cap = next_pow2((int)std::min<double>(1 << 20, 4.0 * expect + 32.0));
                    cap = std::max(cap, 32);
                }
                rounds.push_back({(int)seen, (int)end, S, (int)tps, cap});
                seen = end;
            }
        }
        size_t arenaBytes = 0, countBytes = 0;
        for (auto& r : rounds) {
            size_t units = (size_t)qPairs * r.slices;
            arenaBytes = std::max(arenaBytes, units * kSegsPerUnit * (size_t)r.cap * sizeof(uint2));
            countBytes = std::max(countBytes, units * kSegsPerUnit * sizeof(int));
        }
        auto arena = res->temp(device, arenaBytes);
        auto counts = res->temp(device, countBytes);

        const int selWarps = (int)std::max<size_t>(1, std::min<size_t>(8, (48 * 1024) / SmemTopK<int>::bytes(LIST, kSelectBuf)));
        const size_t selSmem = SmemTopK<int>::bytes(LIST, kSelectBuf) * selWarps;
        CUDA_VERIFY(cudaFuncSetAttribute(tc_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)selSmem));

        GpuMemoryReservation contrib;
        if (shard)
            contrib = res->temp(device, sizeof(float) * 2 * nq);
        for (auto& r : rounds) {
            TcParams p{};
            p.slices = r.slices;
            p.qPairs = (int)qPairs;
            p.numUnits = (int)(qPairs * r.slices);
            CUtensorMap mapQ = makeTileMap(q16.as<__half>(), qPairs * kUnitM, dpad, kTileM);
            p.tileBegin = (int)std::min<int64_t>(r.begin, T); // schedule laid out over the largest shard: clamp to ours
            p.tileEnd = (int)std::min<int64_t>(r.end, T);
            p.tilesPerSlice = r.tilesPerSlice;
            p.permA = A;
            p.permB = B;
            p.numTiles = (unsigned long long)T;
            p.KB = KB;
            p.ksplit = sp.ksplit;
            p.kSteps = (d + 15) / 16;
            p.yStages = sp.yStages;
            p.invScalePtr = sc + 2;
            p.bias = bias;
            p.tileMaxBias = tileMaxBias;
            p.tileMinBias = tileMaxBias + T + 1; // second half of the array (see tc_tile_max_bias_kernel)
            p.thr = thr.as<float>();
            p.eps = eps.as<float>();
            p.cand = arena.as<uint2>();
            p.cap = r.cap;
            p.candCount = counts.as<int>();
            p.dump = nullptr;
            p.dumpLd = 0;
            p.nq = (int)nq;
            if (p.tileBegin < p.tileEnd) {
                launchTc<false>(mapQ, mapY, p, std::min(p.numUnits, sms), sp.bytes, stream, streaming);
            } else { // this shard has no tiles in this round of the common schedule: no candidates
                CUDA_VERIFY(cudaMemsetAsync(counts.data, 0, (size_t)p.numUnits * kSegsPerUnit * sizeof(int), stream));
            }
            if (streaming) { // select + exact re-rank fused: one warp per query
                const int fw = 8;
                float* oD1 = outD + qb;
                idx_t* oI1 = outI + qb;
                KernelTiming::begin("tc_argmin_finish", stream);
                auto launchFin = [&](auto kern) {
                    kern<<<(unsigned)ceil_div(nq, fw), fw * 32, 0, stream>>>(
                            (int)nq, d, r.slices, parts, arena.as<uint2>(), r.cap, counts.as<int>(), eps.as<float>(), Qb, Y, perm,
                            oD1, oI1, flags.as<int>());
                };
                if (metric == METRIC_L2)
                    yHalf ? launchFin(tc_argmin_finish_kernel<true, true>) : launchFin(tc_argmin_finish_kernel<true, false>);
                else
                    yHalf ? launchFin(tc_argmin_finish_kernel<false, true>) : launchFin(tc_argmin_finish_kernel<false, false>);
                KernelTiming::end("tc_argmin_finish", stream);
                CUDA_CHECK_LAST();
                continue;
            }
            KernelTiming::begin("tc_select", stream);
            if (useBisect) {
                const size_t bsmem = sizeof(uint2) * kSelCap * kSelWarps;
                CUDA_VERIFY(cudaFuncSetAttribute(tc_select_bisect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsmem));
                tc_select_bisect_kernel<<<(unsigned)ceil_div(nq, kSelWarps), kSelWarps * 32, bsmem, stream>>>(
                        (int)nq, k, LIST, r.slices, parts, arena.as<uint2>(), r.cap, counts.as<int>(), eps.as<float>(),
                        baseKey.as<float>(), baseId.as<int>(), thr.as<float>(), flags.as<int>(),
                        shard ? contrib.as<float>() : nullptr, kFrac);
            } else {
                tc_select_kernel<<<(unsigned)ceil_div(nq, selWarps), selWarps * 32, selSmem, stream>>>(
                        (int)nq,
                        k,
                        LIST,
                        r.slices,
                        parts,
                        arena.as<uint2>(),
                        r.cap,
                        counts.as<int>(),
                        eps.as<float>(),
                        baseKey.as<float>(),
                        baseId.as<int>(),
                        thr.as<float>(),
                        flags.as<int>(),
                        shard ? contrib.as<float>() : nullptr,
                        kFrac);
            }
            KernelTiming::end("tc_select", stream);
            CUDA_CHECK_LAST();
            if (shard) {
                KernelTiming::begin("tc_pool", stream);
                // ONE small all-reduce per round (2 floats per query): every shard then filters against a
                // threshold certified by the pooled evidence of all shards
                shard->comm->allReduceMax(contrib.as<float>(), (size_t)2 * nq, stream);
                tc_pooled_thr_kernel<<<(unsigned)ceil_div(nq, 256), 256, 0, stream>>>(
                        (int)nq, contrib.as<float>(), eps.as<float>(), thr.as<float>());
                KernelTiming::end("tc_pool", stream);
                CUDA_CHECK_LAST();
            }
        }

        // ---- exact re-rank
        if (!streaming) {
            const int rrWarps = (int)std::max<size_t>(1, std::min<size_t>(8, (48 * 1024) / SmemTopK<int>::bytes(KL, 64)));
            const size_t rrSmem = SmemTopK<int>::bytes(KL, 64) * rrWarps;
            float* oD = outD + qb * k;
            idx_t* oI = outI + qb * k;
            auto launchRr = [&](auto kern) {
                CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rrSmem));
                kern<<<(unsigned)ceil_div(nq, rrWarps), rrWarps * 32, rrSmem, stream>>>(
                        (int)nq, d, k, LIST, KL, Qb, Y, perm, baseId.as<int>(), baseKey.as<float>(),
                        shard ? thr.as<float>() : nullptr, oD, oI);
            };
            KernelTiming::begin("tc_rerank", stream);
            if (metric == METRIC_L2)
                yHalf ? launchRr(tc_rerank_kernel<true, true>) : launchRr(tc_rerank_kernel<true, false>);
            else
                yHalf ? launchRr(tc_rerank_kernel<false, true>) : launchRr(tc_rerank_kernel<false, false>);
            KernelTiming::end("tc_rerank", stream);
            CUDA_CHECK_LAST();
        }

        // ---- certificate failures -> exact SIMT recompute
        {
            auto list = res->temp(device, sizeof(int) * nq);
            int* countDev = flags.as<int>() + nq;
            tc_collect_flags_kernel<<<(unsigned)ceil_div(nq, 256), 256, 0, stream>>>(
                    flags.as<int>(), (int)nq, list.as<int>(), countDev);
            CUDA_CHECK_LAST();
            int nflag = 0;
            CUDA_VERIFY(cudaMemcpyAsync(&nflag, countDev, sizeof(int), cudaMemcpyDeviceToHost, stream));
            CUDA_VERIFY(cudaStreamSynchronize(stream));
            if (nflag > 0) {
                auto fq = res->temp(device, sizeof(float) * (size_t)nflag * d);
                auto fD = res->temp(device, sizeof(float) * (size_t)nflag * k);
                auto fI = res->temp(device, sizeof(idx_t) * (size_t)nflag * k);
                tc_gather_queries_kernel<<<nflag, 128, 0, stream>>>(Qb, list.as<int>(), d, fq.as<float>());
                CUDA_CHECK_LAST();
                runFlatExact(res, device, fq.as<float>(), nflag, Y, n, d, k, metric, 0, fD.as<float>(), fI.as<idx_t>(), stream, yHalf);
                tc_scatter_results_kernel<<<nflag, 128, 0, stream>>>(
                        fD.as<float>(), fI.as<idx_t>(), list.as<int>(), k, outD + qb * k, outI + qb * k);
                CUDA_CHECK_LAST();
                CUDA_VERIFY(cudaStreamSynchronize(stream));
            }
            lastFlatTcFallbacks() = nflag;
        }
    }
}

int& lastFlatTcFallbacks() {
    static thread_local int v = 0;
    return v;
}

} // namespace fb200
