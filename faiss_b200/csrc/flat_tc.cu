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
//     two consumer warpgroups that each run 64x256xK wgmma tiles into register accumulators (at
//     112 < d <= 128: four that each run 64x128xK, one per query half and column half) and filter
//     them in place: each thread holds two query rows and 64 (or 32) of a tile's 256 columns of each, folds the
//     RAW accumulators with a max tree and compares one bound per 32 of them against the query's
//     threshold held in a register -- the fp16 copy
//     is stored sorted by norm, so the tile's maximum bias bounds every row's bias tightly.  Scores
//     never reach HBM; only the rare survivors are appended to a per-(query, column part) candidate segment.
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
#include "flat_tc.h"
#include "kernels.h"
#include "select.cuh"
#include "tc_ptx.cuh"
#include "flat_tc_kernel.cuh"

namespace fb200 {
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

__global__ void fill_float_kernel(float* out, int64_t n, float v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        out[i] = v;
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

// bias copy with -inf at rows whose mask bit is clear: out[p] = mask[perm[p]] ? bias[p] : -inf for p < n (perm null:
// identity), -inf for n <= p < padRows
__global__ void mask_bias_kernel(
        const float* __restrict__ bias, const int* __restrict__ perm, const uint32_t* __restrict__ mask, int64_t n,
        int64_t padRows, float* __restrict__ out) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= padRows)
        return;
    float b = -CUDART_INF_F;
    if (p < n) {
        const int64_t r = perm ? perm[p] : p;
        if ((mask[r >> 5] >> (r & 31)) & 1u)
            b = bias[p];
    }
    out[p] = b;
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
        float yScale,
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
        // |approx score - score implied by the exact kernel's fp32 distance| <= eps (DESIGN.md 3.1, error model):
        //   c1*|q||y|          fp16 input rounding + fp32 accumulation of q.y
        //   c2*(|q|+|y|)^2     fp32 rounding of the bias (norms), of the final FMA and of the exact kernel's own sum
        //   1.01*(uq*|y| + uy*|q| + uq*uy)   elements in fp16's subnormal range, off by up to 2^-25 / s absolute
        //                      rather than 2^-11 relative.  s is the whole batch's scale (yScale the database's), so
        //                      next to a much larger query this bounds the extra error norm: u = sqrt(dpad) 2^-25 / s
        const float u0 = sqrtf((float)dpad) * ldexpf(1.f, -25);
        const float uq = u0 / scale, uy = u0 / yScale;
        const float qy = qn + yMaxNorm;
        eps[row] = c1 * qn * yMaxNorm + c2 * qy * qy + 1.01f * (uq * yMaxNorm + uy * qn + uq * uy);
        thr[row] = -CUDART_INF_F;
    }
}

// ---- int8 layout (DESIGN.md 3.1, "int8 scoring").  Centring, quantisation and the certificate's database constants.
constexpr int kDpad8 = 128; // s8 per stored row: one 128-byte swizzle row

// per-dimension min / max of the rows (order-preserving keys; NaN and inf are ignored); one thread per dimension
__global__ void tc_col_range_kernel(const void* __restrict__ Y, int yHalf, int64_t n, int d, unsigned* __restrict__ range) {
    const int j = threadIdx.x;
    if (j >= d)
        return;
    unsigned lo = 0xffffffffu, hi = 0u;
    for (int64_t r = blockIdx.x; r < n; r += gridDim.x) {
        const float v = yHalf ? row_load1<true>(Y, r * d + j) : reinterpret_cast<const float*>(Y)[r * d + j];
        if (v == v && fabsf(v) <= FLT_MAX) {
            lo = min(lo, float_to_ordered(v));
            hi = max(hi, float_to_ordered(v));
        }
    }
    atomicMin(range + j, lo);
    atomicMax(range + d + j, hi);
}

// centre c = per-dimension midrange (0 for a dimension without a finite value), and the database scale
// s_y = 127 / max |fl(y - c)| (fl is monotone: the extremes of y give the extremes of fl(y - c)); one block of kDpad8
__global__ void tc_center_kernel(const unsigned* __restrict__ range, int d, float* __restrict__ center, float* __restrict__ scale) {
    __shared__ float red[kDpad8 / 32];
    const int j = threadIdx.x;
    float a = 0.f;
    if (j < d) {
        const unsigned lo = range[j], hi = range[d + j];
        float c = 0.f;
        if (lo <= hi) {
            const float mn = ordered_to_float(lo), mx = ordered_to_float(hi);
            c = 0.5f * mn + 0.5f * mx;
            a = fmaxf(mx - c, c - mn);
        }
        center[j] = c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        a = fmaxf(a, __shfl_xor_sync(kFullMask, a, o));
    if (lane_id() == 0)
        red[j >> 5] = a;
    __syncthreads();
    if (j == 0) {
        float m = 0.f;
        for (int w = 0; w < kDpad8 / 32; w++)
            m = fmaxf(m, red[w]);
        *scale = m > 0.f ? 127.f / m : 1.f;
    }
}

// one warp per row, lane l holds dimensions 4l .. 4l + 3 of fl(y - c).  Without Y8: the squared centred norm (the sort
// key) and the plain norm |y| (for the fitness test).  With Y8: the row at stored position `row` (source perm[row])
// quantised to Y8 = rn(fl(y - c) * s_y) in [-127, 127], zero padded to 128, its bias -|y - c|^2 / 2 and, into
// stats[0..2] (max of non-negative floats as ints), |Y8 / s_y|^2, |fl(y - c) - Y8 / s_y|^2 and |y - c|^2.
__global__ void tc_prepare_rows8_kernel(
        const void* __restrict__ Y,
        int yHalf,
        int64_t n,
        int d,
        const float* __restrict__ center,
        const float* __restrict__ scale,
        const int* __restrict__ perm,
        int8_t* __restrict__ Y8,
        float* __restrict__ bias,
        float* __restrict__ keys,
        float* __restrict__ norms,
        float* __restrict__ stats) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n)
        return;
    const int64_t src = (perm ? (int64_t)perm[row] : row) * d;
    const float sy = *scale;
    float yc2 = 0.f, y2 = 0.f, r2 = 0.f;
    int h2 = 0;
    uint32_t packed = 0;
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int i = 4 * lane_id() + u;
        float y = 0.f, v = 0.f;
        if (i < d) {
            y = yHalf ? row_load1<true>(Y, src + i) : reinterpret_cast<const float*>(Y)[src + i];
            v = y - center[i];
        }
        yc2 = fmaf(v, v, yc2);
        y2 = fmaf(y, y, y2);
        const int c = (int)fminf(127.f, fmaxf(-127.f, rintf(v * sy)));
        h2 += c * c;
        const float r = v - (float)c / sy;
        r2 = fmaf(r, r, r2);
        packed |= (uint32_t)(uint8_t)(int8_t)c << (8 * u);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        yc2 += __shfl_xor_sync(kFullMask, yc2, o);
        y2 += __shfl_xor_sync(kFullMask, y2, o);
        r2 += __shfl_xor_sync(kFullMask, r2, o);
        h2 += __shfl_xor_sync(kFullMask, h2, o);
    }
    if (!Y8) {
        if (lane_id() == 0) {
            keys[row] = yc2;
            norms[row] = sqrtf(y2);
        }
        return;
    }
    reinterpret_cast<uint32_t*>(Y8 + row * kDpad8)[lane_id()] = packed;
    if (lane_id() == 0) {
        bias[row] = -0.5f * yc2;
        const float hn = (float)h2 / (sy * sy);
        atomicMax(reinterpret_cast<int*>(stats + 0), __float_as_int(hn));
        atomicMax(reinterpret_cast<int*>(stats + 1), __float_as_int(r2));
        atomicMax(reinterpret_cast<int*>(stats + 2), __float_as_int(yc2));
    }
}

// int8 query preparation, one warp per query (lane l: dimensions 4l .. 4l + 3): q_c = fl(q - c), its own scale
// s_q = 127 / max|q_c|, Q8 = rn(q_c * s_q), inv = fl(1 / (s_q * s_y)) and the certificate (DESIGN.md 3.1)
//   eps = |q^|*maxR + |r_q|*maxY^ + |r_q|*maxR   (quantisation; q^ = Q8 / s_q, r_q = q_c - q^)
//       + 2^-20 * |q^| * maxY^                     (inv and the FMA's rounding of acc * inv, residuals computed in fp32)
//       + c2 * (|q_c| + maxYc)^2                    (bias, centring, the FMA's rounding of the bias, the exact kernel)
__global__ void tc_prepare_queries8_kernel(
        const float* __restrict__ Q,
        int64_t nq,
        int d,
        const float* __restrict__ center,
        const float* __restrict__ yScale,
        float maxYhat,
        float maxRy,
        float maxYc,
        float c2,
        int8_t* __restrict__ Q8,
        float* __restrict__ invQ,
        float* __restrict__ eps,
        float* __restrict__ thr) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= nq)
        return;
    float v[4];
    float a = 0.f;
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int i = 4 * lane_id() + u;
        v[u] = i < d ? Q[row * d + i] - center[i] : 0.f;
        a = fmaxf(a, fabsf(v[u]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        a = fmaxf(a, __shfl_xor_sync(kFullMask, a, o));
    const float sq = a > 0.f ? 127.f / a : 1.f;
    float qc2 = 0.f, r2 = 0.f;
    int h2 = 0;
    uint32_t packed = 0;
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int c = (int)fminf(127.f, fmaxf(-127.f, rintf(v[u] * sq)));
        qc2 = fmaf(v[u], v[u], qc2);
        h2 += c * c;
        const float r = v[u] - (float)c / sq;
        r2 = fmaf(r, r, r2);
        packed |= (uint32_t)(uint8_t)(int8_t)c << (8 * u);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        qc2 += __shfl_xor_sync(kFullMask, qc2, o);
        r2 += __shfl_xor_sync(kFullMask, r2, o);
        h2 += __shfl_xor_sync(kFullMask, h2, o);
    }
    reinterpret_cast<uint32_t*>(Q8 + row * kDpad8)[lane_id()] = packed;
    if (lane_id() == 0) {
        const float qh = sqrtf((float)h2) / sq * 1.0001f;
        const float rq = sqrtf(r2) * 1.0001f;
        const float qc = sqrtf(qc2) * 1.0001f;
        const float s = qc + maxYc;
        eps[row] = (qh * maxRy + rq * maxYhat + rq * maxRy) * 1.0001f + ldexpf(1.f, -20) * qh * maxYhat + c2 * s * s;
        invQ[row] = 1.f / (sq * *yScale);
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
        constexpr int kMaxListIter = 16; // LIST <= 512 (int8 scoring: 4k entries at k <= 128)
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

// int8 matrix [rows][128] viewed as (128, rows, 1); one box = 128 bytes x boxRows rows, 128-byte swizzle
CUtensorMap makeTileMap8(const int8_t* base, int64_t rows, int boxRows) {
    CUtensorMap m;
    cuuint64_t dims[3] = {(cuuint64_t)kDpad8, (cuuint64_t)rows, 1};
    cuuint64_t strides[2] = {(cuuint64_t)kDpad8, (cuuint64_t)rows * kDpad8};
    cuuint32_t box[3] = {(cuuint32_t)kDpad8, (cuuint32_t)boxRows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = getEncodeTiled()(
            &m,
            CU_TENSOR_MAP_DATA_TYPE_UINT8,
            3,
            const_cast<int8_t*>(base),
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

struct SmemPlan {
    int yStages;
    size_t bytes;
    int ksplit; // ring stages hold single K-blocks (see flat_tc_kernel)
    bool quad;  // four consumer warpgroups over half-tile ring stages (flat_tc_kernel QUAD)
    int boxRows; // database rows per TMA copy of mapY
    bool s8;    // int8 operands (flat_tc_kernel S8)
};

constexpr int kMaxKB = 4; // d <= 256: the query tile (16 KB per K-block) + at least three 32 KB K-block stages in 227 KB

// 112 < d <= 128: half-tile stages (32 KB: six of them, which the QUAD kernel takes as a constant); other d <= 128:
// whole-tile stages (64 KB at d = 128: three of them); beyond, K-block stages (see flat_tc_kernel)
SmemPlan planSmem(int KB, int kSteps, bool s8 = false) {
    FB_THROW_IF_NOT_MSG(KB <= kMaxKB, "dimension too large for the tensor-core Flat kernel");
    if (s8) { // int8, QUAD: 16 KB query tile and half-tile stages, and the bias ring
        const size_t fixed = 1024 + 512 + kQuadCountBytes + (size_t)kTileM * kDpad8 + (size_t)kS8BiasSlots * kS8BiasSlotBytes;
        return {kS8Stages, fixed + (size_t)kS8Stages * kHalfN * kDpad8, 0, true, kHalfN, true};
    }
    const int ksplit = KB > 2 ? 1 : 0;
    const bool quad = tc_quad(KB, kSteps);
    const int boxRows = quad ? kHalfN : kTileN;
    const size_t qtile = (size_t)KB * kTileM * kKBlock * 2;
    const size_t fixed = 1024 /*align slack*/ + 512 /*barriers*/ + (quad ? kQuadCountBytes : 0) + qtile;
    const size_t stage = (size_t)(ksplit ? 1 : KB) * boxRows * kKBlock * 2;
    const size_t budget = 227 * 1024; // the opt-in limit per CTA
    int ys = (int)std::min<size_t>(kMaxYStages, (budget - fixed) / stage);
    FB_THROW_IF_NOT(ys >= 3 && (!quad || ys == kMaxYStages));
    return {ys, fixed + ys * stage, ksplit, quad, boxRows, false};
}

// the kernel's parameters for one round over nq queries (the search's pointers are filled in by the caller)
TcParams roundParams(const SmemPlan& sp, int KB, int kSteps, int64_t nq, int64_t qPairs, const FlatTcRound& r, int64_t T,
                     unsigned long long permA, unsigned long long permB, const float* invScale) {
    TcParams p{};
    p.slices = r.slices;
    p.qPairs = (int)qPairs;
    p.numUnits = (int)(qPairs * r.slices);
    p.tileBegin = (int)std::min<int64_t>(r.begin, T); // schedule laid out over the largest shard: clamp to ours
    p.tileEnd = (int)std::min<int64_t>(r.end, T);
    p.tilesPerSlice = r.tilesPerSlice;
    p.permA = permA;
    p.permB = permB;
    p.numTiles = (unsigned long long)T;
    p.permStep = (int)(permA % (unsigned long long)T);
    p.KB = KB;
    p.ksplit = sp.ksplit;
    p.kSteps = kSteps;
    p.yStages = sp.yStages;
    p.invScalePtr = invScale;
    p.cap = r.cap;
    p.nq = (int)nq;
    return p;
}

template <bool DUMP>
void launchTc(const CUtensorMap& mq, const CUtensorMap& my, const TcParams& p, int grid, const SmemPlan& sp, cudaStream_t stream, bool self = false) {
    const size_t smem = sp.bytes;
    // QUAD: a segment's count is a 16-bit shared-memory counter (flat_tc_kernel.cuh)
    FB_THROW_IF_NOT_FMT(!sp.quad || p.cap <= kQuadMaxCap, "candidate cap %d too large for the 16-bit segment counts", p.cap);
    // the int8 search bulk-copies each half-tile's biases into shared memory, which takes a 16-byte aligned source
    FB_THROW_IF_NOT_MSG(!sp.s8 || DUMP || reinterpret_cast<uintptr_t>(p.bias) % 16 == 0, "int8 search: bias array not 16-byte aligned");
    auto kern = sp.quad ? flat_tc_kernel<DUMP, false, true> : flat_tc_kernel<DUMP>;
    if (self && !DUMP) // k = 1 streaming mode (self-tightening thresholds)
        kern = sp.quad ? flat_tc_kernel<false, true, true> : flat_tc_kernel<false, true>;
    if (sp.s8)
        kern = flat_tc_kernel<DUMP, false, true, true>;
    CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTiming::begin("flat_tc", stream);
    kern<<<grid, tc_threads(sp.quad), smem, stream>>>(mq, my, p);
    KernelTiming::end("flat_tc", stream);
    CUDA_CHECK_LAST();
}

// max |x| over a matrix into a zeroed device scalar (float) -- picks the power-of-two fp16 scale; on non-negative
// values (squared norms), their max
void runAbsMax(const void* x, int64_t count, float* out, cudaStream_t stream, int yHalf = 0) {
    if (count == 0)
        return;
    int blocks = (int)std::min<int64_t>(1184, ceil_div(count, 256));
    absmax_kernel<<<blocks, 256, 0, stream>>>(x, yHalf, count, out);
    CUDA_CHECK_LAST();
}

// per-tile max / min of a stored-order bias array [round_up(n, 256) + 256] (see FlatTcDatabase)
void runTileBias(const float* bias, int64_t n, float* tileBias, cudaStream_t stream) {
    const int warps = 8;
    const int64_t numTiles = ceil_div(n, kTileN);
    tc_tile_max_bias_kernel<<<(unsigned)ceil_div(numTiles, warps), warps * 32, 0, stream>>>(bias, numTiles, tileBias);
    CUDA_CHECK_LAST();
}

} // namespace

bool flatTcSupported(int d, int k, int64_t n) {
    int dpad = (int)round_up(d, kKBlock);
    // k = 1 takes the streaming mode, which pays off from a few tiles on (coarse assignment against nlist >= 2048
    // centroids during add / k-means); the round-based path needs a database worth several rounds
    return dpad <= kMaxKB * kKBlock && k >= 1 && k <= 2048 && n >= (k == 1 ? 2048 : 32768) && n < (int64_t(1) << 31) - 512;
}

FlatTcDatabase::FlatTcDatabase(GpuResources* res, int device, int d)
        : res_(res),
          device_(device),
          d_(d),
          dpad_((int)round_up(d, kKBlock)),
          y16_(res, device, AllocType::FlatData),
          bias_(res, device, AllocType::FlatData),
          perm_(res, device, AllocType::FlatData),
          tileBias_(res, device, AllocType::FlatData),
          y8_(res, device, AllocType::FlatData),
          bias8_(res, device, AllocType::FlatData),
          perm8_(res, device, AllocType::FlatData),
          tileBias8_(res, device, AllocType::FlatData),
          center_(res, device, AllocType::FlatData) {}

void FlatTcDatabase::clear() {
    y16_.clear();
    bias_.clear();
    perm_.clear();
    tileBias_.clear();
    y8_.clear();
    bias8_.clear();
    perm8_.clear();
    tileBias8_.clear();
    center_.clear();
    dirty_ = true;
}

void FlatTcDatabase::prepare(const void* rows, int64_t n, MetricType metric, int yHalf, cudaStream_t) {
    if (!dirty_)
        return;
    rows_ = rows;
    n_ = n;
    metric_ = metric;
    yHalf_ = yHalf;
    fp16Ready_ = false;
    int8Ready_ = false;
    dirty_ = false;
}

void FlatTcDatabase::prepareFp16(cudaStream_t stream) {
    const void* rows = rows_;
    const int64_t n = n_;
    const MetricType metric = metric_;
    const int yHalf = yHalf_;
    const int d = d_, dpad = dpad_;
    const int64_t padRows = round_up(n, 256) + 256; // whole 256-row tiles, -inf beyond n
    y16_.resize((size_t)n * dpad, stream);
    bias_.resize((size_t)padRows, stream);
    tileBias_.resize((size_t)(padRows / 256) * 2, stream); // [T+1] max bias per tile, then [T+1] min bias per tile
    const bool sorted = metric == METRIC_L2; // IP has no bias: row order is kept
    if (sorted)
        perm_.resize((size_t)n, stream);
    else
        perm_.clear();
    auto scal = res_->temp(device_, sizeof(float) * 2);
    auto norms = res_->temp(device_, sizeof(float) * n);
    CUDA_VERIFY(cudaMemsetAsync(scal.data, 0, sizeof(float) * 2, stream));
    runAbsMax(rows, n * (int64_t)d, scal.as<float>(), stream, yHalf);
    float h[2] = {0.f, 0.f};
    CUDA_VERIFY(cudaMemcpyAsync(h, scal.data, sizeof(float), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    float scale = 1.f;
    if (h[0] > 0.f) {
        int e;
        std::frexp(h[0], &e);
        scale = std::ldexp(1.f, 14 - e); // max |y| * scale in [2^13, 2^14)
    }
    fill_float_kernel<<<(unsigned)ceil_div(padRows, 256), 256, 0, stream>>>(bias_.data(), padRows, -INFINITY);
    CUDA_CHECK_LAST();
    const int warps = 8;
    const unsigned rowBlocks = (unsigned)ceil_div(n, warps);
    int* perm = sorted ? perm_.data() : nullptr;
    // squared norms in row order (also feed the max-norm reduction)
    tc_prepare_rows_kernel<<<rowBlocks, warps * 32, 0, stream>>>(
            rows, yHalf, n, d, dpad, scale, sorted, nullptr, nullptr, nullptr, norms.as<float>());
    CUDA_CHECK_LAST();
    if (perm) {
        // stored order = rows sorted by squared norm: the biases of a 256-row tile are then nearly
        // equal, which is what makes the kernel's per-tile score bound tight (flat_tc_kernel.cuh)
        auto keysOut = res_->temp(device_, sizeof(float) * n);
        auto valsIn = res_->temp(device_, sizeof(int) * n);
        tc_iota_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(valsIn.as<int>(), n);
        CUDA_CHECK_LAST();
        size_t tmpBytes = 0;
        CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(
                nullptr, tmpBytes, norms.as<float>(), keysOut.as<float>(), valsIn.as<int>(), perm, (int)n, 0, 32, stream));
        auto tmp = res_->temp(device_, tmpBytes);
        CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(
                tmp.data, tmpBytes, norms.as<float>(), keysOut.as<float>(), valsIn.as<int>(), perm, (int)n, 0, 32, stream));
    }
    tc_prepare_rows_kernel<<<rowBlocks, warps * 32, 0, stream>>>(
            rows, yHalf, n, d, dpad, scale, sorted, perm, y16_.data(), bias_.data(), nullptr);
    CUDA_CHECK_LAST();
    runTileBias(bias_.data(), n, tileBias_.data(), stream);
    runAbsMax(norms.as<float>(), n, scal.as<float>() + 1, stream);
    CUDA_VERIFY(cudaMemcpyAsync(h, scal.data, sizeof(float) * 2, cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    scale_ = scale;
    maxNorm_ = std::sqrt(h[1]) * 1.0001f;
    fp16Ready_ = true;
}

// Fitness of the int8 layout.  The int8 certificate's database term for a query q is about |q|*max|r_y|, the fp16
// one c1*|q|*|y|: the int8 path is taken while max|r_y| <= kInt8Fitness * c1 * (mean |y|).  Uniform data gives about
// 2.2, where the base list of 4k entries holds every entry within 2 eps of the k-th best with room to spare (DESIGN.md
// 3.1); an outlier coordinate that collapses s_y makes max|r_y| as large as the ordinary rows themselves and fails.
constexpr float kInt8Fitness = 4.f;

void FlatTcDatabase::prepareInt8(cudaStream_t stream) {
    const int64_t n = n_;
    const int d = d_;
    const int64_t padRows = round_up(n, 256) + 256;
    y8_.resize((size_t)n * kDpad8, stream);
    bias8_.resize((size_t)padRows, stream);
    tileBias8_.resize((size_t)(padRows / 256) * 2, stream);
    perm8_.resize((size_t)n, stream);
    center_.resize((size_t)d, stream);
    // [0, 2d): column range keys; then s_y, the three stats maxima and the sum of row norms
    auto scratch = res_->temp(device_, sizeof(unsigned) * 2 * d + sizeof(float) * 8);
    unsigned* range = scratch.as<unsigned>();
    float* sc = reinterpret_cast<float*>(range + 2 * d); // [s_y, max|y^|^2, max|r_y|^2, max|y_c|^2, sum |y|]
    CUDA_VERIFY(cudaMemsetAsync(range, 0xff, sizeof(unsigned) * d, stream));
    CUDA_VERIFY(cudaMemsetAsync(range + d, 0, sizeof(unsigned) * d + sizeof(float) * 8, stream));
    tc_col_range_kernel<<<(unsigned)std::min<int64_t>(4096, std::max<int64_t>(1, n)), kDpad8, 0, stream>>>(rows_, yHalf_, n, d, range);
    CUDA_CHECK_LAST();
    tc_center_kernel<<<1, kDpad8, 0, stream>>>(range, d, center_.data(), sc);
    CUDA_CHECK_LAST();
    auto keys = res_->temp(device_, sizeof(float) * n);
    auto norms = res_->temp(device_, sizeof(float) * n);
    const int warps = 8;
    const unsigned rowBlocks = (unsigned)ceil_div(n, warps);
    tc_prepare_rows8_kernel<<<rowBlocks, warps * 32, 0, stream>>>(
            rows_, yHalf_, n, d, center_.data(), sc, nullptr, nullptr, nullptr, keys.as<float>(), norms.as<float>(), nullptr);
    CUDA_CHECK_LAST();
    {
        // stored order = rows sorted by the centred norm, which enters the bias
        auto keysOut = res_->temp(device_, sizeof(float) * n);
        auto valsIn = res_->temp(device_, sizeof(int) * n);
        tc_iota_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(valsIn.as<int>(), n);
        CUDA_CHECK_LAST();
        size_t sortBytes = 0, sumBytes = 0;
        CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(
                nullptr, sortBytes, keys.as<float>(), keysOut.as<float>(), valsIn.as<int>(), perm8_.data(), (int)n, 0, 32, stream));
        CUDA_VERIFY(cub::DeviceReduce::Sum(nullptr, sumBytes, norms.as<float>(), sc + 4, (int)n, stream));
        auto tmp = res_->temp(device_, std::max(sortBytes, sumBytes));
        CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(
                tmp.data, sortBytes, keys.as<float>(), keysOut.as<float>(), valsIn.as<int>(), perm8_.data(), (int)n, 0, 32, stream));
        CUDA_VERIFY(cub::DeviceReduce::Sum(tmp.data, sumBytes, norms.as<float>(), sc + 4, (int)n, stream));
    }
    fill_float_kernel<<<(unsigned)ceil_div(padRows, 256), 256, 0, stream>>>(bias8_.data(), padRows, -INFINITY);
    CUDA_CHECK_LAST();
    tc_prepare_rows8_kernel<<<rowBlocks, warps * 32, 0, stream>>>(
            rows_, yHalf_, n, d, center_.data(), sc, perm8_.data(), y8_.data(), bias8_.data(), nullptr, nullptr, sc + 1);
    CUDA_CHECK_LAST();
    runTileBias(bias8_.data(), n, tileBias8_.data(), stream);
    float h[5];
    CUDA_VERIFY(cudaMemcpyAsync(h, sc, sizeof(h), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    scale8_ = h[0];
    maxYhat_ = std::sqrt(h[1]) * 1.0001f;
    maxRy_ = std::sqrt(h[2]) * 1.0001f;
    maxYc_ = std::sqrt(h[3]) * 1.0001f;
    const float c1 = 1.01f * (ldexpf(1.f, -10) + (float)kDpad8 * ldexpf(1.f, -22));
    const float meanNorm = h[4] / (float)n;
    int8Fit_ = maxRy_ <= kInt8Fitness * c1 * meanNorm && std::isfinite(maxYc_) && std::isfinite(maxYhat_);
    int8Ready_ = true;
    if (!int8Fit_) { // the fp16 layout serves this database: give the memory back
        y8_.clear();
        bias8_.clear();
        perm8_.clear();
        tileBias8_.clear();
    }
}

bool FlatTcDatabase::int8Eligible(int k, const FlatTcShard* shard) const {
    // sharded searches pool thresholds across ranks, and centred scores of shards with different centres differ by a
    // per-query offset: they stay fp16
    return metric_ == METRIC_L2 && d_ > 112 && d_ <= kDpad8 && k >= 2 && k <= 128 && shard == nullptr;
}

// one search call: the schedule, the launch configuration and the bias arrays (the masked copies under a row mask)
struct FlatTcDatabase::Call {
    cudaStream_t stream;
    const FlatTcSchedule& s;
    int KB, kSteps;
    SmemPlan sp;
    const float* bias;
    const float* tileBias;
    CUtensorMap mapY;
    const FlatTcShard* shard;
    bool int8;       // the int8 layout
    const int* perm; // the layout's stored position -> row id (null: identity)
};

// device state of one query batch
struct FlatTcDatabase::Batch {
    const float* Q; // [nq][d]
    int64_t nq, qPairs;
    GpuMemoryReservation q16, scal, eps, thr, flags, baseKey, baseId;
    GpuMemoryReservation invQ; // int8: per-query 1 / (s_q * s_y)
    CUtensorMap mapQ;
};

// the batch's queries -> scaled fp16 (int8: centred, quantised) tiles, eps and thresholds; empty base lists
void FlatTcDatabase::prepareQueries(const Call& c, Batch& b) const {
    const int64_t nq = b.nq, qPairs = b.qPairs;
    cudaStream_t stream = c.stream;
    b.q16 = res_->temp(device_, c.int8 ? (size_t)qPairs * kUnitM * kDpad8 : sizeof(__half) * qPairs * kUnitM * dpad_);
    b.scal = res_->temp(device_, sizeof(float) * 4); // [absmax, qScale, inv, -]
    b.eps = res_->temp(device_, sizeof(float) * nq);
    b.thr = res_->temp(device_, sizeof(float) * nq);
    b.flags = res_->temp(device_, sizeof(int) * (nq + 1));
    b.baseKey = res_->temp(device_, c.s.streaming ? sizeof(float) : sizeof(float) * nq * c.s.LIST);
    b.baseId = res_->temp(device_, c.s.streaming ? sizeof(int) : sizeof(int) * nq * c.s.LIST);

    // error model constants (DESIGN.md): fp16 rounding of both operands + fp32 accumulation slack
    const float c1 = 1.01f * (ldexpf(1.f, -10) + (float)dpad_ * ldexpf(1.f, -22));
    const float c2 = (float)(dpad_ + 16) * ldexpf(1.f, -24);

    CUDA_VERIFY(cudaMemsetAsync(b.scal.data, 0, sizeof(float) * 4, stream));
    CUDA_VERIFY(cudaMemsetAsync(b.flags.data, 0, sizeof(int) * (nq + 1), stream));
    CUDA_VERIFY(cudaMemsetAsync(b.q16.data, 0, b.q16.size, stream));
    if (c.int8) {
        b.invQ = res_->temp(device_, sizeof(float) * nq);
        CUDA_VERIFY(cudaMemcpyAsync(b.scal.data, &scale8_, sizeof(float), cudaMemcpyHostToDevice, stream));
        tc_prepare_queries8_kernel<<<(unsigned)ceil_div(nq, 8), 256, 0, stream>>>(
                b.Q, nq, d_, center_.data(), b.scal.as<float>(), maxYhat_, maxRy_, maxYc_, c2, b.q16.as<int8_t>(),
                b.invQ.as<float>(), b.eps.as<float>(), b.thr.as<float>());
        CUDA_CHECK_LAST();
    } else {
        float* sc = b.scal.as<float>();
        runAbsMax(b.Q, nq * d_, sc + 0, stream);
        tc_query_scale_kernel<<<1, 1, 0, stream>>>(sc + 0, scale_, sc + 1, sc + 2);
        CUDA_CHECK_LAST();
        tc_prepare_queries_kernel<<<(unsigned)ceil_div(nq, 8), 256, 0, stream>>>(
                b.Q, nq, d_, dpad_, sc + 1, scale_, c1, c2, maxNorm_, b.q16.as<__half>(), b.eps.as<float>(),
                b.thr.as<float>());
        CUDA_CHECK_LAST();
    }
    if (!c.s.streaming) {
        int64_t cnt = nq * c.s.LIST;
        tc_init_base_kernel<<<(unsigned)ceil_div(cnt, 256), 256, 0, stream>>>(b.baseKey.as<float>(), b.baseId.as<int>(), cnt);
        CUDA_CHECK_LAST();
    }
    b.mapQ = c.int8 ? makeTileMap8(b.q16.as<int8_t>(), qPairs * kUnitM, kTileM)
                    : makeTileMap(b.q16.as<__half>(), qPairs * kUnitM, dpad_, kTileM);
}

// One round: score its tiles and emit candidates, then fold them into the base lists and thresholds (and, sharded,
// pool the thresholds across the ranks) -- or, streaming, select and re-rank in one pass into outD / outI.
void FlatTcDatabase::runRound(const Call& c, const Batch& b, const FlatTcRound& r, uint2* arena, int* counts, float* contrib,
                              float* outD, idx_t* outI) const {
    const FlatTcSchedule& s = c.s;
    cudaStream_t stream = c.stream;
    const int nq = (int)b.nq;
    TcParams p = roundParams(c.sp, c.KB, c.kSteps, b.nq, b.qPairs, r, s.T, s.permA, s.permB, b.scal.as<float>() + 2);
    p.bias = c.bias;
    p.tileMaxBias = c.tileBias;
    p.tileMinBias = c.tileBias + s.T + 1; // second half of the array (see tc_tile_max_bias_kernel)
    p.thr = b.thr.as<float>();
    p.eps = b.eps.as<float>();
    p.invQ = c.int8 ? b.invQ.as<float>() : nullptr;
    p.cand = arena;
    p.candCount = counts;
    if (p.tileBegin < p.tileEnd) {
        launchTc<false>(b.mapQ, c.mapY, p, std::min(p.numUnits, s.sms), c.sp, stream, s.streaming);
    } else { // this shard has no tiles in this round of the common schedule: no candidates
        CUDA_VERIFY(cudaMemsetAsync(counts, 0, (size_t)p.numUnits * kSegsPerUnit * sizeof(int), stream));
    }
    if (s.streaming) { // select + exact re-rank fused: one warp per query
        const int fw = 8;
        KernelTiming::begin("tc_argmin_finish", stream);
        withBool(metric_ == METRIC_L2, [&](auto l2) {
            withBool(yHalf_ != 0, [&](auto yh) {
                tc_argmin_finish_kernel<l2, yh><<<(unsigned)ceil_div(nq, fw), fw * 32, 0, stream>>>(
                        nq, d_, r.slices, kParts, arena, r.cap, counts, b.eps.as<float>(), b.Q, rows_, perm_.data(), outD, outI,
                        b.flags.as<int>());
            });
        });
        KernelTiming::end("tc_argmin_finish", stream);
        CUDA_CHECK_LAST();
        return;
    }
    // the two selection kernels take the same arguments
    const auto sel = s.useBisect ? tc_select_bisect_kernel : tc_select_kernel;
    const size_t listBytes = SmemTopK<int>::bytes(s.LIST, kSelectBuf);
    const int selWarps = s.useBisect ? kSelWarps : (int)std::max<size_t>(1, std::min<size_t>(8, (48 * 1024) / listBytes));
    const size_t selSmem = s.useBisect ? sizeof(uint2) * kSelCap * kSelWarps : listBytes * selWarps;
    CUDA_VERIFY(cudaFuncSetAttribute(sel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)selSmem));
    KernelTiming::begin("tc_select", stream);
    sel<<<(unsigned)ceil_div(nq, selWarps), selWarps * 32, selSmem, stream>>>(
            nq, s.k, s.LIST, r.slices, kParts, arena, r.cap, counts, b.eps.as<float>(), b.baseKey.as<float>(),
            b.baseId.as<int>(), b.thr.as<float>(), b.flags.as<int>(), contrib, s.kFrac);
    KernelTiming::end("tc_select", stream);
    CUDA_CHECK_LAST();
    if (c.shard) {
        KernelTiming::begin("tc_pool", stream);
        // ONE small all-reduce per round (2 floats per query): every shard then filters against a
        // threshold certified by the pooled evidence of all shards
        c.shard->comm->allReduceMax(contrib, (size_t)2 * nq, stream);
        tc_pooled_thr_kernel<<<(unsigned)ceil_div(nq, 256), 256, 0, stream>>>(nq, contrib, b.eps.as<float>(), b.thr.as<float>());
        KernelTiming::end("tc_pool", stream);
        CUDA_CHECK_LAST();
    }
}

// exact re-rank of the base lists into outD / outI, sorted by (distance, id)
void FlatTcDatabase::rerank(const Call& c, const Batch& b, float* outD, idx_t* outI) const {
    const FlatTcSchedule& s = c.s;
    cudaStream_t stream = c.stream;
    const int rrWarps = (int)std::max<size_t>(1, std::min<size_t>(8, (48 * 1024) / SmemTopK<int>::bytes(s.KL, 64)));
    const size_t rrSmem = SmemTopK<int>::bytes(s.KL, 64) * rrWarps;
    KernelTiming::begin("tc_rerank", stream);
    withBool(metric_ == METRIC_L2, [&](auto l2) {
        withBool(yHalf_ != 0, [&](auto yh) {
            auto kern = tc_rerank_kernel<l2, yh>;
            CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rrSmem));
            kern<<<(unsigned)ceil_div(b.nq, rrWarps), rrWarps * 32, rrSmem, stream>>>(
                    (int)b.nq, d_, s.k, s.LIST, s.KL, b.Q, rows_, c.perm, b.baseId.as<int>(), b.baseKey.as<float>(),
                    c.shard ? b.thr.as<float>() : nullptr, outD, outI);
        });
    });
    KernelTiming::end("tc_rerank", stream);
    CUDA_CHECK_LAST();
}

// certificate failures -> exact SIMT recompute into outD / outI; returns their number
int FlatTcDatabase::recomputeFallbacks(const Call& c, const Batch& b, const uint32_t* rowMask, float* outD, idx_t* outI) const {
    const int k = c.s.k;
    const int64_t nq = b.nq;
    cudaStream_t stream = c.stream;
    auto list = res_->temp(device_, sizeof(int) * nq);
    int* countDev = b.flags.as<int>() + nq;
    tc_collect_flags_kernel<<<(unsigned)ceil_div(nq, 256), 256, 0, stream>>>(b.flags.as<int>(), (int)nq, list.as<int>(), countDev);
    CUDA_CHECK_LAST();
    int nflag = 0;
    CUDA_VERIFY(cudaMemcpyAsync(&nflag, countDev, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    if (nflag > 0) {
        auto fq = res_->temp(device_, sizeof(float) * (size_t)nflag * d_);
        auto fD = res_->temp(device_, sizeof(float) * (size_t)nflag * k);
        auto fI = res_->temp(device_, sizeof(idx_t) * (size_t)nflag * k);
        tc_gather_queries_kernel<<<nflag, 128, 0, stream>>>(b.Q, list.as<int>(), d_, fq.as<float>());
        CUDA_CHECK_LAST();
        runFlatExact(
                res_, device_, fq.as<float>(), nflag, rows_, n_, d_, k, metric_, 0, fD.as<float>(), fI.as<idx_t>(), stream,
                yHalf_, 0.f, rowMask);
        tc_scatter_results_kernel<<<nflag, 128, 0, stream>>>(fD.as<float>(), fI.as<idx_t>(), list.as<int>(), k, outD, outI);
        CUDA_CHECK_LAST();
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
    return nflag;
}

int64_t FlatTcDatabase::search(const float* Q, int64_t nqAll, int k, float* outD, idx_t* outI, cudaStream_t stream,
                               const FlatTcShard* shard, const uint32_t* rowMask) {
    FB_THROW_IF_NOT_MSG(!dirty_, "FlatTcDatabase::search before prepare");
    if (nqAll == 0)
        return 0;
    FB_THROW_IF_NOT(flatTcSupported(d_, k, n_));
    bool int8 = int8Eligible(k, shard);
    if (int8 && !int8Ready_)
        prepareInt8(stream);
    int8 = int8 && int8Fit_;
    if (!int8 && !fp16Ready_)
        prepareFp16(stream);
    lastBits_ = int8 ? 8 : 16;
    const DeviceVector<float>& biasL = int8 ? bias8_ : bias_;
    const DeviceVector<float>& tileBiasL = int8 ? tileBias8_ : tileBias_;
    const int* perm = int8 ? perm8_.data() : perm_.data();
    const float* bias = biasL.data();
    const float* tileBias = tileBiasL.data();
    GpuMemoryReservation maskedBias, maskedTileBias;
    if (rowMask) {
        // an excluded row gets a -inf bias: its score can then never pass a round's threshold, exactly as the
        // padding rows past n.  The certificate's maxima over all rows stay valid bounds.
        maskedBias = res_->temp(device_, sizeof(float) * biasL.size());
        maskedTileBias = res_->temp(device_, sizeof(float) * tileBiasL.size());
        const int64_t padRows = (int64_t)biasL.size();
        mask_bias_kernel<<<(unsigned)ceil_div(padRows, (int64_t)256), 256, 0, stream>>>(
                bias, perm, rowMask, n_, padRows, maskedBias.as<float>());
        CUDA_CHECK_LAST();
        runTileBias(maskedBias.as<float>(), n_, maskedTileBias.as<float>(), stream);
        bias = maskedBias.as<float>();
        tileBias = maskedTileBias.as<float>();
    }
    const int KB = dpad_ / kKBlock;
    const int kSteps = (d_ + 15) / 16;
    const FlatTcSchedule s = planFlatTcSchedule(
            n_, k, res_->numSMs(device_), shard ? shard->comm->size() : 0, shard ? shard->maxTiles : 0, int8);
    const SmemPlan sp = planSmem(KB, kSteps, int8);
    const CUtensorMap mapY = int8 ? makeTileMap8(y8_.data(), n_, sp.boxRows)
                                  : makeTileMap(y16_.data(), n_, dpad_, sp.boxRows, sp.ksplit);
    const Call c{stream, s, KB, kSteps, sp, bias, tileBias, mapY, shard, int8, perm};
    int64_t fallbacks = 0;
    for (int64_t qb = 0; qb < nqAll; qb += s.qBatch) {
        Batch b;
        b.Q = Q + qb * d_;
        b.nq = std::min(s.qBatch, nqAll - qb);
        b.qPairs = ceil_div(b.nq, kUnitM);
        prepareQueries(c, b);
        const FlatTcRounds plan = s.rounds(b.qPairs);
        auto arena = res_->temp(device_, plan.arenaBytes);
        auto counts = res_->temp(device_, plan.countBytes);
        GpuMemoryReservation contrib;
        if (shard)
            contrib = res_->temp(device_, sizeof(float) * 2 * b.nq);
        float* oD = outD + qb * k;
        idx_t* oI = outI + qb * k;
        for (const FlatTcRound& r : plan.rounds)
            runRound(c, b, r, arena.as<uint2>(), counts.as<int>(), contrib.as<float>(), oD, oI);
        if (!s.streaming)
            rerank(c, b, oD, oI);
        fallbacks += recomputeFallbacks(c, b, rowMask, oD, oI);
    }
    return fallbacks;
}

void runFlatTcScoresDebug(const void* Q, int64_t nq, const void* Y, int64_t n, int dpad, bool s8, float* S,
                          cudaStream_t stream) {
    FB_THROW_IF_NOT(dpad % kKBlock == 0 && dpad <= kMaxKB * kKBlock);
    FB_THROW_IF_NOT_MSG(!s8 || dpad == kDpad8, "int8 scores take rows of 128");
    const int KB = dpad / kKBlock;
    const int kSteps = dpad / 16; // debug seam: operands arrive padded
    SmemPlan sp = planSmem(KB, kSteps, s8);
    const size_t rowBytes = s8 ? (size_t)kDpad8 : sizeof(__half) * dpad;
    CUtensorMap my = s8 ? makeTileMap8((const int8_t*)Y, n, sp.boxRows)
                        : makeTileMap((const __half*)Y, n, dpad, sp.boxRows, sp.ksplit);
    const int64_t numTiles = ceil_div(n, kTileN);
    const int64_t qPairs = ceil_div(nq, kUnitM);
    // the kernel reads whole 128-row query tiles: zero-padded private copy
    void* qpad = nullptr;
    CUDA_VERIFY(cudaMallocAsync(&qpad, rowBytes * qPairs * kUnitM, stream));
    CUDA_VERIFY(cudaMemsetAsync(qpad, 0, rowBytes * qPairs * kUnitM, stream));
    CUDA_VERIFY(cudaMemcpyAsync(qpad, Q, rowBytes * nq, cudaMemcpyDeviceToDevice, stream));
    // scale (1.0) for the debug run; the dump path never reads biases
    float* one = nullptr;
    CUDA_VERIFY(cudaMallocAsync(&one, sizeof(float), stream));
    float h1 = 1.f;
    CUDA_VERIFY(cudaMemcpyAsync(one, &h1, sizeof(float), cudaMemcpyHostToDevice, stream));
    // every tile in one slice, unpermuted
    const FlatTcRound all{0, (int)numTiles, 1, (int)numTiles, 0};
    TcParams p = roundParams(sp, KB, kSteps, nq, qPairs, all, numTiles, 1, 0, one);
    CUtensorMap mq = s8 ? makeTileMap8((const int8_t*)qpad, qPairs * kUnitM, kTileM)
                        : makeTileMap((const __half*)qpad, qPairs * kUnitM, dpad, kTileM);
    p.dump = S;
    p.dumpLd = numTiles * kTileN; // S must be [nq][numTiles*128]
    int dev = 0, sms = 0;
    CUDA_VERIFY(cudaGetDevice(&dev));
    CUDA_VERIFY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    launchTc<true>(mq, my, p, (int)std::min<int64_t>(p.numUnits, sms), sp, stream);
    CUDA_VERIFY(cudaFreeAsync(qpad, stream));
    CUDA_VERIFY(cudaFreeAsync(one, stream));
}

} // namespace fb200
