// faiss_b200 -- exact fp32 brute-force k-NN (SIMT) + row-wise merge + small utility kernels.
//
// What it replaces in the reference: runDistance<float> (faiss/gpu/impl/Distance.cu:121-405):
// cuBLAS SGEMM -> materialised fp32 tile in HBM -> l2SelectMinK -> second-level blockSelect.
// Here one kernel computes a [TQ x TN] distance tile in registers and feeds it straight into
// per-query shared-memory top-k lists (select.cuh); distances never reach HBM.  A database split
// (gridDim.y) fills the 132 SMs when nq is small; partial lists are merged by runMergeTopK.
//
// Arithmetic: direct form, accumulated strictly in dimension order with FMA:
//   L2: acc = fma(q_i - y_i, q_i - y_i, acc)     IP: acc = fma(q_i, y_i, acc)
// This is the canonical distance of this library: the tensor-core path re-ranks with the same
// expression, so both paths return bit-identical distances.
//
// The other metrics of the reference (L1, Linf, Lp, Canberra, BrayCurtis, JensenShannon, Jaccard, Gower;
// role of runGeneralDistance, faiss/gpu/impl/Distance.cuh:223-289, which materialises the distance tile
// and selects in a second pass) are further instantiations of the same kernel: the per-component
// distance is a template parameter (the Op* structs below), everything else is shared.
#include <cfloat>

#include <cuda_fp16.h>

#include "kernels.h"
#include "select.cuh"

namespace fb200 {

// ------------------------------------------------------------------------------------------
// norms
// ------------------------------------------------------------------------------------------
__global__ void l2_norms_kernel(const float* __restrict__ x, int64_t n, int d, float* __restrict__ norms) {
    int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n)
        return;
    const float* p = x + row * d;
    float acc = 0.f;
    for (int i = lane_id(); i < d; i += 32) {
        float v = p[i];
        acc = fmaf(v, v, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        acc += __shfl_xor_sync(kFullMask, acc, o);
    if (lane_id() == 0)
        norms[row] = acc;
}

void runL2Norms(const float* x, int64_t n, int d, float* norms, cudaStream_t stream) {
    if (n == 0)
        return;
    int warps = 8;
    l2_norms_kernel<<<(unsigned)ceil_div(n, warps), warps * 32, 0, stream>>>(x, n, d, norms);
    CUDA_CHECK_LAST();
}

// ------------------------------------------------------------------------------------------
// exact tile kernel
// ------------------------------------------------------------------------------------------
constexpr int kDK = 16;

template <int TQ, int TN>
struct ExactCfg {
    static constexpr int kThreads = 256;
    static constexpr int TXN = TN / 4;           // threads along n, 4 vectors each
    static constexpr int TYQ = kThreads / TXN;   // threads along q
    static constexpr int RQ = TQ / TYQ;          // queries per thread
    static constexpr int QS = TQ + 4;            // padded row strides (floats), keep 16B alignment
    static constexpr int YS = TN + 4;
    static constexpr int BUF = 2 * TN;
    static_assert(RQ >= 1, "bad config");
};

// ------------------------------------------------------------------------------------------
// distance ops: accumulator state, a per-component update applied in dimension order, a finish step.
// Each update is the reference CPU expression (VectorDistance<mt>, faiss/utils/simd_impl/
// distances_autovec-inl.h:181-304).  Where a component takes more than one operation, __fadd_rn /
// __fmul_rn keep nvcc (--fmad=true) from contracting them into an FMA the CPU does not do.
//   kSimilarity  larger is better: keys are the negated distance, so every list, merge and the k = 1
//                packed atomicMin keep "smaller key is better"
//   kPadNeutral  a zero-filled component (q = y = 0) leaves the state unchanged; the others stop the last
//                16-component chunk at d instead
//   kSentinel    a distance that is NaN or not strictly better than the missing-result sentinel (FLT_MAX,
//                -FLT_MAX for a similarity) is never kept: the CPU heap inserts only when C::cmp(top, d)
//                holds against its neutral element.  L2 / IP keep their original filter (NaN only).
// ------------------------------------------------------------------------------------------
struct Acc1 {
    float s;
};
struct Acc2 {
    float a, b;
};

struct OpL2 {
    static constexpr bool kSimilarity = false, kPadNeutral = true, kSentinel = false;
    using Acc = Acc1;
    __device__ static void init(Acc& a) { a.s = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) {
        const float t = q - y;
        a.s = fmaf(t, t, a.s);
    }
    __device__ static float finish(const Acc& a, float) { return a.s; }
};
struct OpIP {
    static constexpr bool kSimilarity = true, kPadNeutral = true, kSentinel = false;
    using Acc = Acc1;
    __device__ static void init(Acc& a) { a.s = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) { a.s = fmaf(q, y, a.s); }
    __device__ static float finish(const Acc& a, float) { return a.s; }
};
struct OpL1 {
    static constexpr bool kSimilarity = false, kPadNeutral = true, kSentinel = true;
    using Acc = Acc1;
    __device__ static void init(Acc& a) { a.s = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) { a.s = a.s + fabsf(q - y); }
    __device__ static float finish(const Acc& a, float) { return a.s; }
};
struct OpLinf {
    static constexpr bool kSimilarity = false, kPadNeutral = true, kSentinel = true;
    using Acc = Acc1;
    __device__ static void init(Acc& a) { a.s = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) { a.s = fmaxf(a.s, fabsf(q - y)); }
    __device__ static float finish(const Acc& a, float) { return a.s; }
};
// powf(0, p) is 0 only for p > 0: padding is bounded for every p
struct OpLp {
    static constexpr bool kSimilarity = false, kPadNeutral = false, kSentinel = true;
    using Acc = Acc1;
    __device__ static void init(Acc& a) { a.s = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float p) { a.s = __fadd_rn(a.s, powf(fabsf(q - y), p)); }
    __device__ static float finish(const Acc& a, float) { return a.s; }
};
// a = b = 0 is 0/0 = NaN, as on the CPU: such rows are excluded, and padding must not produce it
struct OpCanberra {
    static constexpr bool kSimilarity = false, kPadNeutral = false, kSentinel = true;
    using Acc = Acc1;
    __device__ static void init(Acc& a) { a.s = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) {
        a.s = __fadd_rn(a.s, fabsf(q - y) / __fadd_rn(fabsf(q), fabsf(y)));
    }
    __device__ static float finish(const Acc& a, float) { return a.s; }
};
struct OpBrayCurtis {
    static constexpr bool kSimilarity = false, kPadNeutral = true, kSentinel = true;
    using Acc = Acc2;
    __device__ static void init(Acc& a) { a.a = a.b = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) {
        a.a = a.a + fabsf(q - y);
        a.b = a.b + fabsf(q + y);
    }
    __device__ static float finish(const Acc& a, float) { return a.a / a.b; }
};
// 0.5 * sum(-a log(m/a) - b log(m/b)), m = (a+b)/2; a zero component gives NaN, as on the CPU
struct OpJensenShannon {
    static constexpr bool kSimilarity = false, kPadNeutral = false, kSentinel = true;
    using Acc = Acc1;
    __device__ static void init(Acc& a) { a.s = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) {
        const float m = __fmul_rn(0.5f, __fadd_rn(q, y));
        const float kl1 = __fmul_rn(-q, logf(m / q));
        const float kl2 = __fmul_rn(-y, logf(m / y));
        a.s = __fadd_rn(a.s, __fadd_rn(kl1, kl2));
    }
    __device__ static float finish(const Acc& a, float) { return __fmul_rn(0.5f, a.s); }
};
struct OpJaccard {
    static constexpr bool kSimilarity = true, kPadNeutral = true, kSentinel = true;
    using Acc = Acc2;
    __device__ static void init(Acc& a) { a.a = a.b = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) {
        a.a = a.a + fminf(q, y);
        a.b = a.b + fmaxf(q, y);
    }
    __device__ static float finish(const Acc& a, float) { return a.a / a.b; }
};
// a = sum, b = valid dimensions; a NaN sum is the "invalid pair" state (out-of-range numeric value, or a
// numeric value against a categorical one) and survives every later add.  Padding would count as a valid
// numeric dimension.
struct OpGower {
    static constexpr bool kSimilarity = false, kPadNeutral = false, kSentinel = true;
    using Acc = Acc2;
    __device__ static void init(Acc& a) { a.a = a.b = 0.f; }
    __device__ static void update(Acc& a, float q, float y, float) {
        if (q != q || y != y)
            return;
        if (q >= 0.f && y >= 0.f)
            a.a = (q > 1.f || y > 1.f) ? CUDART_NAN_F : a.a + fabsf(q - y);
        else if (q < 0.f && y < 0.f)
            a.a = a.a + (q != y ? 1.f : 0.f);
        else
            a.a = CUDART_NAN_F;
        a.b = a.b + 1.f;
    }
    // b = 0 (no valid dimension) gives 0/0 = NaN, as the CPU returns
    __device__ static float finish(const Acc& a, float) { return a.a / a.b; }
};

// What a CTA does with its distance tile:
//   List    offer it to per-query shared-memory top-k lists (k > 1)
//   Argmin  keep the best (key, row) per query with a packed atomicMin (k = 1)
//   Store   write every Op::finish value to D[q * ldD + row] (all-pairs distances, no selection, no lists);
//           the raw distance, not the key, and NaN as computed
enum class Epi { List, Argmin, Store };

// MASK: only rows whose bit is set in rowMask (bit r & 31 of word r >> 5) enter the results (SearchParameters::sel)
template <int TQ, int TN, class Op, Epi E, bool MASK>
__global__ void __launch_bounds__(256) flat_exact_kernel(
        const float* __restrict__ Q,
        int nq,
        const void* __restrict__ Yv, // [n][d] fp32, or fp16 when yHalf (useFloat16 storage: widened on load, same arithmetic)
        int yHalf,
        int64_t n,
        int d,
        int k,
        int LIST,
        int64_t rowsPerSplit,
        float arg,                  // metric_arg (the exponent of METRIC_Lp)
        float* __restrict__ partD,  // [nq, nsplit, k]   keys ("smaller is better"); Store: D [nq][ldD]
        idx_t* __restrict__ partI,  // [nq, nsplit, k]   row index (or -1)
        const uint32_t* __restrict__ rowMask,
        int64_t ldD)
{
    constexpr bool K1 = E == Epi::Argmin;
    constexpr bool STORE = E == Epi::Store;
    using C = ExactCfg<TQ, TN>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* Qs = reinterpret_cast<float*>(smem_raw);            // [kDK][QS]
    float* Ys = Qs + kDK * C::QS;                              // [kDK][YS]
    int* cntS = reinterpret_cast<int*>(Ys + kDK * C::YS);      // [TQ]
    float* thrS = reinterpret_cast<float*>(cntS + TQ);         // [TQ]
    unsigned long long* best = reinterpret_cast<unsigned long long*>(thrS + TQ); // [TQ] (K1)
    unsigned char* listBase = reinterpret_cast<unsigned char*>(best + TQ);
    const size_t perQuery = E == Epi::List ? SmemTopK<int>::bytes(LIST, C::BUF) : 0;

    const int tid = threadIdx.x;
    const int tx = tid % C::TXN;
    const int ty = tid / C::TXN;
    const int warp = tid >> 5;
    const int q0 = blockIdx.x * TQ;
    const int split = blockIdx.y;
    const int nsplit = gridDim.y;
    const int64_t r0 = (int64_t)split * rowsPerSplit;
    const int64_t r1 = min(n, r0 + rowsPerSplit);

    auto queueOf = [&](int q) {
        SmemTopK<int> s;
        unsigned char* base = listBase + perQuery * q;
        s.keys = reinterpret_cast<float*>(base);
        s.ids = reinterpret_cast<int*>(base + sizeof(float) * (LIST + C::BUF));
        s.bkeys = s.keys + LIST;
        s.bids = s.ids + LIST;
        s.LIST = LIST;
        s.BUF = C::BUF;
        s.k = k;
        return s;
    };

    if (!STORE && tid < TQ) {
        cntS[tid] = 0;
        thrS[tid] = CUDART_INF_F;
        best[tid] = ~0ull;
    }
    if (E == Epi::List) {
        for (int q = warp; q < TQ; q += 8) {
            SmemTopK<int> s = queueOf(q);
            s.init();
        }
    }
    __syncthreads();

    const bool vec4 = ((d & 3) == 0);
    const float* Y = reinterpret_cast<const float*>(Yv);
    const __half* Yh = reinterpret_cast<const __half*>(Yv);

    for (int64_t nb = r0; nb < r1; nb += TN) {
        typename Op::Acc acc[C::RQ][4];
#pragma unroll
        for (int r = 0; r < C::RQ; r++)
#pragma unroll
            for (int c = 0; c < 4; c++)
                Op::init(acc[r][c]);

        for (int kk = 0; kk < d; kk += kDK) {
            // ---- stage Q chunk [TQ x 16] and Y chunk [TN x 16], transposed to [k][row]
            for (int e = tid; e < (TQ + TN) * 4; e += C::kThreads) {
                const bool isQ = e < TQ * 4;
                int ee = isQ ? e : e - TQ * 4;
                int row = ee >> 2, c4 = ee & 3;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                const float* src = nullptr;
                if (isQ) {
                    if (q0 + row < nq)
                        src = Q + (int64_t)(q0 + row) * d;
                } else {
                    if (nb + row < r1 && !yHalf)
                        src = Y + (nb + row) * d;
                }
                int col = kk + c4 * 4;
                if (!isQ && yHalf) {
                    if (nb + row < r1) {
                        const __half* hs = Yh + (nb + row) * d;
                        if (vec4 && col + 3 < d) {
                            const uint2 u = *reinterpret_cast<const uint2*>(hs + col);
                            const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
                            const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
                            v = make_float4(lo.x, lo.y, hi.x, hi.y);
                        } else {
                            if (col + 0 < d)
                                v.x = __half2float(hs[col + 0]);
                            if (col + 1 < d)
                                v.y = __half2float(hs[col + 1]);
                            if (col + 2 < d)
                                v.z = __half2float(hs[col + 2]);
                            if (col + 3 < d)
                                v.w = __half2float(hs[col + 3]);
                        }
                    }
                } else if (src) {
                    if (vec4 && col + 3 < d) {
                        v = *reinterpret_cast<const float4*>(src + col);
                    } else {
                        if (col + 0 < d)
                            v.x = src[col + 0];
                        if (col + 1 < d)
                            v.y = src[col + 1];
                        if (col + 2 < d)
                            v.z = src[col + 2];
                        if (col + 3 < d)
                            v.w = src[col + 3];
                    }
                }
                float* dst = isQ ? (Qs + row) : (Ys + row);
                const int stride = isQ ? C::QS : C::YS;
                dst[(c4 * 4 + 0) * stride] = v.x;
                dst[(c4 * 4 + 1) * stride] = v.y;
                dst[(c4 * 4 + 2) * stride] = v.z;
                dst[(c4 * 4 + 3) * stride] = v.w;
            }
            __syncthreads();
            auto component = [&](int i) {
                float4 yv = *reinterpret_cast<const float4*>(Ys + i * C::YS + tx * 4);
                float qv[C::RQ];
#pragma unroll
                for (int r = 0; r < C::RQ; r++)
                    qv[r] = Qs[i * C::QS + ty * C::RQ + r];
#pragma unroll
                for (int r = 0; r < C::RQ; r++) {
                    Op::update(acc[r][0], qv[r], yv.x, arg);
                    Op::update(acc[r][1], qv[r], yv.y, arg);
                    Op::update(acc[r][2], qv[r], yv.z, arg);
                    Op::update(acc[r][3], qv[r], yv.w, arg);
                }
            };
            if (Op::kPadNeutral || kk + kDK <= d) {
#pragma unroll
                for (int i = 0; i < kDK; i++)
                    component(i);
            } else {
                // last, partial chunk of an op for which a zero-filled component is not neutral
                for (int i = 0; i < d - kk; i++)
                    component(i);
            }
            __syncthreads();
        }

        if constexpr (STORE) {
            // this thread's 4 consecutive rows of each of its query rows: one 16-byte streaming store when the
            // 4 are in range and D's rows keep 16-byte alignment (nb - r0 and tx * 4 are multiples of 4)
            const int64_t c0 = nb + tx * 4;
            const bool vecStore = (ldD & 3) == 0 && (reinterpret_cast<uintptr_t>(partD) & 15) == 0 && c0 + 3 < r1;
#pragma unroll
            for (int r = 0; r < C::RQ; r++) {
                const int q = ty * C::RQ + r;
                if (q0 + q >= nq)
                    continue;
                float* out = partD + (int64_t)(q0 + q) * ldD + c0;
                if (vecStore) {
                    __stcs(reinterpret_cast<float4*>(out),
                           make_float4(Op::finish(acc[r][0], arg), Op::finish(acc[r][1], arg), Op::finish(acc[r][2], arg),
                                       Op::finish(acc[r][3], arg)));
                } else {
#pragma unroll
                    for (int c = 0; c < 4; c++)
                        if (c0 + c < r1)
                            __stcs(out + c, Op::finish(acc[r][c], arg));
                }
            }
        } else {
            // ---- offer the tile to the per-query lists
#pragma unroll
            for (int r = 0; r < C::RQ; r++) {
                const int q = ty * C::RQ + r;
                if (q0 + q >= nq)
                    continue;
                if (K1) {
                    unsigned long long mine = ~0ull;
#pragma unroll
                    for (int c = 0; c < 4; c++) {
                        int64_t row = nb + tx * 4 + c;
                        if (row < r1 && (!MASK || ((rowMask[row >> 5] >> (row & 31)) & 1u))) {
                            const float dist = Op::finish(acc[r][c], arg);
                            float key = Op::kSimilarity ? -dist : dist;
                            if (key == key && (!Op::kSentinel || key < FLT_MAX)) { // NaN never wins
                                unsigned long long p =
                                        ((unsigned long long)float_to_ordered(key) << 32) | (unsigned)(row - r0);
                                mine = min(mine, p);
                            }
                        }
                    }
                    if (mine < best[q])
                        atomicMin(&best[q], mine);
                } else {
                    const float thr = thrS[q];
                    SmemTopK<int> s = queueOf(q);
#pragma unroll
                    for (int c = 0; c < 4; c++) {
                        int64_t row = nb + tx * 4 + c;
                        const float dist = Op::finish(acc[r][c], arg);
                        float key = Op::kSimilarity ? -dist : dist;
                        if (row < r1 && key <= thr && (!Op::kSentinel || key < FLT_MAX) &&
                            (!MASK || ((rowMask[row >> 5] >> (row & 31)) & 1u))) {
                            int pos = atomicAdd(&cntS[q], 1);
                            s.keys[LIST + pos] = key;
                            s.ids[LIST + pos] = (int)(row - r0);
                        }
                    }
                }
            }
            if (!K1) {
                __syncthreads();
                for (int q = warp; q < TQ; q += 8) {
                    int c = cntS[q];
                    if (c > TN) {
                        SmemTopK<int> s = queueOf(q);
                        s.flush(c);
                        if (lane_id() == 0) {
                            cntS[q] = 0;
                            thrS[q] = s.threshold();
                        }
                    }
                }
                __syncthreads();
            }
        }
    }

    // ---- write partial results
    if (K1) {
        __syncthreads();
        if (tid < TQ && q0 + tid < nq) {
            unsigned long long b = best[tid];
            int64_t o = ((int64_t)(q0 + tid) * nsplit + split);
            if (b == ~0ull) {
                partD[o] = CUDART_INF_F;
                partI[o] = -1;
            } else {
                partD[o] = ordered_to_float((unsigned)(b >> 32));
                partI[o] = r0 + (int64_t)(unsigned)(b & 0xffffffffu);
            }
        }
    } else if (E == Epi::List) {
        for (int q = warp; q < TQ; q += 8) {
            if (q0 + q >= nq)
                continue;
            SmemTopK<int> s = queueOf(q);
            int c = cntS[q];
            if (c > 0)
                s.flush(c);
            __syncwarp();
            int64_t o = ((int64_t)(q0 + q) * nsplit + split) * k;
            for (int j = lane_id(); j < k; j += 32) {
                int id = s.ids[j];
                bool ok = id != IdLimits<int>::max();
                partD[o + j] = s.keys[j];
                partI[o + j] = ok ? r0 + id : -1;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// row-wise merge: [rows, nlists, kin] -> [rows, k]
// ------------------------------------------------------------------------------------------
template <bool IN_KEYSPACE>
__global__ void merge_topk_kernel(
        const float* __restrict__ inD,
        const idx_t* __restrict__ inI,
        int64_t rows,
        int nlists,
        int kin,
        const idx_t* __restrict__ idOffsets,
        int k,
        int LIST,
        int lowerIsBetter, // 0: a similarity (inner product, Jaccard), keys are the negated distances
        int64_t idBase,
        int64_t rowStride,  // elements between consecutive rows of one list
        int64_t listStride, // elements between consecutive lists of one row
        float* __restrict__ outD,
        idx_t* __restrict__ outI) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = lane_id();
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (row >= rows)
        return;
    constexpr int BUF = 64;
    unsigned char* base = smem_raw + SmemTopK<long long>::bytes(LIST, BUF) * warp;
    WarpTopK<long long> w;
    w.init(reinterpret_cast<float*>(base), reinterpret_cast<long long*>(base + sizeof(float) * (LIST + BUF)), LIST, BUF, k);

    const int64_t total = (int64_t)nlists * kin;
    const float* D = inD + row * rowStride;
    const idx_t* I = inI + row * rowStride;
    for (int64_t e0 = 0; e0 < total; e0 += 32) {
        int64_t e = e0 + lane;
        bool valid = e < total;
        float key = 0.f;
        long long id = -1;
        if (valid) {
            const int64_t l = e / kin;
            const int64_t at = l * listStride + (e - l * kin);
            id = I[at];
            key = D[at];
            if (id == -1) { // the "no result" marker; any other id is a stored one (IVF ids may be negative)
                valid = false;
            } else {
                if (idOffsets)
                    id += idOffsets[l];
                if (!IN_KEYSPACE && !lowerIsBetter)
                    key = -key;
            }
        }
        w.add(valid, key, id);
    }
    w.finish();
    for (int j = lane; j < k; j += 32) {
        long long id = w.q.ids[j];
        bool ok = id != IdLimits<long long>::max();
        float key = w.q.keys[j];
        float dis = lowerIsBetter ? key : -key;
        outD[row * k + j] = ok ? dis : (lowerIsBetter ? FLT_MAX : -FLT_MAX); // faiss/gpu/impl/Distance.cu:152-164
        outI[row * k + j] = ok ? (idx_t)id + idBase : -1;
    }
}

static int listSizeFor(int k, int minList) {
    return std::max(minList, next_pow2(k));
}

static void launchMerge(
        bool inKeyspace,
        const float* inD,
        const idx_t* inI,
        int64_t rows,
        int nlists,
        int kin,
        const idx_t* idOffsets,
        int k,
        MetricType metric,
        int64_t idBase,
        float* outD,
        idx_t* outI,
        cudaStream_t stream,
        bool listMajor = false) {
    if (rows == 0)
        return;
    int LIST = listSizeFor(k, 64);
    size_t per = SmemTopK<long long>::bytes(LIST, 64);
    int warps = (int)std::max<size_t>(1, std::min<size_t>(4, (96 * 1024) / per));
    size_t smem = per * warps;
    auto kern = inKeyspace ? merge_topk_kernel<true> : merge_topk_kernel<false>;
    CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)ceil_div(rows, warps), warps * 32, smem, stream>>>(
            inD, inI, rows, nlists, kin, idOffsets, k, LIST, is_similarity_metric(metric) ? 0 : 1, idBase,
            listMajor ? (int64_t)kin : (int64_t)nlists * kin, listMajor ? rows * (int64_t)kin : (int64_t)kin, outD, outI);
    CUDA_CHECK_LAST();
}

void runMergeTopK(
        const float* inD,
        const idx_t* inI,
        int64_t rows,
        int nlists,
        int kin,
        const idx_t* idOffsets,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream) {
    launchMerge(false, inD, inI, rows, nlists, kin, idOffsets, k, metric, 0, outD, outI, stream);
}

// inputs laid out [nlists][rows][kin] -- exactly what an all-gather of per-shard [rows][kin] results produces
void runMergeTopKListMajor(
        const float* inD,
        const idx_t* inI,
        int64_t rows,
        int nlists,
        int kin,
        const idx_t* idOffsets,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream) {
    launchMerge(false, inD, inI, rows, nlists, kin, idOffsets, k, metric, 0, outD, outI, stream, true);
}

// internal: inputs already in key space (IP negated)
void runMergeTopKKeyspace(
        const float* inD,
        const idx_t* inI,
        int64_t rows,
        int nlists,
        int kin,
        int k,
        MetricType metric,
        int64_t idBase,
        float* outD,
        idx_t* outI,
        cudaStream_t stream) {
    launchMerge(true, inD, inI, rows, nlists, kin, nullptr, k, metric, idBase, outD, outI, stream);
}

// ------------------------------------------------------------------------------------------
// host driver
// ------------------------------------------------------------------------------------------
template <int TQ, int TN, Epi E>
static void launchExact(
        const float* Q,
        int64_t nq,
        const void* Y,
        int yHalf,
        int64_t n,
        int d,
        int k,
        int LIST,
        MetricType metric,
        float metricArg,
        int nsplit,
        int64_t rowsPerSplit,
        float* partD,
        idx_t* partI,
        const uint32_t* rowMask,
        cudaStream_t stream,
        int64_t ldD = 0) {
    using C = ExactCfg<TQ, TN>;
    size_t smem = sizeof(float) * kDK * (C::QS + C::YS);
    if (E != Epi::Store)
        smem += TQ * (sizeof(int) + sizeof(float) + sizeof(unsigned long long));
    if (E == Epi::List)
        smem += SmemTopK<int>::bytes(LIST, C::BUF) * TQ;
    dim3 grid((unsigned)ceil_div(nq, TQ), (unsigned)nsplit);
    auto launch = [&](auto kern) {
        CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, C::kThreads, smem, stream>>>(
                Q, (int)nq, Y, yHalf, n, d, k, LIST, rowsPerSplit, metricArg, partD, partI, rowMask, ldD);
    };
    auto launchOp = [&](auto op) {
        using Op = decltype(op);
        if constexpr (E == Epi::Store)
            launch(flat_exact_kernel<TQ, TN, Op, E, false>);
        else if (rowMask)
            launch(flat_exact_kernel<TQ, TN, Op, E, true>);
        else
            launch(flat_exact_kernel<TQ, TN, Op, E, false>);
    };
    // METRIC_Lp arrives here with p != 1, 2: GpuIndexFlat::searchMetric_ sends those to L1 / L2
    switch (metric) {
        case METRIC_L2:
            launchOp(OpL2{});
            break;
        case METRIC_INNER_PRODUCT:
            launchOp(OpIP{});
            break;
        case METRIC_L1:
            launchOp(OpL1{});
            break;
        case METRIC_Linf:
            launchOp(OpLinf{});
            break;
        case METRIC_Lp:
            launchOp(OpLp{});
            break;
        case METRIC_Canberra:
            launchOp(OpCanberra{});
            break;
        case METRIC_BrayCurtis:
            launchOp(OpBrayCurtis{});
            break;
        case METRIC_JensenShannon:
            launchOp(OpJensenShannon{});
            break;
        case METRIC_Jaccard:
            launchOp(OpJaccard{});
            break;
        case METRIC_GOWER:
            launchOp(OpGower{});
            break;
        default:
            FB_THROW_FMT("unimplemented metric type %d", (int)metric); // faiss/gpu/impl/Distance.cuh:289
    }
    CUDA_CHECK_LAST();
}

// database split (gridDim.y): enough blocks to fill the chip (2 waves), slices of >= 8 tiles, < 2^31 rows
static void databaseSplit(int64_t ctas, int64_t nq, int TQ, int64_t n, int TN, int64_t& nsplit, int64_t& rowsPerSplit) {
    int64_t qTiles = ceil_div(nq, TQ);
    int64_t wantSplit = std::max<int64_t>(1, (ctas + qTiles - 1) / qTiles);
    int64_t maxSplit = std::max<int64_t>(1, n / (8 * TN));
    nsplit = std::min(wantSplit, maxSplit);
    nsplit = std::max(nsplit, ceil_div(n, (int64_t(1) << 30)));
    nsplit = std::min<int64_t>(nsplit, 65535);
    rowsPerSplit = n > 0 ? round_up(ceil_div(n, nsplit), TN) : TN;
    nsplit = n > 0 ? ceil_div(n, rowsPerSplit) : 1;
}

static void flatExactImpl(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        const void* Y,
        int yHalf,
        int64_t n,
        int d,
        int k,
        MetricType metric,
        float metricArg,
        int64_t idBase,
        float* outD,
        idx_t* outI,
        const uint32_t* rowMask,
        cudaStream_t stream) {
    if (!is_implemented_metric(metric))
        FB_THROW_FMT("unimplemented metric type %d", (int)metric);
    if (nq == 0)
        return;
    FB_THROW_IF_NOT(k >= 1 && k <= kMaxK);
    FB_THROW_IF_NOT_MSG(nq < (int64_t(1) << 31), "too many queries in one call");
    const bool K1 = (k == 1);
    int TQ, TN, LIST;
    if (K1) {
        TQ = 32;
        TN = 64;
        LIST = 0;
    } else {
        int p2 = next_pow2(k);
        if (p2 <= 256) {
            TQ = 32;
            TN = 64;
            LIST = std::max(128, p2);
        } else if (p2 <= 1024) {
            TQ = 16;
            TN = 64;
            LIST = p2;
        } else {
            TQ = 8;
            TN = 128;
            LIST = p2;
        }
    }
    int64_t nsplit, rowsPerSplit;
    databaseSplit(2 * res->numSMs(device), nq, TQ, n, TN, nsplit, rowsPerSplit);

    auto partD = res->temp(device, sizeof(float) * nq * nsplit * k);
    auto partI = res->temp(device, sizeof(idx_t) * nq * nsplit * k);

#define LAUNCH(TQ_, TN_, E_)                                                                         \
    launchExact<TQ_, TN_, E_>(                                                                       \
            Q, nq, Y, yHalf, n, d, k, LIST, metric, metricArg, (int)nsplit, rowsPerSplit, partD.as<float>(), partI.as<idx_t>(), rowMask, stream)
    if (K1) {
        LAUNCH(32, 64, Epi::Argmin);
    } else if (TQ == 32) {
        LAUNCH(32, 64, Epi::List);
    } else if (TQ == 16) {
        LAUNCH(16, 64, Epi::List);
    } else {
        LAUNCH(8, 128, Epi::List);
    }
#undef LAUNCH
    runMergeTopKKeyspace(
            partD.as<float>(), partI.as<idx_t>(), nq, (int)nsplit, k, k, metric, idBase, outD, outI, stream);
}

void runFlatExact(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        const void* Y,
        int64_t n,
        int d,
        int k,
        MetricType metric,
        int64_t idBase,
        float* outD,
        idx_t* outI,
        cudaStream_t stream,
        int yHalf,
        float metricArg,
        const uint32_t* rowMask) {
    flatExactImpl(res, device, Q, nq, Y, yHalf, n, d, k, metric, metricArg, idBase, outD, outI, rowMask, stream);
}

void runFlatArgmin(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        const float* Y,
        int64_t n,
        int d,
        MetricType metric,
        float* outD,
        idx_t* outI,
        cudaStream_t stream) {
    if (nq == 0)
        return;
    GpuMemoryReservation tmp;
    if (!outD) {
        tmp = res->temp(device, sizeof(float) * nq);
        outD = tmp.as<float>();
    }
    flatExactImpl(res, device, Q, nq, Y, 0, n, d, 1, metric, 0.f, 0, outD, outI, nullptr, stream);
}

void runFlatPairwise(
        GpuResources* res,
        int device,
        const float* Q,
        int64_t nq,
        const float* Y,
        int64_t n,
        int d,
        MetricType metric,
        float metricArg,
        float* D,
        int64_t ldD,
        cudaStream_t stream) {
    if (!is_implemented_metric(metric))
        FB_THROW_FMT("unimplemented metric type %d", (int)metric);
    if (nq == 0 || n == 0)
        return;
    FB_THROW_IF_NOT_MSG(nq < (int64_t(1) << 31), "too many queries in one call");
    // every CTA does the same work, so a split finer than the k-NN's keeps the last wave's imbalance small
    int64_t nsplit, rowsPerSplit;
    databaseSplit(32 * res->numSMs(device), nq, 32, n, 64, nsplit, rowsPerSplit);
    launchExact<32, 64, Epi::Store>(
            Q, nq, Y, 0, n, d, 0, 0, metric, metricArg, (int)nsplit, rowsPerSplit, D, nullptr, nullptr, stream, ldD);
}

// ------------------------------------------------------------------------------------------
// residual / gather
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float row_elem(const void* base, int yHalf, int64_t idx) {
    return yHalf ? __half2float(reinterpret_cast<const __half*>(base)[idx]) : reinterpret_cast<const float*>(base)[idx];
}

__global__ void calc_residual_kernel(
        const float* __restrict__ x,
        const void* __restrict__ c,
        int yHalf,
        const idx_t* __restrict__ assign,
        int64_t n,
        int d,
        float* __restrict__ out) {
    int64_t i = blockIdx.x;
    idx_t a = assign[i];
    for (int j = threadIdx.x; j < d; j += blockDim.x) {
        out[i * d + j] = (a < 0) ? CUDART_NAN_F : x[i * d + j] - row_elem(c, yHalf, a * d + j); // VectorResidual.cu:26-60
    }
}

void runCalcResidual(
        const float* x,
        const void* centroids,
        const idx_t* assign,
        int64_t n,
        int d,
        float* out,
        cudaStream_t stream,
        int yHalf) {
    if (n == 0)
        return;
    FB_THROW_IF_NOT(n < (int64_t(1) << 31));
    calc_residual_kernel<<<(unsigned)n, std::min(d, 256), 0, stream>>>(x, centroids, yHalf, assign, n, d, out);
    CUDA_CHECK_LAST();
}

__global__ void gather_rows_kernel(
        const void* __restrict__ src,
        int yHalf,
        const idx_t* __restrict__ ids,
        int64_t n,
        int d,
        float* __restrict__ out,
        bool missingAllOnes) {
    int64_t i = blockIdx.x;
    idx_t a = ids[i];
    for (int j = threadIdx.x; j < d; j += blockDim.x) {
        out[i * d + j] = a < 0 ? (missingAllOnes ? __int_as_float(-1) : CUDART_NAN_F) : row_elem(src, yHalf, a * d + j);
    }
}

void runGatherRows(
        const void* src, const idx_t* ids, int64_t n, int d, float* out, cudaStream_t stream, int yHalf, bool missingAllOnes) {
    if (n == 0)
        return;
    FB_THROW_IF_NOT(n < (int64_t(1) << 31));
    gather_rows_kernel<<<(unsigned)n, std::min(d, 256), 0, stream>>>(
            src, yHalf, ids, n, d, out, missingAllOnes);
    CUDA_CHECK_LAST();
}

} // namespace fb200
