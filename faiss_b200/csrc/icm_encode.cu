// faiss_b200 -- GpuIcmEncoder: one fused kernel runs LocalSearchQuantizer::icm_encode_impl for a page of rows
// (faiss/impl/LocalSearchQuantizer.cpp:539-795): every ILS iteration's perturbation, icm_iters x M conditional steps,
// evaluation and keep-best, with the codes, the best codes and the best error on chip.
//
// One warp per row.  obj[K] is spread over the lanes, k = j * 32 + lane, KPL = K / 32 (rounded up to a power of 2)
// floats per lane in registers; the argmin is a shuffle reduction.  Each step reads one row of K inner products
// x·C_mᵀ from the page's table and M - 1 rows of K contiguous floats from the C·Cᵀ table ([M*K][M*K], L2-resident:
// 16 MB at M = 8, K = 256), row (m2 * K + code[m2]) at column m * K, which is the CPU's binaries[m2][m][code[m2]][.].
//
// fp32 parity with the CPU:
//   unary   u = -2·ip + ‖C_m[k]‖²: the CPU's sgemm with alpha = -2 then fvec_add; the scaling by -2 is exact and the
//           add is one rounding (__fadd_rn keeps nvcc from contracting it into an FMA)
//   binary  obj[k] += 2·ip for m2 = 0 .. M-1, m2 != m, in ascending order, one rounding per add (:617-652)
//   argmin  HeapWithBucketsCMaxFloat<16, 1>::addn (:655-658): per bucket the first of equal values, buckets merged on
//           (value, index), leftovers only when strictly smaller -- for finite objectives that is the smallest k
//           among the minima, which is what the reduction on (value, k) computes
//   decode  0 + C_0[c_0] + C_1[c_1] + ... in m order (:774-779); the squared error is summed in lane order, so it
//           equals the CPU's fvec_L2sqr where fp32 is exact (integer data) and agrees to rounding elsewhere
//   keep    the new codes only when their error is strictly below the best so far (:571)
#include <math_constants.h>

#include <algorithm>
#include <exception>
#include <thread>

#include "icm_encode.h"
#include "index.h"
#include "kernels.h"

namespace fb200 {

namespace {

constexpr int kIcmWarps = 4; // rows per CTA
constexpr unsigned kMask = 0xffffffffu;

// error flags the kernel raises (checked on the host after each page)
constexpr int kBadCode = 1;
constexpr int kBadDraw = 2;

// squared L2 error of row x against the decode of `code`, the same value in every lane
__device__ __forceinline__ float icm_evaluate(
        const float* __restrict__ x,
        const float* __restrict__ cb,
        const int32_t* code,
        int M,
        int K,
        int d,
        int lane) {
    float acc = 0.f;
    for (int c = lane; c < d; c += 32) {
        float r = 0.f;
        for (int m = 0; m < M; m++)
            r = __fadd_rn(r, __ldg(cb + ((int64_t)m * K + code[m]) * d + c));
        const float diff = __fsub_rn(__ldg(x + c), r);
        acc = __fmaf_rn(diff, diff, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        acc += __shfl_xor_sync(kMask, acc, o);
    // the butterfly can round differently per lane: every lane takes lane 0's sum so that keep-best agrees
    return __shfl_sync(kMask, acc, 0);
}

template <int KPL>
__global__ void __launch_bounds__(kIcmWarps * 32) icm_encode_kernel(
        const float* __restrict__ ip,    // [rows][M*K]  x·Cᵀ
        const float* __restrict__ norms, // [M*K]        ‖C_m[k]‖²
        const float* __restrict__ cc,    // [M*K][M*K]   C·Cᵀ
        const float* __restrict__ cb,    // [M*K][d]     codebooks
        const float* __restrict__ x,     // [rows][d]
        int32_t* __restrict__ codes,     // [rows][M]    in: start codes, out: best codes
        const int2* __restrict__ draws,  // [ils][rows][nperts]  (m, k)
        int64_t rows,
        int M,
        int K,
        int d,
        int ils,
        int nperts,
        int icm_iters,
        int* __restrict__ bad) {
    extern __shared__ int32_t icm_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kIcmWarps + warp;
    if (i >= rows)
        return;
    int32_t* cur = icm_smem + warp * 2 * M;
    int32_t* best = cur + M;
    const int64_t MK = (int64_t)M * K;
    const float* xi = x + i * d;
    const float* ui = ip + i * MK;

    for (int m = lane; m < M; m += 32) {
        int32_t c = codes[i * M + m];
        if (c < 0 || c >= K) {
            atomicOr(bad, kBadCode);
            c = 0;
        }
        cur[m] = c;
        best[m] = c;
    }
    __syncwarp();
    float bestErr = icm_evaluate(xi, cb, cur, M, K, d, lane);

    for (int it = 0; it < ils; it++) {
        // perturb_codes (:673-688): the draws come in the CPU's order, later ones overwrite earlier ones
        if (lane == 0) {
            const int2* dr = draws + ((int64_t)it * rows + i) * nperts;
            for (int j = 0; j < nperts; j++) {
                const int2 p = dr[j];
                if (p.x < 0 || p.x >= M || p.y < 0 || p.y >= K)
                    atomicOr(bad, kBadDraw);
                else
                    cur[p.x] = p.y;
            }
        }
        __syncwarp();

        // icm_encode_step (:594-672)
        for (int iter = 0; iter < icm_iters; iter++) {
            for (int m = 0; m < M; m++) {
                float obj[KPL];
#pragma unroll
                for (int j = 0; j < KPL; j++) {
                    const int k = j * 32 + lane;
                    obj[j] = k < K ? __fadd_rn(-2.f * __ldg(ui + (int64_t)m * K + k), __ldg(norms + (int64_t)m * K + k))
                                   : CUDART_INF_F;
                }
                for (int m2 = 0; m2 < M; m2++) {
                    if (m2 == m)
                        continue;
                    const float* row = cc + ((int64_t)m2 * K + cur[m2]) * MK + (int64_t)m * K;
#pragma unroll
                    for (int j = 0; j < KPL; j++) {
                        const int k = j * 32 + lane;
                        if (k < K)
                            obj[j] = __fadd_rn(obj[j], 2.f * __ldg(row + k));
                    }
                }
                float bv = obj[0];
                int bk = lane;
#pragma unroll
                for (int j = 1; j < KPL; j++) {
                    if (obj[j] < bv) {
                        bv = obj[j];
                        bk = j * 32 + lane;
                    }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float ov = __shfl_xor_sync(kMask, bv, o);
                    const int ok = __shfl_xor_sync(kMask, bk, o);
                    if (ov < bv || (ov == bv && ok < bk)) {
                        bv = ov;
                        bk = ok;
                    }
                }
                __syncwarp(); // every lane has read cur[] before it changes
                if (lane == 0)
                    cur[m] = bk;
                __syncwarp();
            }
        }

        const float err = icm_evaluate(xi, cb, cur, M, K, d, lane);
        const bool better = err < bestErr;
        if (better)
            bestErr = err;
        for (int m = lane; m < M; m += 32) {
            if (better)
                best[m] = cur[m];
            else
                cur[m] = best[m];
        }
        __syncwarp();
    }
    for (int m = lane; m < M; m += 32)
        codes[i * M + m] = best[m];
}

void runIcmEncodeKernel(
        const float* ip,
        const float* norms,
        const float* cc,
        const float* cb,
        const float* x,
        int32_t* codes,
        const int2* draws,
        int64_t rows,
        int M,
        int K,
        int d,
        int ils,
        int nperts,
        int icm_iters,
        int* bad,
        cudaStream_t stream) {
    if (rows == 0)
        return;
    const unsigned grid = (unsigned)ceil_div(rows, kIcmWarps);
    const size_t smem = sizeof(int32_t) * 2 * M * kIcmWarps;
    auto launch = [&](auto kernel) {
        if (smem > 48 * 1024)
            CUDA_VERIFY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kernel<<<grid, kIcmWarps * 32, smem, stream>>>(ip, norms, cc, cb, x, codes, draws, rows, M, K, d, ils, nperts, icm_iters, bad);
        CUDA_CHECK_LAST();
    };
    const int kpl = next_pow2((int)ceil_div(K, 32));
    switch (kpl) {
        case 1: launch(icm_encode_kernel<1>); break;
        case 2: launch(icm_encode_kernel<2>); break;
        case 4: launch(icm_encode_kernel<4>); break;
        case 8: launch(icm_encode_kernel<8>); break;
        case 16: launch(icm_encode_kernel<16>); break;
        case 32: launch(icm_encode_kernel<32>); break;
        default: FB_THROW_FMT("K = %d is not supported", K);
    }
}

} // namespace

struct GpuIcmEncoder::Shard {
    std::shared_ptr<GpuResources> res;
    int device;
    GpuMemoryReservation codebooks; // [M*K][d]
    GpuMemoryReservation norms;     // [M*K]
    GpuMemoryReservation cc;        // [M*K][M*K]
};

GpuIcmEncoder::GpuIcmEncoder(
        int M_,
        int K_,
        int d_,
        std::vector<std::shared_ptr<GpuResources>> res,
        std::vector<int> devices)
        : M(M_), K(K_), d(d_) {
    FB_THROW_IF_NOT_FMT(M >= 1, "M = %d: GpuIcmEncoder needs M >= 1", M);
    FB_THROW_IF_NOT_FMT(K >= 1 && K <= kIcmMaxK, "K = %d: GpuIcmEncoder takes 1 <= K <= 1024", K);
    FB_THROW_IF_NOT_FMT(d >= 1, "d = %d: GpuIcmEncoder needs d >= 1", d);
    FB_THROW_IF_NOT_MSG(!res.empty() && res.size() == devices.size(), "one resources object per device is needed");
    int ndev = 0;
    CUDA_VERIFY(cudaGetDeviceCount(&ndev));
    for (size_t s = 0; s < res.size(); s++) {
        FB_THROW_IF_NOT_MSG(res[s] != nullptr, "null resources");
        FB_THROW_IF_NOT_FMT(devices[s] >= 0 && devices[s] < ndev, "device %d does not exist", devices[s]);
        for (size_t t = 0; t < s; t++) {
            // shards run on threads of their own; a resources object's allocator is not shared between threads
            FB_THROW_IF_NOT_MSG(res[t] != res[s], "each device needs a resources object of its own");
        }
        auto sh = std::make_unique<Shard>();
        sh->res = res[s];
        sh->device = devices[s];
        shards_.push_back(std::move(sh));
    }
}

GpuIcmEncoder::~GpuIcmEncoder() = default;

void GpuIcmEncoder::setBinaryTerm(const float* codebooks) {
    FB_THROW_IF_NOT_MSG(codebooks != nullptr, "null codebooks");
    const int64_t MK = (int64_t)M * K;
    haveBinaryTerm_ = false;
    for (auto& s : shards_) {
        DeviceScope scope(s->device);
        cudaStream_t stream = s->res->getDefaultStream(s->device);
        s->codebooks = s->res->device_alloc(s->device, sizeof(float) * MK * d, AllocType::Other);
        s->norms = s->res->device_alloc(s->device, sizeof(float) * MK, AllocType::Other);
        s->cc = s->res->device_alloc(s->device, sizeof(float) * MK * MK, AllocType::Other);
        CUDA_VERIFY(cudaMemcpyAsync(s->codebooks.data, codebooks, sizeof(float) * MK * d, cudaMemcpyDefault, stream));
        const float* cb = s->codebooks.as<float>();
        runL2Norms(cb, MK, d, s->norms.as<float>(), stream);
        runFlatPairwise(s->res.get(), s->device, cb, MK, cb, MK, d, METRIC_INNER_PRODUCT, 0.f, s->cc.as<float>(), MK, stream);
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
    haveBinaryTerm_ = true;
}

void GpuIcmEncoder::encode(
        int32_t* codes,
        const float* x,
        idx_t n,
        size_t ils_iters,
        size_t nperts,
        size_t icm_iters,
        const int32_t* perturbations,
        size_t pageBytes) const {
    FB_THROW_IF_NOT_MSG(haveBinaryTerm_, "setBinaryTerm must be called before encode");
    FB_THROW_IF_NOT_FMT(nperts <= (size_t)M, "nperts = %zu: must be <= M = %d", nperts, M);
    FB_THROW_IF_NOT_FMT(n >= 0, "n = %lld: must be >= 0", (long long)n);
    FB_THROW_IF_NOT_MSG(ils_iters < (size_t(1) << 31) && icm_iters < (size_t(1) << 31), "iteration count too large");
    FB_THROW_IF_NOT_MSG(pageBytes > 0, "page budget must be > 0");
    if (n == 0)
        return;
    FB_THROW_IF_NOT_MSG(codes != nullptr && x != nullptr, "null codes or x");
    FB_THROW_IF_NOT_MSG(perturbations != nullptr || ils_iters == 0 || nperts == 0, "null perturbations");

    // contiguous row ranges, the first n % nshards shards one row longer (faiss/gpu/GpuIcmEncoder.cu:96-111)
    const idx_t ns = (idx_t)shards_.size();
    auto range = [&](idx_t s, idx_t& i0, idx_t& ni) {
        const idx_t base = n / ns;
        i0 = s * base + std::min(s, n % ns);
        ni = base + (s < n % ns ? 1 : 0);
    };
    if (ns == 1) {
        encodeShard(*shards_[0], codes, x, n, 0, n, ils_iters, nperts, icm_iters, perturbations, pageBytes);
        return;
    }
    std::vector<std::exception_ptr> errs(ns);
    std::vector<std::thread> th;
    for (idx_t s = 0; s < ns; s++) {
        th.emplace_back([&, s] {
            try {
                idx_t i0, ni;
                range(s, i0, ni);
                encodeShard(*shards_[s], codes, x, n, i0, ni, ils_iters, nperts, icm_iters, perturbations, pageBytes);
            } catch (...) {
                errs[s] = std::current_exception();
            }
        });
    }
    for (auto& t : th)
        t.join();
    for (auto& e : errs)
        if (e)
            std::rethrow_exception(e);
}

void GpuIcmEncoder::encodeShard(
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
        size_t pageBytes) const {
    if (ni == 0)
        return;
    DeviceScope scope(s.device);
    GpuResources* res = s.res.get();
    cudaStream_t stream = res->getDefaultStream(s.device);
    const int64_t MK = (int64_t)M * K;
    const size_t drawRow = sizeof(int2) * nperts; // one row's draws of one ILS iteration
    const size_t perRow = sizeof(float) * (MK + d) + sizeof(int32_t) * M + drawRow * ils_iters;
    const idx_t pageRows = std::min<idx_t>(ni, std::max<idx_t>(1, (idx_t)(pageBytes / perRow)));

    GpuMemoryReservation ipBuf = res->temp(s.device, sizeof(float) * MK * pageRows);
    GpuMemoryReservation xBuf = res->temp(s.device, sizeof(float) * d * pageRows);
    GpuMemoryReservation codeBuf = res->temp(s.device, sizeof(int32_t) * M * pageRows);
    GpuMemoryReservation drawBuf = res->temp(s.device, std::max<size_t>(1, drawRow * ils_iters * pageRows));
    GpuMemoryReservation badBuf = res->temp(s.device, sizeof(int));

    for (idx_t r0 = i0; r0 < i0 + ni; r0 += pageRows) {
        InterruptCallback::check(); // between pages
        const idx_t rp = std::min(pageRows, i0 + ni - r0);
        CUDA_VERIFY(cudaMemsetAsync(badBuf.data, 0, sizeof(int), stream));
        CUDA_VERIFY(cudaMemcpyAsync(xBuf.data, x + r0 * d, sizeof(float) * d * rp, cudaMemcpyDefault, stream));
        CUDA_VERIFY(cudaMemcpyAsync(codeBuf.data, codes + r0 * M, sizeof(int32_t) * M * rp, cudaMemcpyDefault, stream));
        if (ils_iters > 0 && nperts > 0) {
            // [ils][n][nperts] -> [ils][rp][nperts]: one strided copy, ILS iteration by ILS iteration
            CUDA_VERIFY(cudaMemcpy2DAsync(
                    drawBuf.data, drawRow * rp, perturbations + 2 * r0 * nperts, drawRow * n, drawRow * rp, ils_iters,
                    cudaMemcpyDefault, stream));
        }
        KernelTiming::begin("icm_unary", stream);
        runFlatPairwise(res, s.device, xBuf.as<float>(), rp, s.codebooks.as<float>(), MK, d, METRIC_INNER_PRODUCT, 0.f,
                        ipBuf.as<float>(), MK, stream);
        KernelTiming::end("icm_unary", stream);
        KernelTiming::begin("icm_encode", stream);
        runIcmEncodeKernel(
                ipBuf.as<float>(), s.norms.as<float>(), s.cc.as<float>(), s.codebooks.as<float>(), xBuf.as<float>(),
                codeBuf.as<int32_t>(), reinterpret_cast<const int2*>(drawBuf.data), rp, M, K, d, (int)ils_iters,
                (int)nperts, (int)icm_iters, badBuf.as<int>(), stream);
        KernelTiming::end("icm_encode", stream);
        int bad = 0;
        CUDA_VERIFY(cudaMemcpyAsync(&bad, badBuf.data, sizeof(int), cudaMemcpyDeviceToHost, stream));
        CUDA_VERIFY(cudaStreamSynchronize(stream));
        if (bad & kBadCode)
            FB_THROW_FMT("an input code is outside [0, K = %d)", K);
        if (bad & kBadDraw)
            FB_THROW_FMT("a perturbation is outside m in [0, M = %d), k in [0, K = %d)", M, K);
        CUDA_VERIFY(cudaMemcpyAsync(codes + r0 * M, codeBuf.data, sizeof(int32_t) * M * rp, cudaMemcpyDefault, stream));
    }
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

} // namespace fb200
