// faiss_b200 -- k-means centroid update on the device.
//
// The reference runs Lloyd's update on the CPU every iteration (compute_centroids,
// faiss/impl/ClusteringHelpers.cpp:101-172: every OpenMP thread scans all n assignments) after
// re-uploading the training set for the GPU assignment step.  Here the training set stays in HBM;
// assignment is the Flat k=1 kernel and the update sorts the points by assignment, then adds each
// centroid's points in index order, so the sums are bit-reproducible run to run.
#include <cub/cub.cuh>

#include "kernels.h"
#include "select.cuh"

namespace fb200 {

__global__ void kmeans_accum_smem_kernel(
        const float* __restrict__ x,
        const idx_t* __restrict__ assign,
        int64_t n,
        int d,
        int k,
        int64_t pointsPerBlock,
        float* __restrict__ sums,
        float* __restrict__ counts) {
    extern __shared__ float sm[]; // [k*d] sums + [k] counts
    float* ssum = sm;
    float* scnt = sm + (size_t)k * d;
    for (int i = threadIdx.x; i < k * d + k; i += blockDim.x)
        sm[i] = 0.f;
    __syncthreads();
    const int64_t p0 = (int64_t)blockIdx.x * pointsPerBlock;
    const int64_t p1 = min(n, p0 + pointsPerBlock);
    // flat element loop: element e of the slice = (point, dim)
    for (int64_t e = p0 * d + threadIdx.x; e < p1 * d; e += blockDim.x) {
        int64_t pt = e / d;
        int j = (int)(e - pt * d);
        idx_t c = assign[pt];
        if (c >= 0 && c < k) {
            atomicAdd(&ssum[c * d + j], x[e]);
            if (j == 0)
                atomicAdd(&scnt[c], 1.f);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < k * d; i += blockDim.x) {
        float v = ssum[i];
        if (v != 0.f)
            atomicAdd(&sums[i], v);
    }
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        float v = scnt[i];
        if (v != 0.f)
            atomicAdd(&counts[i], v);
    }
}

__global__ void kmeans_accum_global_kernel(
        const float* __restrict__ x,
        const idx_t* __restrict__ assign,
        int64_t n,
        int d,
        int64_t k,
        float* __restrict__ sums,
        float* __restrict__ counts) {
    const int64_t pt = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pt >= n)
        return;
    const idx_t c = assign[pt];
    if (c < 0 || c >= k)
        return;
    const float* xp = x + pt * d;
    float* sp = sums + c * d;
    for (int j = lane_id(); j < d; j += 32)
        atomicAdd(&sp[j], xp[j]);
    if (lane_id() == 0)
        atomicAdd(&counts[c], 1.f);
}

// ---- deterministic update: sort the points by assignment, then one warp per centroid adds its points in
// index order (no atomics: the sums are bit-reproducible run to run, like the reference's CPU
// compute_centroids, faiss/impl/ClusteringHelpers.cpp:101-172; SURVEY 7 step 5)
__global__ void kmeans_keys_kernel(const idx_t* __restrict__ assign, int64_t n, int64_t k, unsigned* __restrict__ keys, unsigned* __restrict__ vals) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const idx_t a = assign[i];
    keys[i] = (a >= 0 && a < k) ? (unsigned)a : (unsigned)k; // unassigned points sort last
    vals[i] = (unsigned)i;
}

__global__ void kmeans_segment_sum_kernel(
        const float* __restrict__ x,
        const unsigned* __restrict__ keys, // sorted
        const unsigned* __restrict__ rows, // point index, stable order inside a key
        int64_t n,
        int d,
        int64_t k,
        float* __restrict__ sums,
        float* __restrict__ counts) {
    const int64_t c = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (c >= k)
        return;
    // [lo, hi) = the run of key c (binary searches, warp-uniform)
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < (unsigned)c)
            lo = mid + 1;
        else
            hi = mid;
    }
    int64_t e = lo, hi2 = n;
    while (e < hi2) {
        const int64_t mid = (e + hi2) >> 1;
        if (keys[mid] <= (unsigned)c)
            e = mid + 1;
        else
            hi2 = mid;
    }
    const int lane = lane_id();
    for (int j0 = 0; j0 < d; j0 += 128) { // 4 dimensions per lane and pass
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        const int j = j0 + lane;
        int64_t i = lo;
        // four points per step: the row loads are independent, the adds keep the index order
        for (; i + 4 <= e; i += 4) {
            const float* p0 = x + (int64_t)rows[i] * d;
            const float* p1 = x + (int64_t)rows[i + 1] * d;
            const float* p2 = x + (int64_t)rows[i + 2] * d;
            const float* p3 = x + (int64_t)rows[i + 3] * d;
            float v[4][4];
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const int jj = j + 32 * t;
                v[0][t] = jj < d ? p0[jj] : 0.f;
                v[1][t] = jj < d ? p1[jj] : 0.f;
                v[2][t] = jj < d ? p2[jj] : 0.f;
                v[3][t] = jj < d ? p3[jj] : 0.f;
            }
#pragma unroll
            for (int pnt = 0; pnt < 4; pnt++) {
                a0 += v[pnt][0];
                a1 += v[pnt][1];
                a2 += v[pnt][2];
                a3 += v[pnt][3];
            }
        }
        for (; i < e; i++) {
            const float* xp = x + (int64_t)rows[i] * d;
            if (j < d)
                a0 += xp[j];
            if (j + 32 < d)
                a1 += xp[j + 32];
            if (j + 64 < d)
                a2 += xp[j + 64];
            if (j + 96 < d)
                a3 += xp[j + 96];
        }
        float* sp = sums + c * d;
        if (j < d)
            sp[j] += a0;
        if (j + 32 < d)
            sp[j + 32] += a1;
        if (j + 64 < d)
            sp[j + 64] += a2;
        if (j + 96 < d)
            sp[j + 96] += a3;
    }
    if (lane == 0)
        counts[c] += (float)(e - lo);
}

static void runKmeansAccumulateSorted(
        const float* x, const idx_t* assign, int64_t n, int d, int64_t k, float* sums, float* counts, cudaStream_t stream) {
    FB_THROW_IF_NOT_MSG(n < (int64_t(1) << 32) - 1 && k < (int64_t(1) << 32) - 1, "k-means update: too many points / centroids");
    unsigned *keysIn = nullptr, *keysOut = nullptr, *valsIn = nullptr, *valsOut = nullptr;
    void* tmp = nullptr;
    CUDA_VERIFY(cudaMallocAsync(&keysIn, sizeof(unsigned) * n * 4, stream));
    keysOut = keysIn + n;
    valsIn = keysOut + n;
    valsOut = valsIn + n;
    kmeans_keys_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(assign, n, k, keysIn, valsIn);
    CUDA_CHECK_LAST();
    int endBit = 1;
    while ((int64_t(1) << endBit) <= k)
        endBit++;
    size_t tmpBytes = 0;
    CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(nullptr, tmpBytes, keysIn, keysOut, valsIn, valsOut, (int)n, 0, endBit, stream));
    CUDA_VERIFY(cudaMallocAsync(&tmp, tmpBytes, stream));
    CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(tmp, tmpBytes, keysIn, keysOut, valsIn, valsOut, (int)n, 0, endBit, stream));
    const int warps = 8;
    kmeans_segment_sum_kernel<<<(unsigned)ceil_div(k, warps), warps * 32, 0, stream>>>(x, keysOut, valsOut, n, d, k, sums, counts);
    CUDA_CHECK_LAST();
    CUDA_VERIFY(cudaFreeAsync(tmp, stream));
    CUDA_VERIFY(cudaFreeAsync(keysIn, stream));
}

void runKmeansAccumulate(
        const float* x,
        const idx_t* assign,
        int64_t n,
        int d,
        int64_t k,
        float* sums,
        float* counts,
        cudaStream_t stream) {
    if (n == 0)
        return;
    if (n < (int64_t(1) << 31)) {
        runKmeansAccumulateSorted(x, assign, n, d, k, sums, counts, stream);
        return;
    }
    // n >= 2^31 exceeds the radix sort's int item count: atomic accumulation, not order-deterministic.
    // Codebooks whose k*d floats fit in shared memory (e.g. the 256 x dsub PQ codebooks) are accumulated
    // per block with shared atomics and flushed once; larger ones take one warp per point with global RED.
    size_t smem = sizeof(float) * ((size_t)k * d + k);
    if (smem <= 64 * 1024) {
        int64_t ppb = std::max<int64_t>(256, ceil_div(n, 132 * 4));
        CUDA_VERIFY(cudaFuncSetAttribute(
                kmeans_accum_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kmeans_accum_smem_kernel<<<(unsigned)ceil_div(n, ppb), 256, smem, stream>>>(
                x, assign, n, d, (int)k, ppb, sums, counts);
    } else {
        int warps = 8;
        kmeans_accum_global_kernel<<<(unsigned)ceil_div(n, warps), warps * 32, 0, stream>>>(
                x, assign, n, d, k, sums, counts);
    }
    CUDA_CHECK_LAST();
}

__global__ void kmeans_finalize_kernel(
        const float* __restrict__ sums,
        const float* __restrict__ counts,
        int64_t k,
        int d,
        float* __restrict__ centroids) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k * d)
        return;
    float c = counts[i / d];
    if (c > 0.f) {
        // faiss/impl/ClusteringHelpers.cpp:160-170: multiply by 1/count
        float norm = 1.f / c;
        centroids[i] = sums[i] * norm;
    }
}

void runKmeansFinalize(
        const float* sums,
        const float* counts,
        int64_t k,
        int d,
        float* centroids,
        cudaStream_t stream) {
    kmeans_finalize_kernel<<<(unsigned)ceil_div(k * d, 256), 256, 0, stream>>>(sums, counts, k, d, centroids);
    CUDA_CHECK_LAST();
}

// post_process_centroids (faiss/Clustering.cpp:35-45): spherical -> fvec_renorm_L2 (rows with non-zero norm
// scaled by 1/sqrtf(||row||^2), faiss/utils/distances.cpp:238-251); int_centroids -> roundf.  One warp per row.
__global__ void kmeans_post_process_kernel(float* __restrict__ c, int64_t k, int d, int spherical, int intCentroids) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= k)
        return;
    float* r = c + row * d;
    if (spherical) {
        float acc = 0.f;
        for (int j = lane_id(); j < d; j += 32)
            acc = fmaf(r[j], r[j], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            acc += __shfl_xor_sync(kFullMask, acc, o);
        if (acc > 0.f) {
            const float inv = 1.0f / sqrtf(acc);
            for (int j = lane_id(); j < d; j += 32)
                r[j] *= inv;
        }
    }
    if (intCentroids) {
        __syncwarp();
        for (int j = lane_id(); j < d; j += 32)
            r[j] = roundf(r[j]);
    }
}

void runKmeansPostProcess(float* centroids, int64_t k, int d, bool spherical, bool intCentroids, cudaStream_t stream) {
    if (k == 0 || (!spherical && !intCentroids))
        return;
    const int warps = 8;
    kmeans_post_process_kernel<<<(unsigned)ceil_div(k, warps), warps * 32, 0, stream>>>(
            centroids, k, d, spherical ? 1 : 0, intCentroids ? 1 : 0);
    CUDA_CHECK_LAST();
}

} // namespace fb200
