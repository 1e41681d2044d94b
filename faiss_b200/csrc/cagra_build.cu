// faiss_b200 -- GpuIndexCagra graph build: IVF-PQ candidates, exact refine, and the graph optimisation.
//
// The build rule (restated in numpy by oracle/oracle_cagra_np.py; DESIGN "GpuIndexCagra"):
//   candidates  every row searches a GpuIndexIVFPQ over the dataset for C = ceil(refine_rate * K0) + 1 ids
//   refine      exact fp32 distances of the candidates, the row itself and -1 dropped, best K0 by (distance, id)
//               (IP: larger first) -> G0 [N][K0]; a row left with fewer than K0 is re-searched exactly
//   detours     c[u][j] = #{ i < j : some p < j has G0[G0[u][i]][p] = G0[u][j] }
//   prune       P[u] = the K entries of G0[u] with the smallest (c, j), in that order
//   reverse     R[w] = every u with w in P[u], ordered by (position of w in P[u], u)
//   merge       G[u] = P[u][0:K/2], then the entries of R[u] not present yet, then the rest of P[u], cut to K
#include "index.h"

#include <cub/cub.cuh>
#include <math_constants.h>

#include <algorithm>
#include <chrono>
#include <cmath>

namespace fb200 {

namespace {

constexpr uint32_t kNoEdge = 0xFFFFFFFFu;

__device__ __forceinline__ bool kv_less_u(float ka, uint32_t ia, float kb, uint32_t ib) {
    return ka < kb || (ka == kb && ia < ib);
}

// one CTA per row of the batch
__global__ void cagra_refine_kernel(
        const float* __restrict__ data, int64_t n, int d, bool ip, int64_t row0, const idx_t* __restrict__ cand,
        int nc, int ncPow2, int K0, uint32_t* __restrict__ G0, int* __restrict__ valid) {
    extern __shared__ __align__(16) unsigned char smem[];
    float* key = reinterpret_cast<float*>(smem);
    uint32_t* id = reinterpret_cast<uint32_t*>(key + ncPow2);
    float* q = reinterpret_cast<float*>(id + ncPow2);
    const int64_t bi = blockIdx.x;
    const int64_t u = row0 + bi;
    for (int j = threadIdx.x; j < d; j += blockDim.x)
        q[j] = data[u * d + j];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nWarps = blockDim.x >> 5;
    for (int c = warp; c < ncPow2; c += nWarps) {
        const idx_t v = c < nc ? cand[bi * nc + c] : -1;
        const bool ok = v >= 0 && v < n && v != u;
        float acc = 0.f;
        if (ok) {
            const float* y = data + v * d;
            for (int j = lane; j < d; j += 32) {
                if (ip) {
                    acc = fmaf(q[j], y[j], acc);
                } else {
                    const float t = q[j] - y[j];
                    acc = fmaf(t, t, acc);
                }
            }
            for (int o = 16; o > 0; o >>= 1)
                acc += __shfl_xor_sync(0xffffffffu, acc, o);
        }
        if (lane == 0) {
            key[c] = ok ? (ip ? -acc : acc) : CUDART_INF_F;
            id[c] = ok ? (uint32_t)v : kNoEdge;
        }
    }
    __syncthreads();
    for (int size = 2; size <= ncPow2; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < (ncPow2 >> 1); t += blockDim.x) {
                const int a = 2 * t - (t & (stride - 1)), b = a + stride;
                const bool up = (a & size) == 0;
                if (kv_less_u(key[b], id[b], key[a], id[a]) == up) {
                    const float tk = key[a];
                    key[a] = key[b];
                    key[b] = tk;
                    const uint32_t ti = id[a];
                    id[a] = id[b];
                    id[b] = ti;
                }
            }
            __syncthreads();
        }
    }
    for (int j = threadIdx.x; j < K0; j += blockDim.x)
        G0[u * K0 + j] = j < ncPow2 ? id[j] : kNoEdge;
    if (threadIdx.x == 0) {
        int cnt = 0;
        while (cnt < K0 && cnt < ncPow2 && id[cnt] != kNoEdge)
            cnt++;
        valid[bi] = cnt;
    }
}

// detour counts and the prune, one CTA per row u.  Shared memory: G0[u], an id -> rank hash of it, the detour bit
// matrix hit[j][i] (bit i of row j: a two-hop route to G0[u][j] through G0[u][i]) and the counts.
__global__ void cagra_prune_kernel(
        const uint32_t* __restrict__ G0, int64_t n, int K0, int K, int hashBits, uint32_t* __restrict__ P) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int W = (K0 + 31) >> 5;
    uint32_t* row = reinterpret_cast<uint32_t*>(smem);
    uint32_t* hkey = row + K0;
    uint32_t* hval = hkey + (1 << hashBits);
    uint32_t* hit = hval + (1 << hashBits);
    int* cnt = reinterpret_cast<int*>(hit + K0 * W);
    const int64_t u = blockIdx.x;
    const uint32_t hmask = (1u << hashBits) - 1;
    for (int i = threadIdx.x; i < (1 << hashBits); i += blockDim.x)
        hkey[i] = kNoEdge;
    for (int i = threadIdx.x; i < K0 * W; i += blockDim.x)
        hit[i] = 0;
    for (int j = threadIdx.x; j < K0; j += blockDim.x)
        row[j] = G0[u * K0 + j];
    __syncthreads();
    for (int j = threadIdx.x; j < K0; j += blockDim.x) {
        const uint32_t v = row[j];
        uint32_t s = (v * 0x9E3779B1u) >> (32 - hashBits);
        while (true) {
            const uint32_t prev = atomicCAS(hkey + s, kNoEdge, v);
            if (prev == kNoEdge) {
                hval[s] = (uint32_t)j;
                break;
            }
            s = (s + 1) & hmask;
        }
    }
    __syncthreads();
    // pairs (i, p): w = G0[G0[u][i]][p] with rank j in G0[u]; counted when i < j and p < j
    const int64_t pairs = (int64_t)(K0 - 1) * K0;
    for (int64_t t = threadIdx.x; t < pairs; t += blockDim.x) {
        const int i = (int)(t / K0), p = (int)(t - (int64_t)i * K0);
        const uint32_t v = row[i];
        if (p >= K0 - 1 || v >= (uint32_t)n)
            continue;
        const uint32_t w = __ldg(G0 + (int64_t)v * K0 + p);
        if (w == kNoEdge)
            continue;
        uint32_t s = (w * 0x9E3779B1u) >> (32 - hashBits);
        while (true) {
            const uint32_t h = hkey[s];
            if (h == kNoEdge)
                break;
            if (h == w) {
                const int j = (int)hval[s];
                if (j > i && j > p)
                    atomicOr(hit + j * W + (i >> 5), 1u << (i & 31));
                break;
            }
            s = (s + 1) & hmask;
        }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < K0; j += blockDim.x) {
        int c = 0;
        for (int w = 0; w < W; w++)
            c += __popc(hit[j * W + w]);
        cnt[j] = c;
    }
    __syncthreads();
    // stable order by count: rank of j = #{ j' : (c[j'], j') < (c[j], j) }
    for (int j = threadIdx.x; j < K0; j += blockDim.x) {
        const int cj = cnt[j];
        int r = 0;
        for (int jj = 0; jj < K0; jj++) {
            const int c = cnt[jj];
            r += (c < cj || (c == cj && jj < j)) ? 1 : 0;
        }
        if (r < K)
            P[u * K + r] = row[j];
    }
}

// reverse-edge list input: edge e = pos * n + u carries (key P[u][pos], value u), so a stable sort by key leaves every
// key's values in (pos, u) order
__global__ void cagra_reverse_edges_kernel(const uint32_t* __restrict__ P, int64_t n, int K, uint32_t* keys, uint32_t* vals) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * K)
        return;
    const int64_t pos = e / n, u = e - pos * n;
    keys[e] = P[u * K + pos];
    vals[e] = (uint32_t)u;
}

__device__ int64_t lower_bound_u32(const uint32_t* a, int64_t len, uint32_t v) {
    int64_t lo = 0, hi = len;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < v)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// G[u] from P[u] and R[u] (the sorted reverse edges), one CTA of >= K threads per row
__global__ void cagra_merge_kernel(
        const uint32_t* __restrict__ P, const uint32_t* __restrict__ rkeys, const uint32_t* __restrict__ rvals, int64_t nEdges,
        int K, uint32_t* __restrict__ G) {
    extern __shared__ __align__(16) unsigned char smem[];
    uint32_t* p = reinterpret_cast<uint32_t*>(smem);
    uint32_t* r = p + K;
    int* newR = reinterpret_cast<int*>(r + K);
    int* posR = newR + K;
    int* dupP = posR + K;
    __shared__ int64_t lo;
    __shared__ int nR, nTake;
    const int64_t u = blockIdx.x;
    const int half = K / 2;
    const int t = threadIdx.x;
    if (t == 0) {
        lo = lower_bound_u32(rkeys, nEdges, (uint32_t)u);
        const int64_t hi = lower_bound_u32(rkeys, nEdges, (uint32_t)u + 1);
        nR = (int)(hi - lo < K ? hi - lo : K);
    }
    if (t < K)
        p[t] = P[u * K + t];
    __syncthreads();
    if (t < nR) {
        const uint32_t v = rvals[lo + t];
        r[t] = v;
        int fresh = 1;
        for (int j = 0; j < half; j++)
            fresh &= p[j] != v;
        newR[t] = fresh;
    }
    __syncthreads();
    if (t == 0) {
        int c = 0;
        for (int i = 0; i < nR; i++) {
            posR[i] = newR[i] && c < K - half ? half + c : -1;
            c += newR[i] && c < K - half;
        }
        nTake = c;
    }
    __syncthreads();
    if (t < K && t >= half) {
        int dup = 0;
        for (int i = 0; i < nR; i++)
            dup |= posR[i] >= 0 && r[i] == p[t];
        dupP[t] = dup;
    }
    if (t < nR && posR[t] >= 0)
        G[u * K + posR[t]] = r[t];
    __syncthreads();
    if (t == 0) {
        int o = half + nTake;
        for (int j = half; j < K && o < K; j++)
            if (!dupP[j])
                G[u * K + o++] = p[j];
    }
    if (t < half)
        G[u * K + t] = p[t];
}

// bad[0] = 1 when some G0[u][j] >= n (a -1 read as uint32, or out of range), bad[1] = 1 when some G0[u][j] == u
__global__ void cagra_check_g0_kernel(const uint32_t* __restrict__ G0, int64_t n, int K0, int* bad) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * K0)
        return;
    const uint32_t v = G0[e];
    if (v >= (uint64_t)n)
        bad[0] = 1;
    else if (v == (uint64_t)(e / K0))
        bad[1] = 1;
}

double secondsSince(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

} // namespace

void runCagraRefine(
        const float* data, int64_t n, int d, MetricType metric, int64_t row0, int64_t nb, const idx_t* cand, int nc,
        int K0, uint32_t* G0, int* valid, cudaStream_t stream) {
    FB_THROW_IF_NOT(nc >= 1 && nc <= kMaxK);
    if (nb == 0)
        return;
    const int ncPow2 = next_pow2(nc);
    const size_t smem = 8 * (size_t)ncPow2 + sizeof(float) * d;
    FB_THROW_IF_NOT_MSG(smem <= 200 * 1024, "dimension too large for the CAGRA refine kernel");
    CUDA_VERIFY(cudaFuncSetAttribute(cagra_refine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cagra_refine_kernel<<<(unsigned)nb, 256, smem, stream>>>(
            data, n, d, metric == METRIC_INNER_PRODUCT, row0, cand, nc, ncPow2, K0, G0, valid);
    CUDA_CHECK_LAST();
}

void checkCagraG0(GpuResources* res, int device, const uint32_t* G0, int64_t n, int K0, cudaStream_t stream) {
    if (n == 0 || K0 <= 0)
        return;
    auto bad = res->device_alloc(device, 2 * sizeof(int), AllocType::Other);
    CUDA_VERIFY(cudaMemsetAsync(bad.data, 0, 2 * sizeof(int), stream));
    cagra_check_g0_kernel<<<(unsigned)ceil_div(n * K0, 256), 256, 0, stream>>>(G0, n, K0, bad.as<int>());
    CUDA_CHECK_LAST();
    int h[2] = {0, 0};
    CUDA_VERIFY(cudaMemcpyAsync(h, bad.data, sizeof(h), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    FB_THROW_IF_NOT_MSG(!h[0], "CAGRA optimize: a G0 entry is >= n (no edge, or out of range)");
    FB_THROW_IF_NOT_MSG(!h[1], "CAGRA optimize: a G0 row holds its own id");
}

void runCagraOptimize(GpuResources* res, int device, const uint32_t* G0, int64_t n, int K0, int K, uint32_t* G, cudaStream_t stream) {
    FB_THROW_IF_NOT_FMT(K >= 1 && K <= K0 && K0 <= 1024, "CAGRA optimize needs 1 <= graph_degree <= intermediate degree <= 1024 (%d, %d)", K, K0);
    FB_THROW_IF_NOT_MSG(n < (int64_t(1) << 31) - 1 && n * K < (int64_t(1) << 31), "CAGRA optimize: too many edges");
    if (n == 0)
        return;
    int hashBits = 1;
    while ((1 << hashBits) < 2 * K0)
        hashBits++;
    const int W = (K0 + 31) / 32;
    const size_t pruneSmem = sizeof(uint32_t) * ((size_t)K0 + 2 * (size_t(1) << hashBits) + (size_t)K0 * W + K0);
    CUDA_VERIFY(cudaFuncSetAttribute(cagra_prune_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pruneSmem));
    auto P = res->device_alloc(device, sizeof(uint32_t) * n * K, AllocType::Other);
    cagra_prune_kernel<<<(unsigned)n, 256, pruneSmem, stream>>>(G0, n, K0, K, hashBits, P.as<uint32_t>());
    CUDA_CHECK_LAST();

    const int64_t nEdges = n * K;
    auto keys = res->device_alloc(device, sizeof(uint32_t) * nEdges * 4, AllocType::Other);
    uint32_t* kIn = keys.as<uint32_t>();
    uint32_t* vIn = kIn + nEdges;
    uint32_t* kOut = vIn + nEdges;
    uint32_t* vOut = kOut + nEdges;
    cagra_reverse_edges_kernel<<<(unsigned)ceil_div(nEdges, 256), 256, 0, stream>>>(P.as<uint32_t>(), n, K, kIn, vIn);
    CUDA_CHECK_LAST();
    int endBit = 1;
    while ((int64_t(1) << endBit) < n)
        endBit++;
    size_t tmpBytes = 0;
    CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(nullptr, tmpBytes, kIn, kOut, vIn, vOut, (int)nEdges, 0, endBit, stream));
    auto tmp = res->device_alloc(device, std::max<size_t>(tmpBytes, 16), AllocType::Other);
    CUDA_VERIFY(cub::DeviceRadixSort::SortPairs(tmp.data, tmpBytes, kIn, kOut, vIn, vOut, (int)nEdges, 0, endBit, stream));

    const int threads = (int)round_up(std::max(K, 32), 32);
    const size_t mergeSmem = sizeof(uint32_t) * 5 * (size_t)K;
    cagra_merge_kernel<<<(unsigned)n, threads, mergeSmem, stream>>>(P.as<uint32_t>(), kOut, vOut, nEdges, K, G);
    CUDA_CHECK_LAST();
    CUDA_VERIFY(cudaStreamSynchronize(stream)); // the scratch buffers die here
}

void cagraBuildGraph(
        std::shared_ptr<GpuResources> res, int device, const float* xDev, idx_t n, int d, MetricType metric,
        const GpuIndexCagraConfig& cfg, int K0, int K, DeviceVector<uint32_t>& graph, double seconds[3]) {
    auto stream = res->getDefaultStream(device);
    const IVFPQBuildCagraConfig& bp = cfg.ivf_pq_params;
    const IVFPQSearchCagraConfig& sp = cfg.ivf_pq_search_params;
    const int nc = (int)std::ceil((double)cfg.refine_rate * K0) + 1;
    FB_THROW_IF_NOT_FMT(nc <= kMaxK, "refine_rate * intermediate_graph_degree gives %d candidates per row (max %d)", nc, kMaxK);
    auto G0 = res->device_alloc(device, sizeof(uint32_t) * n * K0, AllocType::Other);
    std::vector<int> hValid((size_t)n, 0);

    // (a) candidates from an IVF-PQ index over the dataset, (b) refined batch by batch
    auto t0 = std::chrono::steady_clock::now();
    const idx_t nTrain = std::max<idx_t>(1, std::min<idx_t>(n, (idx_t)((double)n * bp.kmeans_trainset_fraction)));
    std::unique_ptr<GpuIndexIVFPQ> ivfpq;
    if (nTrain >= (idx_t(1) << bp.pq_bits)) { // else the PQ cannot be trained: every row is searched exactly below
        const idx_t nlist = std::max<idx_t>(1, std::min<idx_t>((idx_t)bp.n_lists, nTrain / 39));
        int M = (int)bp.pq_dim;
        if (M == 0) {
            M = 1;
            for (int m = std::min(32, d / 2); m >= 1; m--)
                if (d % m == 0) {
                    M = m;
                    break;
                }
        }
        GpuIndexIVFPQConfig pc;
        pc.device = device;
        pc.interleavedLayout = bp.pq_bits != 8;
        ivfpq.reset(new GpuIndexIVFPQ(res, d, nlist, M, bp.pq_bits, metric, pc));
        ivfpq->cp.niter = (int)bp.kmeans_n_iters;
        GpuMemoryReservation sub;
        idx_t ns = n;
        const float* xs = subsampleRowsDevice(res.get(), device, ns, d, nTrain, 1234, xDev, sub, stream);
        ivfpq->train(ns, xs);
        ivfpq->add(n, xDev);
        ivfpq->nprobe = std::min<size_t>(std::max<uint32_t>(sp.n_probes, 1), (size_t)nlist);
    }
    seconds[0] = 0;
    double tRefine = 0;
    const idx_t batch = std::max<idx_t>(1, (idx_t)sp.max_internal_batch_size);
    auto valid = res->device_alloc(device, sizeof(int) * std::min(batch, n), AllocType::Other);
    if (ivfpq) {
        auto cand = res->device_alloc(device, sizeof(idx_t) * std::min(batch, n) * nc, AllocType::Other);
        auto dis = res->device_alloc(device, sizeof(float) * std::min(batch, n) * nc, AllocType::Other);
        seconds[0] = secondsSince(t0);
        for (idx_t b0 = 0; b0 < n; b0 += batch) {
            InterruptCallback::check();
            const idx_t nb = std::min(batch, n - b0);
            auto ts = std::chrono::steady_clock::now();
            ivfpq->search(nb, xDev + (size_t)b0 * d, nc, dis.as<float>(), cand.as<idx_t>());
            CUDA_VERIFY(cudaStreamSynchronize(stream));
            seconds[0] += secondsSince(ts);
            ts = std::chrono::steady_clock::now();
            runCagraRefine(xDev, n, d, metric, b0, nb, cand.as<idx_t>(), nc, K0, G0.as<uint32_t>(), valid.as<int>(), stream);
            CUDA_VERIFY(cudaMemcpyAsync(hValid.data() + b0, valid.data, sizeof(int) * nb, cudaMemcpyDeviceToHost, stream));
            CUDA_VERIFY(cudaStreamSynchronize(stream));
            tRefine += secondsSince(ts);
        }
        ivfpq.reset();
    } else {
        seconds[0] = secondsSince(t0);
    }

    // rows left with fewer than K0 candidates: the exact Flat kernel, K0 + 1 results (the row itself among them)
    auto ts = std::chrono::steady_clock::now();
    std::vector<idx_t> short_;
    for (idx_t i = 0; i < n; i++)
        if (hValid[i] < K0)
            short_.push_back(i);
    const idx_t exBatch = std::max<idx_t>(1, std::min<idx_t>(batch, (idx_t(1) << 28) / ((idx_t)(K0 + 1) * 12)));
    for (size_t s0 = 0; s0 < short_.size(); s0 += exBatch) {
        const idx_t m = std::min<idx_t>(exBatch, (idx_t)short_.size() - s0);
        DeviceView<idx_t> rows(res.get(), device, short_.data() + s0, m, stream);
        auto q = res->temp(device, sizeof(float) * m * d);
        runGatherRows(xDev, rows.ptr, m, d, q.as<float>(), stream);
        auto eD = res->temp(device, sizeof(float) * m * (K0 + 1));
        auto eI = res->temp(device, sizeof(idx_t) * m * (K0 + 1));
        runFlatExact(res.get(), device, q.as<float>(), m, xDev, n, d, K0 + 1, metric, 0, eD.as<float>(), eI.as<idx_t>(), stream);
        std::vector<idx_t> hI((size_t)m * (K0 + 1));
        CUDA_VERIFY(cudaMemcpyAsync(hI.data(), eI.data, hI.size() * sizeof(idx_t), cudaMemcpyDeviceToHost, stream));
        CUDA_VERIFY(cudaStreamSynchronize(stream));
        std::vector<uint32_t> rowsOut((size_t)m * K0);
        for (idx_t r = 0; r < m; r++) {
            const idx_t u = short_[s0 + r];
            int o = 0;
            for (int j = 0; j <= K0 && o < K0; j++) {
                const idx_t v = hI[(size_t)r * (K0 + 1) + j];
                if (v >= 0 && v != u)
                    rowsOut[(size_t)r * K0 + o++] = (uint32_t)v;
            }
            FB_THROW_IF_NOT_MSG(o == K0, "exact re-search returned too few neighbours");
        }
        for (idx_t r = 0; r < m; r++)
            CUDA_VERIFY(cudaMemcpyAsync(
                    G0.as<uint32_t>() + (size_t)short_[s0 + r] * K0, rowsOut.data() + (size_t)r * K0, sizeof(uint32_t) * K0,
                    cudaMemcpyHostToDevice, stream));
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
    seconds[1] = tRefine + secondsSince(ts);

    // (c) optimise
    ts = std::chrono::steady_clock::now();
    graph.clear();
    graph.resize((size_t)n * K, stream);
    runCagraOptimize(res.get(), device, G0.as<uint32_t>(), n, K0, K, graph.data(), stream);
    seconds[2] = secondsSince(ts);
}

} // namespace fb200
