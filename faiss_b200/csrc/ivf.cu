// faiss_b200 -- IVF kernels: PQ encoding, device-side list append bookkeeping, IVF-Flat scan,
// IVF-PQ scan (LUT in shared memory + code walk + running top-k).
//
// Reference roles (faiss/gpu/impl/): IVFAppend.cu:29-620, IVFBase.cu:693-905 (host bookkeeping,
// here on the device), IVFInterleaved.cuh:39-224 / IVFFlatScan.cu (IVF-Flat scan),
// PQCodeDistances-inl.cuh:34-285 + PQScanMultiPassNoPrecomputed-inl.cuh:174-270 +
// IVFUtilsSelect1/2.cu (IVF-PQ: LUT to HBM, distances to HBM, two select passes).  Here the LUT
// and the distances never leave the SM.
//
// Storage layout ("arena"): all inverted lists live in one allocation; list l occupies elements
// [listStart[l], listStart[l] + listLen[l]) with capacity slack behind it.  Codes are stored
// vector-major ([len][codeSize] bytes), which is exactly the CPU ArrayInvertedLists byte layout
// (faiss/invlists/InvertedLists.h) -- copyFrom/copyTo are plain memcpys.
#include <cub/cub.cuh>

#include <cfloat>

#include "ivf_scan.cuh"
#include "kernels.h"
#include "select.cuh"

namespace fb200 {

// ------------------------------------------------------------------------------------------
// PQ encode
// ------------------------------------------------------------------------------------------
template <int DSUB>
__global__ void pq_encode_kernel(
        const float* __restrict__ resid,
        int64_t n,
        int d,
        int M,
        int ksub,
        int dsubRt,
        const float* __restrict__ pq,
        uint8_t* __restrict__ codes,
        bool stageInSmem) {
    extern __shared__ float centSmem[]; // [ksub][dsub] when staged
    const int dsub = DSUB > 0 ? DSUB : dsubRt;
    const int m = blockIdx.y;
    const float* src = pq + (size_t)m * ksub * dsub;
    const float* cent = src; // a codebook larger than shared memory (ksub * dsub * 4 > 227 KiB) is read from L1/L2
    if (stageInSmem) { // block-uniform
        for (int i = threadIdx.x; i < ksub * dsub; i += blockDim.x)
            centSmem[i] = src[i];
        __syncthreads();
        cent = centSmem;
    }
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const float* rp = resid + i * d + (size_t)m * dsub;
    float best = CUDART_INF_F;
    int bestc = 0;
    if (DSUB > 0) {
        float r[DSUB > 0 ? DSUB : 1];
#pragma unroll
        for (int j = 0; j < DSUB; j++)
            r[j] = rp[j];
        for (int c = 0; c < ksub; c++) {
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < DSUB; j++) {
                float df = r[j] - cent[c * DSUB + j];
                acc = fmaf(df, df, acc);
            }
            if (acc < best) { // first minimum wins (ProductQuantizer.cpp compute_code)
                best = acc;
                bestc = c;
            }
        }
    } else {
        for (int c = 0; c < ksub; c++) {
            float acc = 0.f;
            for (int j = 0; j < dsub; j++) {
                float df = rp[j] - cent[c * dsub + j];
                acc = fmaf(df, df, acc);
            }
            if (acc < best) {
                best = acc;
                bestc = c;
            }
        }
    }
    codes[i * M + m] = (uint8_t)bestc;
}

void runPQEncode(
        const float* resid,
        int64_t n,
        int d,
        int M,
        int ksub,
        const float* pq,
        uint8_t* codes,
        cudaStream_t stream) {
    if (n == 0)
        return;
    FB_THROW_IF_NOT(ksub <= 256 && d % M == 0);
    const int dsub = d / M;
    // the sub-quantiser's codebook is staged in shared memory when it fits the per-block opt-in limit; with
    // ksub = 256 that holds up to dsub = 227, and larger sub-vectors (e.g. d = 1024, M = 4) read it from global
    int device = 0, smemOptin = 0;
    CUDA_VERIFY(cudaGetDevice(&device));
    CUDA_VERIFY(cudaDeviceGetAttribute(&smemOptin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    const bool stage = sizeof(float) * ksub * dsub <= (size_t)smemOptin;
    const size_t smem = stage ? sizeof(float) * ksub * dsub : 0;
    dim3 grid((unsigned)ceil_div(n, 128), (unsigned)M);
#define PQENC(DS)                                                                                      \
    do {                                                                                               \
        CUDA_VERIFY(cudaFuncSetAttribute(                                                              \
                pq_encode_kernel<DS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));        \
        pq_encode_kernel<DS><<<grid, 128, smem, stream>>>(resid, n, d, M, ksub, dsub, pq, codes, stage); \
    } while (0)
    switch (dsub) {
        case 1:
            PQENC(1);
            break;
        case 2:
            PQENC(2);
            break;
        case 3:
            PQENC(3);
            break;
        case 4:
            PQENC(4);
            break;
        case 6:
            PQENC(6);
            break;
        case 8:
            PQENC(8);
            break;
        case 12:
            PQENC(12);
            break;
        case 16:
            PQENC(16);
            break;
        case 32:
            PQENC(32);
            break;
        default:
            PQENC(0);
            break;
    }
#undef PQENC
    CUDA_CHECK_LAST();
}

// PQEncoderGeneric (faiss/impl/ProductQuantizer-inl.h): the M codes of a vector, nbits each, LSB-first in a
// bitstring of ceil(M * nbits / 8) bytes.  One thread per output byte, so no byte is written twice.
__global__ void pq_pack_kernel(const uint8_t* __restrict__ codes, int64_t n, int M, int nbits, int codeSize, uint8_t* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * codeSize)
        return;
    const int64_t i = e / codeSize;
    const int b = (int)(e - i * codeSize);
    const uint8_t* c = codes + i * M;
    unsigned acc = 0;
    for (int m = (b * 8) / nbits; m < M && m * nbits < (b + 1) * 8; m++) {
        const int shift = m * nbits - b * 8; // bit position of code m relative to byte b (negative: starts earlier)
        acc |= shift >= 0 ? (unsigned)c[m] << shift : (unsigned)c[m] >> -shift;
    }
    out[e] = (uint8_t)acc;
}

void runPQPack(const uint8_t* codes, int64_t n, int M, int nbits, uint8_t* packed, cudaStream_t stream) {
    if (n == 0)
        return;
    FB_THROW_IF_NOT(nbits >= 1 && nbits <= 8);
    const int codeSize = (M * nbits + 7) / 8;
    pq_pack_kernel<<<(unsigned)ceil_div(n * codeSize, (int64_t)256), 256, 0, stream>>>(codes, n, M, nbits, codeSize, packed);
    CUDA_CHECK_LAST();
}

// ------------------------------------------------------------------------------------------
// append bookkeeping
// ------------------------------------------------------------------------------------------
__global__ void ivf_count_kernel(const idx_t* __restrict__ assign, int64_t n, int64_t nlist, int* counts) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        idx_t a = assign[i];
        if (a >= 0 && a < nlist)
            atomicAdd(&counts[a], 1);
    }
}

void runIvfCountAssign(const idx_t* assign, int64_t n, int64_t nlist, int* counts, cudaStream_t stream) {
    if (n == 0)
        return;
    ivf_count_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(assign, n, nlist, counts);
    CUDA_CHECK_LAST();
}

__global__ void ivf_keys_kernel(const idx_t* __restrict__ assign, int64_t n, int64_t nlist, int* keys, int* vals) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        idx_t a = assign[i];
        keys[i] = (a >= 0 && a < nlist) ? (int)a : (int)nlist;
        vals[i] = (int)i;
    }
}

// after the stable sort: position p holds vector vals[p] of list keys[p]; rank within its list is
// p - (first position of that list) ; first positions via a boundary scan
__global__ void ivf_offsets_kernel(
        const int* __restrict__ keysSorted,
        const int* __restrict__ valsSorted,
        int64_t n,
        int64_t nlist,
        const int* __restrict__ batchStart, // [nlist+1] exclusive scan of the batch histogram
        const int* __restrict__ listLenBefore,
        int* __restrict__ offsets) {
    int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) {
        int l = keysSorted[p];
        int v = valsSorted[p];
        offsets[v] = (l < nlist) ? listLenBefore[l] + (int)(p - batchStart[l]) : -1;
    }
}

void runIvfAppendOffsets(
        const idx_t* assign,
        int64_t n,
        int64_t nlist,
        const int* listLenBefore,
        int* offsets,
        int* scratch,
        cudaStream_t stream) {
    // `scratch` is unused by this implementation (kept for ABI stability); temp storage is
    // allocated stream-ordered.
    (void)scratch;
    if (n == 0)
        return;
    FB_THROW_IF_NOT(n < (int64_t(1) << 31) && nlist < (int64_t(1) << 31) - 1);
    int *keys, *vals, *keys2, *vals2, *hist, *start;
    CUDA_VERIFY(cudaMallocAsync(&keys, sizeof(int) * n * 4, stream));
    vals = keys + n;
    keys2 = vals + n;
    vals2 = keys2 + n;
    CUDA_VERIFY(cudaMallocAsync(&hist, sizeof(int) * (nlist + 2) * 2, stream));
    start = hist + nlist + 2;
    CUDA_VERIFY(cudaMemsetAsync(hist, 0, sizeof(int) * (nlist + 2) * 2, stream));
    ivf_keys_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(assign, n, nlist, keys, vals);
    CUDA_CHECK_LAST();
    ivf_count_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(assign, n, nlist, hist);
    CUDA_CHECK_LAST();
    int endBit = 1;
    while ((int64_t(1) << endBit) <= nlist)
        endBit++;
    size_t tb1 = 0, tb2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb1, keys, keys2, vals, vals2, (int)n, 0, endBit, stream);
    cub::DeviceScan::ExclusiveSum(nullptr, tb2, hist, start, (int)(nlist + 1), stream);
    void* tmp;
    CUDA_VERIFY(cudaMallocAsync(&tmp, std::max(tb1, tb2), stream));
    cub::DeviceRadixSort::SortPairs(tmp, tb1, keys, keys2, vals, vals2, (int)n, 0, endBit, stream);
    cub::DeviceScan::ExclusiveSum(tmp, tb2, hist, start, (int)(nlist + 1), stream);
    ivf_offsets_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(
            keys2, vals2, n, nlist, start, listLenBefore, offsets);
    CUDA_CHECK_LAST();
    CUDA_VERIFY(cudaFreeAsync(tmp, stream));
    CUDA_VERIFY(cudaFreeAsync(hist, stream));
    CUDA_VERIFY(cudaFreeAsync(keys, stream));
}

__global__ void ivf_scatter_kernel(
        const uint8_t* __restrict__ rows,
        const idx_t* __restrict__ ids,
        const idx_t* __restrict__ assign,
        const int* __restrict__ offsets,
        int64_t n,
        int codeSize,
        const int64_t* __restrict__ listStart,
        uint8_t* __restrict__ arenaCodes,
        idx_t* __restrict__ arenaIds) {
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n)
        return;
    const int off = offsets[i];
    if (off < 0)
        return;
    const int64_t pos = listStart[assign[i]] + off;
    const uint8_t* src = rows + i * codeSize;
    uint8_t* dst = arenaCodes + pos * codeSize;
    if ((codeSize & 15) == 0) {
        for (int j = lane_id(); j < (codeSize >> 4); j += 32)
            reinterpret_cast<uint4*>(dst)[j] = reinterpret_cast<const uint4*>(src)[j];
    } else if ((codeSize & 3) == 0) {
        for (int j = lane_id(); j < (codeSize >> 2); j += 32)
            reinterpret_cast<uint32_t*>(dst)[j] = reinterpret_cast<const uint32_t*>(src)[j];
    } else {
        for (int j = lane_id(); j < codeSize; j += 32)
            dst[j] = src[j];
    }
    if (lane_id() == 0)
        arenaIds[pos] = ids[i];
}

void runIvfScatter(
        const uint8_t* rows,
        const idx_t* ids,
        const idx_t* assign,
        const int* offsets,
        int64_t n,
        int codeSize,
        const int64_t* listStart,
        uint8_t* arenaCodes,
        idx_t* arenaIds,
        cudaStream_t stream) {
    if (n == 0)
        return;
    int warps = 8;
    ivf_scatter_kernel<<<(unsigned)ceil_div(n, warps), warps * 32, 0, stream>>>(
            rows, ids, assign, offsets, n, codeSize, listStart, arenaCodes, arenaIds);
    CUDA_CHECK_LAST();
}

// ------------------------------------------------------------------------------------------
// IVF-Flat scan: block per (query, chunk of its probes).  The per-warp top-k lists and thresholds live
// across the probes of the chunk (list ids = arena positions), so threshold passes grow with
// log(vectors per CTA) instead of with the number of (query, probe) pairs.
// ------------------------------------------------------------------------------------------
template <bool IS_L2, typename IdT, bool MASKED>
__global__ void __launch_bounds__(kScanWarps * 32) ivfflat_scan_kernel(
        const float* __restrict__ Q,
        int d,
        const idx_t* __restrict__ probes,
        int nprobe,
        int probesPerCta,
        const int64_t* __restrict__ listStart,
        const int* __restrict__ listLen,
        const float* __restrict__ arenaVecs,
        const idx_t* __restrict__ arenaIds,
        int k,
        int LIST,
        float* __restrict__ partD, // [nq, chunks, k] keys
        idx_t* __restrict__ partI,
        const uint32_t* __restrict__ slotMask) { // MASKED: the selector's arena mask
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int q = blockIdx.y, chunk = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = lane_id();
    float* qs = reinterpret_cast<float*>(smem_raw); // [d]
    unsigned char* lists = smem_raw + round_up(sizeof(float) * d, 16);
    const size_t perWarp = SmemTopK<IdT>::bytes(LIST, kScanBuf);
    float* oD = partD + ((int64_t)q * gridDim.x + chunk) * k;
    idx_t* oI = partI + ((int64_t)q * gridDim.x + chunk) * k;

    for (int i = threadIdx.x; i < d; i += blockDim.x)
        qs[i] = Q[(int64_t)q * d + i];
    WarpTopK<IdT> w;
    unsigned char* mine = lists + perWarp * warp;
    w.init(reinterpret_cast<float*>(mine), reinterpret_cast<IdT*>(mine + sizeof(float) * (LIST + kScanBuf)), LIST, kScanBuf, k);
    __syncthreads();
    const int pBegin = chunk * probesPerCta, pEnd = min(nprobe, pBegin + probesPerCta);

    if ((d & 127) == 0 && d <= 512) {
        // Fast path (d multiple of 128): lane t owns dims [128c + 4t, +4) for c < d/128, kept in registers.
        // A group of 32 vectors = 32 x d/128 coalesced 128-bit loads per lane, issued 8 vectors at a time
        // (memory-level parallelism); the 32 per-lane partial sums are reduced with one transposing
        // butterfly (31 shuffles per 32 vectors instead of 160).
        const int nch = d >> 7;
        float4 qv[4];
#pragma unroll
        for (int c = 0; c < 4; c++)
            qv[c] = c < nch ? *reinterpret_cast<const float4*>(qs + c * 128 + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        for (int p = pBegin; p < pEnd; p++) {
            const idx_t l = probes[(int64_t)q * nprobe + p];
            if (l < 0) // NaN query / missing probe (PQScanMultiPassNoPrecomputed-inl.cuh:199-202)
                continue;
            const int len = listLen[l];
            const int64_t ls = listStart[l];
            const float* base = arenaVecs + ls * d;
            for (int v0 = warp * 32; v0 < len; v0 += kScanWarps * 32) {
                float vals[32];
#pragma unroll
                for (int b8 = 0; b8 < 4; b8++) {
                    float4 y[8];
#pragma unroll
                    for (int c = 0; c < 4; c++) {
                        if (c < nch) {
#pragma unroll
                            for (int j = 0; j < 8; j++) {
                                const int v = min(v0 + b8 * 8 + j, len - 1); // clamped tail, masked at add()
                                y[j] = __ldg(reinterpret_cast<const float4*>(base + (int64_t)v * d + c * 128) + lane);
                            }
#pragma unroll
                            for (int j = 0; j < 8; j++) {
                                float acc = c == 0 ? 0.f : vals[b8 * 8 + j];
                                if (IS_L2) {
                                    float d0 = qv[c].x - y[j].x, d1 = qv[c].y - y[j].y, d2 = qv[c].z - y[j].z, d3 = qv[c].w - y[j].w;
                                    acc = fmaf(d0, d0, acc);
                                    acc = fmaf(d1, d1, acc);
                                    acc = fmaf(d2, d2, acc);
                                    acc = fmaf(d3, d3, acc);
                                } else {
                                    acc = fmaf(qv[c].x, y[j].x, acc);
                                    acc = fmaf(qv[c].y, y[j].y, acc);
                                    acc = fmaf(qv[c].z, y[j].z, acc);
                                    acc = fmaf(qv[c].w, y[j].w, acc);
                                }
                                vals[b8 * 8 + j] = acc;
                            }
                        }
                    }
                }
                // transposing butterfly: afterwards lane t holds the full sum of vector v0 + t
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
                w.add(v0 + lane < len && slotSelected<MASKED>(slotMask, ls + v0), IS_L2 ? vals[0] : -vals[0],
                      (IdT)(ls + v0 + lane));
            }
        }
        block_merge_and_write<IdT>(w, warp, lists, perWarp, LIST, k, arenaIds, 0.f, oD, oI);
        return;
    }
    // generic path: each warp takes groups of 32 vectors; lanes stride the dimension
    for (int p = pBegin; p < pEnd; p++) {
        const idx_t l = probes[(int64_t)q * nprobe + p];
        if (l < 0)
            continue;
        const int len = listLen[l];
        const int64_t ls = listStart[l];
        const float* base = arenaVecs + ls * d;
        for (int v0 = warp * 32; v0 < len; v0 += kScanWarps * 32) {
            float mineKey = 0.f;
            const int cntv = min(32, len - v0);
            for (int v = 0; v < cntv; v++) {
                const float* row = base + (int64_t)(v0 + v) * d;
                float acc = 0.f;
                for (int i = lane; i < d; i += 32) {
                    float a = qs[i], b = row[i];
                    if (IS_L2) {
                        float df = a - b;
                        acc = fmaf(df, df, acc);
                    } else {
                        acc = fmaf(a, b, acc);
                    }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1)
                    acc += __shfl_xor_sync(kFullMask, acc, o);
                if (lane == v)
                    mineKey = IS_L2 ? acc : -acc;
            }
            w.add(lane < cntv && slotSelected<MASKED>(slotMask, ls + v0), mineKey, (IdT)(ls + v0 + lane));
        }
    }
    block_merge_and_write<IdT>(w, warp, lists, perWarp, LIST, k, arenaIds, 0.f, oD, oI);
}

// CTAs per query: 1 when the queries alone fill the machine several times over, else the probes are
// split so that ~8 CTAs per SM exist
int ivfScanChunks(int device, int64_t nq, int nprobe, int* probesPerCta) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    const int64_t wantCtas = (int64_t)sms * 8;
    int chunks = (int)std::min<int64_t>(nprobe, std::max<int64_t>(1, ceil_div(wantCtas, nq)));
    *probesPerCta = ceil_div(nprobe, chunks);
    return ceil_div(nprobe, *probesPerCta);
}

void runIvfScanBatches(
        GpuResources* res,
        int device,
        const IvfScanCall& call,
        bool oneProbePerCta,
        const char* timingName,
        const std::function<void(const IvfScanBatch&)>& launch) {
    const int64_t nq = call.nq;
    const int k = call.k;
    if (nq == 0)
        return;
    int probesPerCta = 1;
    const int ctasPerQuery = oneProbePerCta ? call.nprobe : ivfScanChunks(device, nq, call.nprobe, &probesPerCta);
    // query batches bound the partial-result scratch
    const int64_t maxQ =
            std::max<int64_t>(1, std::min<int64_t>(65535, (int64_t(1) << 30) / ((int64_t)ctasPerQuery * k * 12)));
    for (int64_t q0 = 0; q0 < nq; q0 += maxQ) {
        const int64_t nb = std::min(maxQ, nq - q0);
        auto partD = res->temp(device, sizeof(float) * nb * ctasPerQuery * k);
        auto partI = res->temp(device, sizeof(idx_t) * nb * ctasPerQuery * k);
        const IvfScanBatch batch{
                q0, nb, dim3((unsigned)ctasPerQuery, (unsigned)nb), probesPerCta, partD.as<float>(), partI.as<idx_t>()};
        KernelTiming::begin(timingName, call.stream);
        launch(batch);
        KernelTiming::end(timingName, call.stream);
        CUDA_CHECK_LAST();
        if (call.slots)
            runIvfMergeTopKSlots(
                    partD.as<float>(), partI.as<idx_t>(), call.slots->arenaIds, nb, ctasPerQuery, k, k, call.metric,
                    call.outD + q0 * k, call.outI + q0 * k, call.slots->outSlot + q0 * k, call.stream);
        else
            runMergeTopKKeyspace(
                    partD.as<float>(), partI.as<idx_t>(), nb, ctasPerQuery, k, k, call.metric, 0, call.outD + q0 * k,
                    call.outI + q0 * k, call.stream);
    }
}

static void runIvfFlatScan(GpuResources* res, int device, const IvfScanLayout& a, const IvfScanCall& c) {
    const int d = a.d, k = c.k, nprobe = c.nprobe;
    const int LIST = std::max(64, next_pow2(k));
    const bool wide = ivfScanWideIds(a);
    const size_t listBytes = wide ? SmemTopK<long long>::bytes(LIST, kScanBuf) : SmemTopK<int>::bytes(LIST, kScanBuf);
    size_t smem = round_up(sizeof(float) * d, 16) + listBytes * kScanWarps;
    FB_THROW_IF_NOT_MSG(smem <= 200 * 1024, "k / d too large for the IVF-Flat scan kernel");
    runIvfScanBatches(res, device, c, false, "ivfflat_scan", [&](const IvfScanBatch& b) {
        withBool(c.metric == METRIC_L2, [&](auto l2) {
            withBool(wide, [&](auto wideIds) {
                withBool(c.mask != nullptr, [&](auto masked) {
                    auto kern = ivfflat_scan_kernel<l2, ScanIdT<decltype(wideIds)>, masked>;
                    CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                    kern<<<b.grid, kScanWarps * 32, smem, c.stream>>>(
                            c.Q + b.q0 * d, d, c.probes + b.q0 * nprobe, nprobe, b.probesPerCta, a.listStart, a.listLen,
                            reinterpret_cast<const float*>(a.codes), a.ids, k, LIST, b.partD, b.partI, c.mask);
                });
            });
        });
    });
}

// ------------------------------------------------------------------------------------------
// IVF-PQ scan: block per (query, probe).  PACKED: codes of ksub = 2^nbits < 256 centroids, stored as the CPU's
// LSB-first bitstring of ceil(M * nbits / 8) bytes per vector; each lane decodes its vector from a 64-bit window.
// ------------------------------------------------------------------------------------------
template <bool IS_L2, bool PACKED, bool MASKED>
__global__ void __launch_bounds__(kScanWarps * 32) ivfpq_scan_kernel(
        const float* __restrict__ Q,
        int d,
        const idx_t* __restrict__ probes,
        const float* __restrict__ coarseDis,
        int nprobe,
        const float* __restrict__ coarse,
        const float* __restrict__ pq,
        int M,
        int ksub,
        const int64_t* __restrict__ listStart,
        const int* __restrict__ listLen,
        const uint8_t* __restrict__ arenaCodes,
        const idx_t* __restrict__ arenaIds,
        int k,
        int LIST,
        float* __restrict__ partD,
        idx_t* __restrict__ partI,
        const uint32_t* __restrict__ slotMask) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int q = blockIdx.y, p = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int dsub = d / M;
    float* lut = reinterpret_cast<float*>(smem_raw);           // [M][ksub]
    float* rs = lut + (size_t)M * ksub;                        // [d] residual (L2) or query (IP)
    unsigned char* lists = reinterpret_cast<unsigned char*>(rs) + round_up(sizeof(float) * d, 16);
    const size_t perWarp = SmemTopK<int>::bytes(LIST, kScanBuf);
    float* oD = partD + ((int64_t)q * nprobe + p) * k;
    idx_t* oI = partI + ((int64_t)q * nprobe + p) * k;

    const idx_t l = probes[(int64_t)q * nprobe + p];
    if (l < 0) {
        for (int j = threadIdx.x; j < k; j += blockDim.x) {
            oD[j] = CUDART_INF_F;
            oI[j] = -1;
        }
        return;
    }
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        float v = Q[(int64_t)q * d + i];
        rs[i] = IS_L2 ? v - coarse[l * d + i] : v;
    }
    WarpTopK<int> w;
    unsigned char* mine = lists + perWarp * warp;
    w.init(reinterpret_cast<float*>(mine), reinterpret_cast<int*>(mine + sizeof(float) * (LIST + kScanBuf)), LIST, kScanBuf, k);
    __syncthreads();
    // ---- LUT: lut[m][c] = ||r_m - pq[m][c]||^2 (L2)  or  q_m . pq[m][c] (IP; negated = key space)
    for (int e = threadIdx.x; e < M * ksub; e += blockDim.x) {
        const int m = e / ksub;
        const float* cp = pq + (size_t)e * dsub;
        const float* rp = rs + m * dsub;
        float acc = 0.f;
        for (int j = 0; j < dsub; j++) {
            if (IS_L2) {
                float df = rp[j] - cp[j];
                acc = fmaf(df, df, acc);
            } else {
                acc = fmaf(rp[j], cp[j], acc);
            }
        }
        lut[e] = IS_L2 ? acc : -acc;
    }
    __syncthreads();

    const int len = listLen[l];
    const int nbits = PACKED ? 31 - __clz(ksub) : 8;
    const int codeSize = PACKED ? (M * nbits + 7) >> 3 : M;
    const uint8_t* codes = arenaCodes + listStart[l] * (int64_t)codeSize;
    const bool vec16 = (M % 16) == 0; // list starts are multiples of 16 elements when M%16==0
    for (int v0 = threadIdx.x; v0 < round_up(len, 32); v0 += blockDim.x) {
        const bool valid = v0 < len;
        float acc = 0.f;
        if (valid) {
            const uint8_t* cp = codes + (int64_t)v0 * codeSize;
            if (PACKED) {
                // bits [0, have) of win are the next codes; refilled 32 bits at a time (have < nbits <= 8, so
                // the window never overflows), bytes past the row's end read as zero
                const unsigned mask = (unsigned)ksub - 1;
                uint64_t win = 0;
                int have = 0, pos = 0;
                for (int m = 0; m < M; m++) {
                    if (have < nbits) {
                        unsigned w = 0;
#pragma unroll
                        for (int b = 0; b < 4; b++)
                            if (pos + b < codeSize)
                                w |= (unsigned)__ldg(cp + pos + b) << (8 * b);
                        win |= (uint64_t)w << have;
                        have += 32;
                        pos += 4;
                    }
                    acc += lut[m * ksub + ((unsigned)win & mask)];
                    win >>= nbits;
                    have -= nbits;
                }
            } else if (vec16) {
                for (int m0 = 0; m0 < M; m0 += 16) {
                    const uint4 c4 = __ldg(reinterpret_cast<const uint4*>(cp + m0));
                    const unsigned wds[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
                    for (int wi = 0; wi < 4; wi++) {
#pragma unroll
                        for (int b = 0; b < 4; b++) {
                            const unsigned code = (wds[wi] >> (8 * b)) & 0xffu;
                            acc += lut[(m0 + wi * 4 + b) * ksub + code];
                        }
                    }
                }
            } else {
                for (int m = 0; m < M; m++)
                    acc += lut[m * ksub + cp[m]];
            }
        }
        w.add(valid && slotSelected<MASKED>(slotMask, listStart[l] + (v0 & ~31)), acc, v0);
    }
    // IP: total = q.c_list + sum_m q_m.pq  -> key = -(coarse + sum) ; L2: residual form, no add
    const float add = IS_L2 ? 0.f : -coarseDis[(int64_t)q * nprobe + p];
    block_merge_and_write(w, warp, lists, perWarp, LIST, k, arenaIds + listStart[l], add, oD, oI);
}

// vector-major codes: 8-bit, or the CPU's packed bitstring below 8 bits
static void runIvfPqScan(GpuResources* res, int device, const IvfScanLayout& a, const IvfScanCall& c) {
    const int d = a.d, k = c.k, nprobe = c.nprobe, M = a.M, nbits = a.nbits;
    FB_THROW_IF_NOT(nbits >= 1 && nbits <= 8);
    const int ksub = 1 << nbits;
    const bool packed = nbits != 8;
    const char* name = packed ? "ivfpq_scan_packed" : "ivfpq_scan";
    const int LIST = std::max(64, next_pow2(k));
    size_t smem = sizeof(float) * M * ksub + round_up(sizeof(float) * d, 16) +
            SmemTopK<int>::bytes(LIST, kScanBuf) * kScanWarps;
    FB_THROW_IF_NOT_MSG(smem <= 220 * 1024, "LUT + top-k lists do not fit shared memory (IVFPQ.cu:596-617)");
    runIvfScanBatches(res, device, c, true, name, [&](const IvfScanBatch& b) {
        withBool(c.metric == METRIC_L2, [&](auto l2) {
            withBool(packed, [&](auto pk) {
                withBool(c.mask != nullptr, [&](auto masked) {
                    auto kern = ivfpq_scan_kernel<l2, pk, masked>;
                    CUDA_VERIFY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                    kern<<<b.grid, kScanWarps * 32, smem, c.stream>>>(
                            c.Q + b.q0 * d, d, c.probes + b.q0 * nprobe, c.coarseDis + b.q0 * nprobe, nprobe,
                            a.centroids, a.pq, M, ksub, a.listStart, a.listLen, a.codes, a.ids, k, LIST, b.partD,
                            b.partI, c.mask);
                });
            });
        });
    });
}

void runIvfScan(GpuResources* res, int device, const IvfScanLayout& lists, const IvfScanCall& call) {
    if (call.nq == 0)
        return;
    IvfScanLayout a = lists;
    if (call.slots) // the scan returns arena positions; the batch merge turns them into the stored ids
        a.ids = call.slots->identity;
    if (a.kind == IVF_STORED_FLAT)
        runIvfFlatScan(res, device, a, call);
    else if (a.kind == IVF_STORED_SQ)
        runIvfSqScan(res, device, a, call);
    else if (a.interleaved)
        runIvfPqScanInterleaved(res, device, a, call);
    else
        runIvfPqScan(res, device, a, call);
}

} // namespace fb200
