// faiss_b200 -- IVF retrieval: from ids to arena slots, from slots to vectors or codes, and the merge of a
// search that keeps the slot of every result.
//
// Semantics are the CPU IndexIVF's (faiss/IndexIVF.cpp:1056-1248): reconstruct_n / reconstruct_batch resolve an
// id stored more than once to the entry last in (list, offset) order, and search_and_reconstruct /
// search_and_return_codes decode the entry the search returned.  Arena positions ascend with (list, offset), so
// "last in (list, offset) order" is "largest arena position": an atomicMax per hit, no persistent id map.
#include <cub/cub.cuh>

#include <cfloat>
#include <climits>

#include "ivf_layout.cuh"
#include "kernels.h"
#include "select.cuh"

namespace fb200 {

// a merge entry of the slot-keeping search: ordered by the stored id first, as the plain search's merge orders
// its ids, then by arena position (entries equal in key and id are indistinguishable in D and I)
struct IdSlot {
    long long id, slot;
};
__device__ __forceinline__ bool operator<(const IdSlot& a, const IdSlot& b) {
    return a.id < b.id || (a.id == b.id && a.slot < b.slot);
}
__device__ __forceinline__ bool operator!=(const IdSlot& a, const IdSlot& b) {
    return a.id != b.id || a.slot != b.slot;
}
template <>
struct IdLimits<IdSlot> {
    static __host__ __device__ constexpr IdSlot max() {
        return IdSlot{LLONG_MAX, LLONG_MAX};
    }
};

namespace {

// The CPU decode of the scalar quantiser (IndexIVFScalarQuantizer::reconstruct_from_offset -> ScalarQuantizer::decode
// -> QuantizerTemplate<..., SIMDLevel::NONE>::decode_vector, quantizers.h:92-146): decode_vector is final in the
// scalar class, so every build and every d takes  xi = (c + 0.5f) / s  (an IEEE division), then  vmin + xi * vdiff,
// which g++ contracts into one fused multiply-add at -O3 -mfma (the C++ default -ffp-contract=fast).
__device__ __forceinline__ float sqDecode(float c, float levels, float vmin, float vdiff) {
    const float xi = __fdiv_rn(__fadd_rn(c, 0.5f), levels);
    return __fmaf_rn(xi, vdiff, vmin);
}

// list of arena slot s: the last list whose start is <= s (starts ascend with the list number; a list of capacity 0
// shares its start with the next one)
__device__ __forceinline__ int64_t slotList(const int64_t* __restrict__ listStart, int64_t nlist, int64_t s) {
    int64_t lo = 0, hi = nlist;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(listStart + mid) <= s)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}

// byte b of the CPU code of the entry at arena slot s (list-relative position v, list start ls)
__device__ __forceinline__ unsigned codeByte(const IvfStoredLayout& a, int64_t s, int64_t ls, int b) {
    if (a.interleaved)
        return __ldg(a.codes + ls * a.codeSize + ivfInterleavedByte(s - ls, b, a.codeSize));
    return __ldg(a.codes + s * a.codeSize + b);
}

constexpr int kRowWarps = 4;

// one warp per output row; slot -1 -> all 0xFF bytes (fillMissing) or the row is left as it is
template <int KIND, int CODEC>
__global__ void __launch_bounds__(kRowWarps * 32) ivf_reconstruct_kernel(
        IvfStoredLayout a, const idx_t* __restrict__ slots, int64_t n, bool fillMissing, float* __restrict__ out) {
    const int64_t row = (int64_t)blockIdx.x * kRowWarps + (threadIdx.x >> 5);
    if (row >= n)
        return;
    const int lane = lane_id();
    const int d = a.d;
    float* o = out + row * d;
    const int64_t s = slots[row];
    if (s < 0) {
        if (fillMissing)
            for (int i = lane; i < d; i += 32)
                o[i] = __int_as_float(-1);
        return;
    }
    const int64_t l = slotList(a.listStart, a.nlist, s);
    const int64_t ls = __ldg(a.listStart + l);
    const float* cent = a.centroids ? a.centroids + l * d : nullptr;
    if (KIND == IVF_STORED_FLAT) {
        const float* y = reinterpret_cast<const float*>(a.codes) + s * d;
        for (int i = lane; i < d; i += 32)
            o[i] = __ldg(y + i);
    } else if (KIND == IVF_STORED_SQ) {
        const uint8_t* cp = a.codes + s * a.codeSize;
        for (int i = lane; i < d; i += 32) {
            float x = sq_row_comp<CODEC>(cp, i);
            if (a.levels > 0.f)
                x = sqDecode(x, a.levels, __ldg(a.vmin + i), __ldg(a.vdiff + i));
            o[i] = cent ? __fadd_rn(x, __ldg(cent + i)) : x;
        }
    } else { // PQ: code m at bits [m nbits, (m + 1) nbits) of the LSB-first bitstring, then + centroid
        const int dsub = d / a.M, ksub = 1 << a.nbits;
        for (int i = lane; i < d; i += 32) {
            const int m = i / dsub, j = i - m * dsub;
            const int bit = m * a.nbits, b = bit >> 3, sh = bit & 7;
            unsigned w = codeByte(a, s, ls, b);
            if (sh + a.nbits > 8)
                w |= codeByte(a, s, ls, b + 1) << 8;
            const unsigned c = (w >> sh) & (unsigned)(ksub - 1);
            const float x = __ldg(a.pq + ((int64_t)m * ksub + c) * dsub + j);
            o[i] = __fadd_rn(x, __ldg(cent + i));
        }
    }
}

// one warp per output row: [listno bytes, little-endian][the CPU code bytes]; slot -1 -> all 0xFF
__global__ void __launch_bounds__(kRowWarps * 32) ivf_gather_codes_kernel(
        IvfStoredLayout a, const idx_t* __restrict__ slots, int64_t n, int listnoBytes, uint8_t* __restrict__ out) {
    const int64_t row = (int64_t)blockIdx.x * kRowWarps + (threadIdx.x >> 5);
    if (row >= n)
        return;
    const int lane = lane_id();
    const int rowBytes = listnoBytes + a.codeSize;
    uint8_t* o = out + row * rowBytes;
    const int64_t s = slots[row];
    if (s < 0) {
        for (int b = lane; b < rowBytes; b += 32)
            o[b] = 0xff;
        return;
    }
    const int64_t l = slotList(a.listStart, a.nlist, s);
    const int64_t ls = __ldg(a.listStart + l);
    for (int b = lane; b < rowBytes; b += 32)
        o[b] = (uint8_t)(b < listnoBytes ? (uint64_t)l >> (8 * b) : codeByte(a, s, ls, b - listnoBytes));
}

// every occupied arena slot whose id is wanted records itself with an atomicMax: range mode (keys == null) into
// hit[id - i0] for i0 <= id < i0 + ni; key mode into hit[first position of id in the sorted keys]
__global__ void ivf_id_slots_kernel(
        IvfStoredLayout a, idx_t i0, idx_t ni, const idx_t* __restrict__ sortedKeys, int64_t nkeys, long long* hit) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.arenaElems)
        return;
    const int64_t l = slotList(a.listStart, a.nlist, s);
    if (s - __ldg(a.listStart + l) >= __ldg(a.listLen + l))
        return;
    const idx_t id = a.ids[s];
    if (!sortedKeys) {
        if (id >= i0 && id - i0 < ni)
            atomicMax(hit + (id - i0), (long long)s);
        return;
    }
    int64_t lo = 0, hi = nkeys; // first key >= id
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(sortedKeys + mid) < id)
            lo = mid + 1;
        else
            hi = mid;
    }
    if (lo < nkeys && __ldg(sortedKeys + lo) == id)
        atomicMax(hit + lo, (long long)s);
}

// sorted key i (originally at perm[i]) takes the hit of its key's first position; any absent key raises *missing
__global__ void ivf_key_slots_kernel(
        const idx_t* __restrict__ sortedKeys, const idx_t* __restrict__ perm, int64_t n, const long long* __restrict__ hit,
        idx_t* __restrict__ slots, int* missing) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const idx_t key = sortedKeys[i];
    int64_t lo = 0, hi = i; // first position of key
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(sortedKeys + mid) < key)
            lo = mid + 1;
        else
            hi = mid;
    }
    const long long s = hit[lo];
    slots[perm[i]] = s;
    if (s < 0)
        *missing = 1;
}

__global__ void iota_kernel(idx_t* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        out[i] = i;
}

// merge_topk_kernel<IN_KEYSPACE = true> (flat_exact.cu) over the scans' arena positions: the position is turned into
// the stored id on the way in and kept beside it, so the keys, ids and their order are those of the plain merge
__global__ void merge_topk_slots_kernel(
        const float* __restrict__ inD,
        const idx_t* __restrict__ inPos,
        const idx_t* __restrict__ arenaIds,
        int64_t rows,
        int nlists,
        int kin,
        int k,
        int LIST,
        int lowerIsBetter,
        float* __restrict__ outD,
        idx_t* __restrict__ outI,
        idx_t* __restrict__ outSlot) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = lane_id();
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (row >= rows)
        return;
    constexpr int BUF = 64;
    unsigned char* base = smem_raw + SmemTopK<IdSlot>::bytes(LIST, BUF) * warp;
    WarpTopK<IdSlot> w;
    w.init(reinterpret_cast<float*>(base), reinterpret_cast<IdSlot*>(base + sizeof(float) * (LIST + BUF)), LIST, BUF, k);
    const int64_t total = (int64_t)nlists * kin;
    const float* D = inD + row * total;
    const idx_t* P = inPos + row * total;
    for (int64_t e0 = 0; e0 < total; e0 += 32) {
        const int64_t e = e0 + lane;
        bool valid = e < total;
        float key = 0.f;
        IdSlot is{-1, -1};
        if (valid) {
            is.slot = P[e];
            key = D[e];
            is.id = is.slot == -1 ? -1 : arenaIds[is.slot];
            valid = is.id != -1; // the plain merge's "no result" marker
        }
        w.add(valid, key, is);
    }
    w.finish();
    for (int j = lane; j < k; j += 32) {
        const IdSlot is = w.q.ids[j];
        const bool ok = is != IdLimits<IdSlot>::max();
        const float key = w.q.keys[j];
        outD[row * k + j] = ok ? (lowerIsBetter ? key : -key) : (lowerIsBetter ? FLT_MAX : -FLT_MAX);
        outI[row * k + j] = ok ? (idx_t)is.id : -1;
        outSlot[row * k + j] = ok ? (idx_t)is.slot : -1;
    }
}

} // namespace

void runIvfIdentitySlots(idx_t* out, int64_t n, cudaStream_t stream) {
    if (n == 0)
        return;
    iota_kernel<<<(unsigned)ceil_div(n, (int64_t)256), 256, 0, stream>>>(out, n);
    CUDA_CHECK_LAST();
}

void runIvfMergeTopKSlots(
        const float* inD,
        const idx_t* inPos,
        const idx_t* arenaIds,
        int64_t rows,
        int nlists,
        int kin,
        int k,
        MetricType metric,
        float* outD,
        idx_t* outI,
        idx_t* outSlot,
        cudaStream_t stream) {
    if (rows == 0)
        return;
    const int LIST = std::max(64, next_pow2(k));
    const size_t per = SmemTopK<IdSlot>::bytes(LIST, 64);
    const int warps = (int)std::max<size_t>(1, std::min<size_t>(4, (96 * 1024) / per));
    const size_t smem = per * warps;
    CUDA_VERIFY(cudaFuncSetAttribute(merge_topk_slots_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    merge_topk_slots_kernel<<<(unsigned)ceil_div(rows, (int64_t)warps), warps * 32, smem, stream>>>(
            inD, inPos, arenaIds, rows, nlists, kin, k, LIST, is_similarity_metric(metric) ? 0 : 1, outD, outI, outSlot);
    CUDA_CHECK_LAST();
}

void runIvfSlotsOfRange(const IvfStoredLayout& a, idx_t i0, idx_t ni, idx_t* slots, cudaStream_t stream) {
    if (ni == 0)
        return;
    CUDA_VERIFY(cudaMemsetAsync(slots, 0xff, sizeof(idx_t) * ni, stream));
    if (a.arenaElems == 0)
        return;
    ivf_id_slots_kernel<<<(unsigned)ceil_div(a.arenaElems, (int64_t)256), 256, 0, stream>>>(
            a, i0, ni, nullptr, 0, reinterpret_cast<long long*>(slots));
    CUDA_CHECK_LAST();
}

bool runIvfSlotsOfKeys(GpuResources* res, int device, const IvfStoredLayout& a, const idx_t* keys, int64_t n, idx_t* slots, cudaStream_t stream) {
    if (n == 0)
        return true;
    FB_THROW_IF_NOT(n < (int64_t(1) << 31));
    auto buf = res->temp(device, sizeof(idx_t) * n * 4 + sizeof(int));
    idx_t* perm0 = buf.as<idx_t>();
    idx_t* sortedKeys = perm0 + n;
    idx_t* perm = sortedKeys + n;
    long long* hit = reinterpret_cast<long long*>(perm + n);
    int* missing = reinterpret_cast<int*>(hit + n);
    runIvfIdentitySlots(perm0, n, stream);
    size_t tb = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, sortedKeys, perm0, perm, (int)n, 0, 64, stream);
    auto tmp = res->temp(device, std::max<size_t>(tb, 16));
    cub::DeviceRadixSort::SortPairs(tmp.data, tb, keys, sortedKeys, perm0, perm, (int)n, 0, 64, stream);
    CUDA_VERIFY(cudaMemsetAsync(hit, 0xff, sizeof(long long) * n, stream));
    CUDA_VERIFY(cudaMemsetAsync(missing, 0, sizeof(int), stream));
    if (a.arenaElems > 0)
        ivf_id_slots_kernel<<<(unsigned)ceil_div(a.arenaElems, (int64_t)256), 256, 0, stream>>>(
                a, 0, 0, sortedKeys, n, hit);
    ivf_key_slots_kernel<<<(unsigned)ceil_div(n, (int64_t)256), 256, 0, stream>>>(sortedKeys, perm, n, hit, slots, missing);
    CUDA_CHECK_LAST();
    int h = 0;
    CUDA_VERIFY(cudaMemcpyAsync(&h, missing, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    return h == 0;
}

void runIvfReconstruct(const IvfStoredLayout& a, const idx_t* slots, int64_t n, bool fillMissing, float* out, cudaStream_t stream) {
    if (n == 0)
        return;
    const unsigned grid = (unsigned)ceil_div(n, (int64_t)kRowWarps);
    auto launch = [&](auto kern) {
        kern<<<grid, kRowWarps * 32, 0, stream>>>(a, slots, n, fillMissing, out);
    };
    if (a.kind == IVF_STORED_FLAT) {
        launch(ivf_reconstruct_kernel<IVF_STORED_FLAT, 0>);
    } else if (a.kind == IVF_STORED_PQ) {
        launch(ivf_reconstruct_kernel<IVF_STORED_PQ, 0>);
    } else {
        switch (a.sqCodec) {
            case SQC_BYTE:
                launch(ivf_reconstruct_kernel<IVF_STORED_SQ, SQC_BYTE>);
                break;
            case SQC_NIBBLE:
                launch(ivf_reconstruct_kernel<IVF_STORED_SQ, SQC_NIBBLE>);
                break;
            case SQC_SIX:
                launch(ivf_reconstruct_kernel<IVF_STORED_SQ, SQC_SIX>);
                break;
            default:
                launch(ivf_reconstruct_kernel<IVF_STORED_SQ, SQC_HALF>);
                break;
        }
    }
    CUDA_CHECK_LAST();
}

void runIvfGatherCodes(const IvfStoredLayout& a, const idx_t* slots, int64_t n, int listnoBytes, uint8_t* out, cudaStream_t stream) {
    if (n == 0)
        return;
    ivf_gather_codes_kernel<<<(unsigned)ceil_div(n, (int64_t)kRowWarps), kRowWarps * 32, 0, stream>>>(
            a, slots, n, listnoBytes, out);
    CUDA_CHECK_LAST();
}

} // namespace fb200
