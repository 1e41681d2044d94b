// faiss_b200 -- helpers shared by the IVF list scans: the host-side batch-and-merge driver and template
// dispatch of every scan launcher (ivf.cu, ivfpq_scan.cu, ivfsq_scan.cu), and the device-side block merge
// of the scans that keep per-warp top-k lists across a chunk of probes (IVF-Flat, the flat-layout IVF-PQ
// scan, IVF-SQ).
#pragma once

#include <cfloat>
#include <functional>
#include <type_traits>

#include "kernels.h"
#include "select.cuh"

namespace fb200 {

// CTAs per query of a chunked scan: each CTA walks *probesPerCta consecutive probes of its query
int ivfScanChunks(int device, int64_t nq, int nprobe, int* probesPerCta);

// one query batch of a scan launch: queries [q0, q0 + nb), grid (CTAs per query, nb), partial results
// [nb][CTAs per query][k] in key space
struct IvfScanBatch {
    int64_t q0, nb;
    dim3 grid;
    int probesPerCta;
    float* partD;
    idx_t* partI;
};

// Splits call.nq queries into batches that bound the partial-result scratch, calls `launch` once per batch (the
// scan kernel launch, bracketed by KernelTiming `timingName`) and merges each batch's partial results into
// call.outD / call.outI.  oneProbePerCta: one CTA per (query, probe); else the probes are split by ivfScanChunks.
// With call.slots, the launch writes arena positions (the scan reads slots->identity as its id table), merged by
// runIvfMergeTopKSlots into outI and slots->outSlot.
void runIvfScanBatches(
        GpuResources* res,
        int device,
        const IvfScanCall& call,
        bool oneProbePerCta,
        const char* timingName,
        const std::function<void(const IvfScanBatch&)>& launch);

// the scans of runIvfScan that live in their own files; `lists.ids` is the id table the scan reads
void runIvfPqScanInterleaved(GpuResources* res, int device, const IvfScanLayout& lists, const IvfScanCall& call);
void runIvfSqScan(GpuResources* res, int device, const IvfScanLayout& lists, const IvfScanCall& call);

// runtime value -> compile-time constant (see withBool): f(std::integral_constant<int, V>{}) for the V of Vs equal to v
template <int... Vs, typename F>
void withInt(int v, F&& f) {
    const bool found = ((v == Vs ? (f(std::integral_constant<int, Vs>{}), true) : false) || ...);
    FB_THROW_IF_NOT(found);
}
// SearchParameters::sel over the arena (idselector.h): is this lane's slot of the group of 32 slots that starts
// at arena position slot0 selected?  Lists start 32-aligned, so a group is one mask word: one broadcast load per
// warp.  MASKED = false (no selector) compiles to nothing.
template <bool MASKED>
__device__ __forceinline__ bool slotSelected(const uint32_t* __restrict__ mask, int64_t slot0) {
    if (!MASKED)
        return true;
    return (__ldg(mask + (slot0 >> 5)) >> lane_id()) & 1u;
}

// list ids of the scans' top-k lists: arena positions, 64-bit once they do not fit an int
template <typename Wide>
using ScanIdT = std::conditional_t<Wide::value, long long, int>;
inline bool ivfScanWideIds(const IvfStoredLayout& lists) {
    return lists.arenaElems >= (int64_t(1) << 31) - 1;
}

// ------------------------------------------------------------------------------------------
// block-level helper: merge the per-warp lists of a block into warp 0's list, write k results
// ------------------------------------------------------------------------------------------
constexpr int kScanWarps = 4;
constexpr int kScanBuf = 64;

template <typename IdT>
__device__ void block_merge_and_write(
        WarpTopK<IdT>& w,
        int warp,
        unsigned char* smemLists,
        size_t perWarp,
        int LIST,
        int k,
        const idx_t* __restrict__ ids, // list ids (arena + listStart), may be null
        float addToKey,
        float* __restrict__ outD,
        idx_t* __restrict__ outI) {
    w.finish();
    __syncthreads();
    if (warp == 0) {
        for (int ow = 1; ow < kScanWarps; ow++) {
            const float* ok = reinterpret_cast<const float*>(smemLists + perWarp * ow);
            const IdT* oi = reinterpret_cast<const IdT*>(smemLists + perWarp * ow + sizeof(float) * (LIST + kScanBuf));
            for (int e0 = 0; e0 < k; e0 += 32) {
                int e = e0 + lane_id();
                bool valid = e < k;
                float key = valid ? ok[e] : 0.f;
                IdT id = valid ? oi[e] : 0;
                valid = valid && id != IdLimits<IdT>::max();
                if (!__any_sync(kFullMask, valid && key <= w.thr))
                    break; // sorted: nothing further can enter
                w.add(valid, key, id);
            }
        }
        w.finish();
        // list ids are arena positions, so the sentinel id marks an empty slot; the result rule applies to the final
        // key (a constant shift per CTA keeps every entry it drops behind the ones it keeps)
        for (int j = lane_id(); j < k; j += 32) {
            IdT id = w.q.ids[j];
            const float key = w.q.keys[j] + addToKey;
            bool ok2 = id != IdLimits<IdT>::max() && isResult(key);
            outD[j] = ok2 ? key : CUDART_INF_F;
            outI[j] = ok2 ? (ids ? ids[id] : (idx_t)id) : -1;
        }
    }
}

} // namespace fb200
