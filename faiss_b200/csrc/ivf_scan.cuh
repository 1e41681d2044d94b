// faiss_b200 -- device helpers shared by the IVF list scans that keep per-warp top-k lists across a
// chunk of probes (ivf.cu: IVF-Flat and the flat-layout IVF-PQ scan; ivfsq_scan.cu: IVF-SQ).
#pragma once

#include <cfloat>

#include "kernels.h"
#include "select.cuh"

namespace fb200 {

// the key-space merge of per-chunk partial results (flat_exact.cu) and the probe split of a scan launch (ivf.cu)
void runMergeTopKKeyspace(
        const float*, const idx_t*, int64_t, int, int, int, MetricType, int64_t, float*, idx_t*, cudaStream_t);
int ivfScanChunks(int device, int64_t nq, int nprobe, int* probesPerCta);

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
        for (int j = lane_id(); j < k; j += 32) {
            IdT id = w.q.ids[j];
            bool ok2 = id != IdLimits<IdT>::max();
            outD[j] = ok2 ? w.q.keys[j] + addToKey : CUDART_INF_F;
            outI[j] = ok2 ? (ids ? ids[id] : (idx_t)id) : -1;
        }
    }
}

} // namespace fb200
