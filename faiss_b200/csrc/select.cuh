// faiss_b200 -- k-selection primitive (device side).
//
// Role of the reference's BlockSelect / WarpSelect + merge networks
// (faiss/gpu/utils/Select.cuh:147-343,439-594; MergeNetworkWarp.cuh; MergeNetworkBlock.cuh),
// re-designed: one shared-memory "sorted list + candidate buffer" per selection problem, owned by
// a single warp.  Candidates that beat the current k-th key are appended to the buffer with a
// ballot-compacted write; when the buffer is more than half full the warp sorts it (bitonic) and
// folds it into the list with one bitonic half-merge (the list stays sorted, only the best LIST
// entries survive).  Steady-state cost per element is one compare + one vote.
//
// Ordering: smaller key is better; ties are broken by smaller id, i.e. the total order
// (key asc, id asc) that the reference CPU result handlers produce
// (faiss/utils/ordered_key_value.h:40-75, faiss/impl/ResultHandler.h:275-282).  Inner-product
// search negates keys on the way in and on the way out.
#pragma once

#include <cuda_runtime.h>
#include <math_constants.h>

#include <cfloat>
#include <cstdint>

namespace fb200 {

constexpr unsigned kFullMask = 0xffffffffu;

template <typename IdT>
struct IdLimits;
template <>
struct IdLimits<int> {
    static __host__ __device__ constexpr int max() {
        return 0x7fffffff;
    }
};
template <>
struct IdLimits<long long> {
    static __host__ __device__ constexpr long long max() {
        return 0x7fffffffffffffffLL;
    }
};

// The reference's result rule, in key space: an entry is a result only if its key is strictly better than the
// missing-result sentinel FLT_MAX (faiss/impl/ResultHandler.h:275-282 against the heap's neutral element,
// faiss/utils/ordered_key_value.h).  That is dis < FLT_MAX for L2 and the other distances, dis > -FLT_MAX for a
// similarity; NaN never qualifies.  Every list and merge also recognises an empty slot by its key (they start at
// +inf), never by the id it holds, so any stored id survives.
__device__ __forceinline__ bool isResult(float key) {
    return key < FLT_MAX;
}

template <typename IdT>
__device__ __forceinline__ bool kv_less(float ka, IdT ia, float kb, IdT ib) {
    return (ka < kb) || (ka == kb && ia < ib);
}

__device__ __forceinline__ int lane_id() {
    return threadIdx.x & 31;
}

// Shared-memory top-k list owned by one warp.
//   keys/ids : arrays of LIST + BUF entries; [0, LIST) sorted ascending, [LIST, LIST+BUF) buffer
//   LIST     : power of two, >= BUF, >= k
//   BUF      : power of two (64 / 128 / 256); flush when more than BUF/2 are pending, so a caller
//              may append up to BUF/2 entries between two `maybe_flush` calls.
template <typename IdT>
struct SmemTopK {
    float* keys;
    IdT* ids;
    float* bkeys; // pending buffer (keys + LIST unless the owner places it elsewhere)
    IdT* bids;
    int LIST;
    int BUF;
    int k;

    __host__ __device__ __forceinline__ static size_t bytes(int LIST, int BUF) {
        return size_t(LIST + BUF) * (sizeof(float) + sizeof(IdT));
    }

    // warp-collective
    __device__ void init() {
        for (int i = lane_id(); i < LIST + BUF; i += 32) {
            keys[i] = CUDART_INF_F;
            ids[i] = IdLimits<IdT>::max();
        }
        __syncwarp();
    }

    __device__ __forceinline__ float threshold() const {
        return keys[k - 1];
    }

    // warp-collective: sort the n_pending buffered entries ascending (bitonic, padded with sentinels to a
    // power of two >= 32); returns the padded size
    __device__ int sort_buffer(int n_pending) {
        const int lane = lane_id();
        float* bk = bkeys;
        IdT* bi = bids;
        int n = 32;
        while (n < n_pending)
            n <<= 1;
        for (int i = n_pending + lane; i < n; i += 32) {
            bk[i] = CUDART_INF_F;
            bi[i] = IdLimits<IdT>::max();
        }
        __syncwarp();
        for (int size = 2; size <= n; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int t = lane; t < (n >> 1); t += 32) {
                    // stride is a power of two: a = 2*stride*(t/stride) + t%stride without the division
                    int a = ((t & ~(stride - 1)) << 1) | (t & (stride - 1));
                    int b = a + stride;
                    bool asc = ((a & size) == 0);
                    float ka = bk[a], kb = bk[b];
                    IdT ia = bi[a], ib = bi[b];
                    bool sw = asc ? kv_less(kb, ib, ka, ia) : kv_less(ka, ia, kb, ib);
                    if (sw) {
                        bk[a] = kb;
                        bk[b] = ka;
                        bi[a] = ib;
                        bi[b] = ia;
                    }
                }
                __syncwarp();
            }
        }
        return n;
    }

    // warp-collective: merge the sorted buffer (n entries, n <= LIST) into the sorted list
    __device__ void merge_sorted_buffer(int n) {
        const int lane = lane_id();
        const float* bk = bkeys;
        const IdT* bi = bids;
        // half-merge stage 0: L[LIST-1-j] = min(L[LIST-1-j], B[j])  (B ascending, L ascending)
        for (int j = lane; j < n; j += 32) {
            int a = LIST - 1 - j;
            float ka = keys[a], kb = bk[j];
            IdT ia = ids[a], ib = bi[j];
            if (kv_less(kb, ib, ka, ia)) {
                keys[a] = kb;
                ids[a] = ib;
            }
        }
        __syncwarp();
        // L is now bitonic and holds the LIST best; finish with a bitonic merge
        for (int stride = LIST >> 1; stride > 0; stride >>= 1) {
            for (int t = lane; t < (LIST >> 1); t += 32) {
                int a = ((t & ~(stride - 1)) << 1) | (t & (stride - 1));
                int b = a + stride;
                float ka = keys[a], kb = keys[b];
                IdT ia = ids[a], ib = ids[b];
                if (kv_less(kb, ib, ka, ia)) {
                    keys[a] = kb;
                    keys[b] = ka;
                    ids[a] = ib;
                    ids[b] = ia;
                }
            }
            __syncwarp();
        }
    }

    // warp-collective: sort buffer (n_pending valid entries), merge into list.
    __device__ void flush(int n_pending) {
        merge_sorted_buffer(sort_buffer(n_pending));
    }
};

// Warp-private streaming interface over SmemTopK: every lane offers one (key,id) per call.
template <typename IdT>
struct WarpTopK {
    SmemTopK<IdT> q;
    int cnt;   // pending entries in the buffer (warp-uniform)
    float thr; // key of the current k-th (warp-uniform)

    __device__ void init(float* keys, IdT* ids, int LIST, int BUF, int k) {
        q.keys = keys;
        q.ids = ids;
        q.bkeys = keys + LIST;
        q.bids = ids + LIST;
        q.LIST = LIST;
        q.BUF = BUF;
        q.k = k;
        q.init();
        cnt = 0;
        thr = CUDART_INF_F;
    }

    // warp-collective; `valid` false lanes offer nothing.  NaN keys never pass.
    __device__ __forceinline__ void add(bool valid, float key, IdT id) {
        bool pass = valid && (key <= thr);
        unsigned m = __ballot_sync(kFullMask, pass);
        if (m) {
            int pos = cnt + __popc(m & ((1u << lane_id()) - 1u));
            if (pass) {
                q.bkeys[pos] = key;
                q.bids[pos] = id;
            }
            cnt += __popc(m);
            if (cnt > q.BUF - 32) {
                __syncwarp();
                q.flush(cnt);
                cnt = 0;
                thr = q.threshold();
            }
        }
    }

    __device__ void finish() {
        __syncwarp();
        if (cnt > 0) {
            q.flush(cnt);
            cnt = 0;
        }
        thr = q.threshold();
        __syncwarp();
    }
};

// CTA-shared top-k: ONE sorted list per CTA plus a small pending buffer per warp.
//
// Why: with a private list per warp each warp's threshold only reflects the 1/W of the stream it has
// seen, so W lists let ~W x more candidates through (k ln(n/(W k)) each) and every one of them costs a
// shared-memory merge -- on the IVF-PQ scan (16 warps, k = 100) that was ~20 % of the kernel's
// shared-memory wavefronts and instructions.  Here every warp filters against the CTA-wide k-th key
// (`sthr`, possibly a little stale -- a stale threshold is only looser, never wrong: the k-th key of a
// subset is an upper bound of the final k-th key), appends survivors to its own buffer with a ballot
// compaction, sorts the buffer privately, and only the final half-merge into the shared list runs
// under a CTA-wide lock.  The result is the exact top-k by (key, id) whatever the interleaving.
template <typename IdT>
struct CtaTopK {
    // a warp offers its buffer to the list once it holds more than kTrigger entries; while the list is busy (another
    // warp merging) and the buffer still has room for one more round of 32 it simply keeps scanning -- it only
    // blocks on the lock when the buffer could overflow
    static constexpr int BUF = 128;
    static constexpr int kTrigger = 32;
    SmemTopK<IdT> q; // q.keys/q.ids = shared list, q.bkeys/q.bids = this warp's buffer
    int* lock;
    volatile float* sthr;
    int cnt;
    float thr;

    __host__ __device__ static size_t bytes(int LIST, int warps) {
        return (size_t)LIST * (sizeof(float) + sizeof(IdT)) + (size_t)warps * BUF * (sizeof(float) + sizeof(IdT));
    }

    // block-collective: carve `mem` (bytes(LIST, warps), 16-byte aligned), initialise the shared list.
    // ctl: two 4-byte words of shared memory (lock, threshold).  Caller must __syncthreads() afterwards.
    __device__ void init(unsigned char* mem, int* ctl, int LIST, int k, int warps) {
        q.keys = reinterpret_cast<float*>(mem);
        q.ids = reinterpret_cast<IdT*>(mem + sizeof(float) * LIST);
        unsigned char* bufs = mem + (size_t)LIST * (sizeof(float) + sizeof(IdT));
        const int warp = threadIdx.x >> 5;
        q.bkeys = reinterpret_cast<float*>(bufs) + warp * BUF;
        q.bids = reinterpret_cast<IdT*>(bufs + sizeof(float) * warps * BUF) + warp * BUF;
        q.LIST = LIST;
        q.BUF = BUF;
        q.k = k;
        lock = ctl;
        sthr = reinterpret_cast<volatile float*>(ctl + 1);
        for (int i = threadIdx.x; i < LIST; i += blockDim.x) {
            q.keys[i] = CUDART_INF_F;
            q.ids[i] = IdLimits<IdT>::max();
        }
        if (threadIdx.x == 0) {
            ctl[0] = 0;
            *sthr = CUDART_INF_F;
        }
        cnt = 0;
        thr = CUDART_INF_F;
    }

    __device__ __forceinline__ void refresh() {
        thr = *sthr;
    }

    // warp-collective; `valid` false lanes offer nothing.  NaN keys never pass.
    __device__ __forceinline__ void add(bool valid, float key, IdT id) {
        const bool pass = valid && (key <= thr);
        const unsigned m = __ballot_sync(kFullMask, pass);
        if (m) {
            const int pos = cnt + __popc(m & ((1u << lane_id()) - 1u));
            if (pass) {
                q.bkeys[pos] = key;
                q.bids[pos] = id;
            }
            cnt += __popc(m);
            if (cnt > kTrigger)
                drain();
        }
    }

    // drop buffered entries that no longer beat the (refreshed) threshold
    __device__ void compact() {
        const int lane = lane_id();
        constexpr int S = BUF / 32;
        float kk[S];
        IdT ii[S];
        bool pp[S];
#pragma unroll
        for (int s = 0; s < S; s++) {
            const bool h = lane + 32 * s < cnt;
            kk[s] = h ? q.bkeys[lane + 32 * s] : 0.f;
            ii[s] = h ? q.bids[lane + 32 * s] : 0;
            pp[s] = h && kk[s] <= thr;
        }
        __syncwarp(); // every entry is in registers before any slot is overwritten
        const unsigned lt = (1u << lane) - 1u;
        int base = 0;
#pragma unroll
        for (int s = 0; s < S; s++) {
            const unsigned m = __ballot_sync(kFullMask, pp[s]);
            if (pp[s]) {
                const int pos = base + __popc(m & lt);
                q.bkeys[pos] = kk[s];
                q.bids[pos] = ii[s];
            }
            base += __popc(m);
        }
        cnt = base;
        __syncwarp();
    }

    // warp-collective: fold the pending buffer into the shared list
    __device__ void drain(bool force = false) {
        __syncwarp();
        const float t = *sthr;
        if (t < thr) { // somebody tightened the threshold since we filtered: re-filter first
            thr = t;
            compact();
            if (!force && cnt <= kTrigger)
                return;
        }
        if (cnt == 0)
            return;
        // the list is busy and the next round of 32 still fits: come back later instead of spinning
        if (!force && cnt <= BUF - 32 && *reinterpret_cast<volatile int*>(lock) != 0)
            return;
        const int n = q.sort_buffer(cnt); // private: no lock needed
        if (lane_id() == 0) {
            unsigned ns = 32;
            while (atomicCAS(lock, 0, 1) != 0) {
                __nanosleep(ns);
                ns = min(ns * 2, 512u);
            }
        }
        __syncwarp();
        __threadfence_block();
        q.merge_sorted_buffer(n);
        const float nt = q.keys[q.k - 1];
        __syncwarp();
        if (lane_id() == 0)
            *sthr = nt;
        __threadfence_block();
        __syncwarp();
        if (lane_id() == 0)
            atomicExch(lock, 0);
        cnt = 0;
        thr = nt;
    }

    __device__ void finish() {
        if (cnt > 0)
            drain(true);
    }
};

// order-preserving float -> uint32 (for packed 64-bit atomicMin argmin)
__device__ __forceinline__ unsigned float_to_ordered(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

} // namespace fb200
