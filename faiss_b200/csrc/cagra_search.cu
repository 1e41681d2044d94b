// faiss_b200 -- GpuIndexCagra search: single-CTA CAGRA graph traversal, one CTA per query.
//
// Shared memory of one CTA (all sizes from CagraSearchPlan):
//   query      [d] fp32
//   itopk      [P2(itopk)] (key, id): the internal top-k, sorted by (key, id); key = L2 distance or -inner product.
//              id bit 31 marks an entry whose neighbours have been gathered (expanded).  Entries past itopk are +inf.
//   cand       [P2(candidates)] (key, id): this iteration's gathered neighbours
//   hash       [2^hashBits] uint32: the visited set (open addressing, linear probing, 0xFFFFFFFF = empty)
//   parents    [search_width] uint32
// One iteration: the best search_width unexpanded entries become parents; their graph_degree neighbours are
// gathered; ids already in the visited set are dropped; teams of team_size lanes compute the distances of the rest
// with 128-bit row loads; the candidates are bitonic-sorted and merged into itopk (a bitonic merge of the sorted
// buffer against the reversed candidates).
//
// The visited set is sized so that it never overflows: before an iteration whose gathers could push the number of
// insertions past hashmap_max_fill_rate, it is cleared and refilled with the ids in itopk.  An id dropped from itopk
// cannot come back (its (key, id) is worse than the current itopk's last entry), so a reset changes nothing but the
// distance count.  Insertions are counted as (parents x graph_degree) per iteration, not as successful inserts, so the
// reset schedule is the same on every run.  Ties between two teams inserting the same id decide only which of them
// computes its distance, so results are bit-identical across runs.
#include "kernels.h"

#include <math_constants.h>

#include <cfloat>

namespace fb200 {

namespace {

constexpr uint32_t kCagraInvalid = 0x7FFFFFFFu; // an empty itopk / candidate slot
constexpr uint32_t kCagraExpanded = 0x80000000u;
constexpr uint32_t kHashEmpty = 0xFFFFFFFFu;
constexpr unsigned kFullMask = 0xffffffffu;

__device__ __forceinline__ bool kl_less(float ka, uint32_t ia, float kb, uint32_t ib) {
    ia &= ~kCagraExpanded;
    ib &= ~kCagraExpanded;
    return ka < kb || (ka == kb && ia < ib);
}

__device__ __forceinline__ void kl_swap_if(float* key, uint32_t* id, int a, int b, bool up) {
    const float ka = key[a], kb = key[b];
    const uint32_t ia = id[a], ib = id[b];
    if (kl_less(kb, ib, ka, ia) == up) {
        key[a] = kb;
        key[b] = ka;
        id[a] = ib;
        id[b] = ia;
    }
}

// full bitonic sort, ascending, of n (a power of two) entries
__device__ void cta_bitonic_sort(float* key, uint32_t* id, int n) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
                const int a = 2 * t - (t & (stride - 1));
                const int b = a + stride;
                kl_swap_if(key, id, a, b, (a & size) == 0);
            }
            __syncthreads();
        }
    }
}

// merge the sorted candidates cand[0:nc) into the sorted buffer buf[0:nb) (both powers of two), keeping the best nb
// of the union; entries at m and past are reset to +inf (the buffer holds m <= nb real entries)
__device__ void cta_merge_into(float* bk, uint32_t* bi, int nb, int m, const float* ck, const uint32_t* ci, int nc) {
    const int lo = nb > nc ? nb - nc : 0;
    for (int i = lo + threadIdx.x; i < nb; i += blockDim.x) {
        const int j = nb - 1 - i; // < nc
        if (kl_less(ck[j], ci[j], bk[i], bi[i])) {
            bk[i] = ck[j];
            bi[i] = ci[j];
        }
    }
    __syncthreads();
    // bk is now bitonic (ascending, then descending): one bitonic merge sorts it
    for (int stride = nb >> 1; stride > 0; stride >>= 1) {
        for (int t = threadIdx.x; t < (nb >> 1); t += blockDim.x) {
            const int a = 2 * t - (t & (stride - 1));
            kl_swap_if(bk, bi, a, a + stride, true);
        }
        __syncthreads();
    }
    for (int i = m + threadIdx.x; i < nb; i += blockDim.x) {
        bk[i] = CUDART_INF_F; // +inf
        bi[i] = kCagraInvalid;
    }
    __syncthreads();
}

__device__ __forceinline__ uint32_t hash_slot(uint32_t id, int bits) {
    return (id * 0x9E3779B1u) >> (32 - bits);
}
// true when id was not in the set (it is now)
__device__ __forceinline__ bool hash_insert(uint32_t* table, int bits, uint32_t id) {
    const uint32_t mask = (1u << bits) - 1;
    uint32_t s = hash_slot(id, bits);
    while (true) {
        const uint32_t prev = atomicCAS(table + s, kHashEmpty, id);
        if (prev == kHashEmpty)
            return true;
        if (prev == id)
            return false;
        s = (s + 1) & mask;
    }
}

// splitmix64 finaliser: the initial random entry ids of a query, a function of (seed, query row in the call, i)
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

template <int VEC>
__device__ __forceinline__ float team_distance(
        const float* __restrict__ q, const float* __restrict__ row, int d, int lane, int team, bool ip) {
    float acc = 0.f;
    if (VEC == 4) {
        const float4* r4 = reinterpret_cast<const float4*>(row);
        const float4* q4 = reinterpret_cast<const float4*>(q);
        for (int j = lane; j < (d >> 2); j += team) {
            const float4 y = __ldg(r4 + j);
            const float4 x = q4[j];
            if (ip) {
                acc = fmaf(x.x, y.x, acc);
                acc = fmaf(x.y, y.y, acc);
                acc = fmaf(x.z, y.z, acc);
                acc = fmaf(x.w, y.w, acc);
            } else {
                float t = x.x - y.x;
                acc = fmaf(t, t, acc);
                t = x.y - y.y;
                acc = fmaf(t, t, acc);
                t = x.z - y.z;
                acc = fmaf(t, t, acc);
                t = x.w - y.w;
                acc = fmaf(t, t, acc);
            }
        }
    } else {
        for (int j = lane; j < d; j += team) {
            const float y = __ldg(row + j), x = q[j];
            if (ip) {
                acc = fmaf(x, y, acc);
            } else {
                const float t = x - y;
                acc = fmaf(t, t, acc);
            }
        }
    }
    for (int o = team >> 1; o > 0; o >>= 1)
        acc += __shfl_xor_sync(kFullMask, acc, o);
    return acc;
}

// team-parallel: score the ids cid[0:n) (kCagraInvalid entries are skipped) into ck / ci, dropping visited ids
template <int VEC>
__device__ void score_candidates(
        const CagraSearchArgs& a, const float* q, float* ck, uint32_t* ci, int n, uint32_t* hash, unsigned long long& count) {
    const int team = a.teamSize;
    const int lane = threadIdx.x & (team - 1);
    const int nTeams = blockDim.x / team;
    const int t0 = threadIdx.x / team;
    const bool ip = a.metric == METRIC_INNER_PRODUCT;
    for (int c0 = 0; c0 < n; c0 += nTeams) { // uniform trip count: the team shuffles need every lane of the warp
        const int c = c0 + t0;
        uint32_t id = c < n ? ci[c] : kCagraInvalid;
        int fresh = 0;
        if (lane == 0 && id != kCagraInvalid)
            fresh = hash_insert(hash, a.hashBits, id) ? 1 : 0;
        fresh = __shfl_sync(kFullMask, fresh, threadIdx.x & 31 & ~(team - 1));
        // every lane of the warp runs the team reduction (a team with nothing to score reduces zeros)
        const float dist = team_distance<VEC>(q, fresh ? a.data + (size_t)id * a.d : q, fresh ? a.d : 0, lane, team, ip);
        const float key = fresh ? (ip ? -dist : dist) : CUDART_INF_F;
        if (!fresh)
            id = kCagraInvalid;
        else if (lane == 0)
            count++;
        if (c < n && lane == 0) {
            ck[c] = key;
            ci[c] = id;
        }
    }
}

template <int VEC>
__global__ void cagra_search_kernel(CagraSearchArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int64_t qi = blockIdx.x;
    float* q = reinterpret_cast<float*>(smem);
    float* bk = q + round_up(a.d, 4);
    uint32_t* bi = reinterpret_cast<uint32_t*>(bk + a.bufSize);
    float* ck = reinterpret_cast<float*>(bi + a.bufSize);
    uint32_t* ci = reinterpret_cast<uint32_t*>(ck + a.candSize);
    uint32_t* hash = ci + a.candSize;
    uint32_t* parents = hash + (1 << a.hashBits);
    __shared__ int nParents;
    __shared__ unsigned long long ctaCount;

    for (int j = threadIdx.x; j < a.d; j += blockDim.x)
        q[j] = a.queries[qi * a.d + j];
    for (int i = threadIdx.x; i < a.bufSize; i += blockDim.x) {
        bk[i] = CUDART_INF_F;
        bi[i] = kCagraInvalid;
    }
    for (int i = threadIdx.x; i < (1 << a.hashBits); i += blockDim.x)
        hash[i] = kHashEmpty;
    if (threadIdx.x == 0)
        ctaCount = 0;
    unsigned long long count = 0;

    // initial candidates: random ids, a function of (seed, the query's row in the whole call, sample number)
    const uint64_t rowKey = mix64(a.seed ^ mix64((uint64_t)(a.rowOffset + qi)));
    for (int i = threadIdx.x; i < a.candSize; i += blockDim.x)
        ci[i] = i < a.numInit ? (uint32_t)(mix64(rowKey + (uint64_t)i) % (uint64_t)a.n) : kCagraInvalid;
    __syncthreads();
    score_candidates<VEC>(a, q, ck, ci, a.numInit, hash, count);
    for (int i = a.numInit + threadIdx.x; i < a.candSize; i += blockDim.x) {
        ck[i] = CUDART_INF_F;
        ci[i] = kCagraInvalid;
    }
    __syncthreads();
    cta_bitonic_sort(ck, ci, a.candSize);
    cta_merge_into(bk, bi, a.bufSize, a.itopk, ck, ci, a.candSize);
    int inserted = a.numInit;

    const int nGather = a.searchWidth * a.graphDegree;
    for (int iter = 0; iter < a.maxIterations; iter++) {
        // parents: the first search_width unexpanded entries of itopk, in order (warp 0, one ballot per 32 entries)
        if (threadIdx.x < 32) {
            int got = 0;
            for (int base = 0; base < a.itopk && got < a.searchWidth; base += 32) {
                const int i = base + (int)threadIdx.x;
                const bool open = i < a.itopk && bi[i] != kCagraInvalid && !(bi[i] & kCagraExpanded);
                const unsigned m = __ballot_sync(kFullMask, open);
                const int rank = got + __popc(m & ((1u << threadIdx.x) - 1));
                if (open && rank < a.searchWidth) {
                    parents[rank] = bi[i];
                    bi[i] |= kCagraExpanded;
                }
                got += __popc(m);
            }
            if (threadIdx.x == 0)
                nParents = min(got, a.searchWidth);
        }
        __syncthreads();
        const int np = nParents;
        // nothing left to expand: no later iteration can change itopk, so stopping here equals running on to
        // min_iterations
        if (np == 0)
            break;
        // the visited set is refilled from itopk before it could pass its fill limit
        if (inserted + nGather > a.hashLimit) {
            for (int i = threadIdx.x; i < (1 << a.hashBits); i += blockDim.x)
                hash[i] = kHashEmpty;
            __syncthreads();
            for (int i = threadIdx.x; i < a.itopk; i += blockDim.x)
                if (bi[i] != kCagraInvalid)
                    hash_insert(hash, a.hashBits, bi[i] & ~kCagraExpanded);
            __syncthreads();
            inserted = a.itopk;
        }
        inserted += nGather;
        for (int c = threadIdx.x; c < a.candSize; c += blockDim.x) {
            uint32_t id = kCagraInvalid;
            if (c < np * a.graphDegree) {
                const uint32_t p = parents[c / a.graphDegree];
                const uint32_t nb = __ldg(a.graph + (size_t)p * a.graphDegree + (c % a.graphDegree));
                if (nb < (uint32_t)a.n) // graph entries of -1 (copyFrom) are skipped
                    id = nb;
            }
            ci[c] = id;
            ck[c] = CUDART_INF_F;
        }
        __syncthreads();
        score_candidates<VEC>(a, q, ck, ci, np * a.graphDegree, hash, count);
        __syncthreads();
        cta_bitonic_sort(ck, ci, a.candSize);
        cta_merge_into(bk, bi, a.bufSize, a.itopk, ck, ci, a.candSize);
    }

    for (int i = threadIdx.x; i < a.k; i += blockDim.x) {
        const uint32_t id = bi[i];
        const bool ok = id != kCagraInvalid;
        a.outI[qi * a.k + i] = ok ? (idx_t)(id & ~kCagraExpanded) : (idx_t)-1;
        const float key = bk[i];
        a.outD[qi * a.k + i] = ok ? (a.metric == METRIC_INNER_PRODUCT ? -key : key)
                                  : (a.metric == METRIC_INNER_PRODUCT ? -FLT_MAX : FLT_MAX);
    }
    if (count)
        atomicAdd(&ctaCount, count);
    __syncthreads();
    if (threadIdx.x == 0 && ctaCount)
        atomicAdd(a.distanceCount, ctaCount);
}

} // namespace

size_t cagraSearchSmemBytes(const CagraSearchArgs& a) {
    return sizeof(float) * round_up(a.d, 4) + 8 * (size_t)a.bufSize + 8 * (size_t)a.candSize +
           sizeof(uint32_t) * ((size_t(1) << a.hashBits) + a.searchWidth);
}

void runCagraSearch(const CagraSearchArgs& a, cudaStream_t stream) {
    if (a.nq == 0)
        return;
    const size_t smem = cagraSearchSmemBytes(a);
    auto launch = [&](auto kernel) {
        CUDA_VERIFY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        KernelTiming::begin("cagra_search", stream);
        kernel<<<(unsigned)a.nq, a.blockSize, smem, stream>>>(a);
        CUDA_CHECK_LAST();
        KernelTiming::end("cagra_search", stream);
    };
    const bool vec4 = (a.d & 3) == 0 && (reinterpret_cast<uintptr_t>(a.data) & 15) == 0;
    if (vec4)
        launch(cagra_search_kernel<4>);
    else
        launch(cagra_search_kernel<1>);
}

} // namespace fb200
