// faiss_b200 -- the schedule of a tensor-core Flat search (flat_tc.cu): everything it decides before it launches.
//
// Pure host arithmetic without CUDA includes, so that a host compiler can build it on its own and the schedule can
// be checked without a GPU.  The launch side (flat_tc.cu) takes the schedule as it is and never recomputes it.
#pragma once

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <numeric>
#include <vector>

namespace fb200 {
namespace tc {

constexpr int kUnitM = 128;  // queries per work unit (the query tile of flat_tc_kernel)
constexpr int kTileN = 256;  // database rows per tile (wgmma N)
constexpr int kParts = 4;    // column parts of a tile per query row (lanes of a quad)
constexpr int kSegsPerUnit = kUnitM * kParts; // candidate segments of a work unit
// threshold selection by bisection holds this many candidates per query and round (tc_select_bisect_kernel)
constexpr int kSelCap = 1536;

// one round of the geometric schedule: positions [begin, end) of the permuted tile order, split into `slices`
// slices of `tilesPerSlice` tiles; `cap` candidates per segment
struct FlatTcRound {
    int begin, end, slices, tilesPerSlice, cap;
};

// the rounds of one query batch and the scratch they need
struct FlatTcRounds {
    std::vector<FlatTcRound> rounds;
    size_t arenaBytes = 0; // candidate arena: (score bits, row) pairs of 8 bytes
    size_t countBytes = 0; // one int count per segment
};

inline int64_t tcCeilDiv(int64_t a, int64_t b) {
    return (a + b - 1) / b;
}

inline int tcNextPow2(int v) {
    int p = 1;
    while (p < v)
        p <<= 1;
    return p;
}

struct FlatTcSchedule {
    int k, sms;
    int nShards;      // ranks of a sharded search, 1 otherwise
    int kFrac;        // ceil(k / nShards): the rows a shard must vouch for
    int LIST;         // base-list entries per query
    int KL;           // re-rank list size (pow2 >= k, >= 64)
    bool useBisect;   // threshold selection by bisection (fp16: LIST <= 256; int8: k <= 128), else sorted base lists
    bool streaming;   // k = 1 without sharding: one pass with self-tightening thresholds and a fused finish
    int64_t T;        // this database's tiles
    int64_t Tsched;   // tiles the rounds are laid out over (the largest shard's in a sharded search)
    int r0Tiles;      // tiles of the first round
    int64_t qBatch;   // queries per batch
    unsigned long long permA, permB; // tile permutation: position p -> tile (p * permA + permB) % T

    // the geometric rounds of a batch of qPairs query units over the permuted tile order
    FlatTcRounds rounds(int64_t qPairs) const {
        FlatTcRounds out;
        const double g = nShards > 1 ? std::max(4.0, std::min(8.0, 2.0 * nShards)) : 4.0; // growth per round
        int64_t seen = 0;
        while (seen < Tsched) {
            int64_t end = seen == 0 ? std::min<int64_t>(Tsched, r0Tiles) : std::min<int64_t>(Tsched, (int64_t)(seen * g));
            if (Tsched - end < end / 4)
                end = Tsched; // do not leave a sliver for an extra round
            if (streaming)
                end = Tsched; // k = 1: ONE pass, thresholds tighten themselves inside the kernel
            int64_t tiles = end - seen;
            // choose the slice count minimising (waves x tiles per slice)
            int bestS = 1;
            double bestCost = 1e300;
            int64_t maxS = std::max<int64_t>(1, std::min<int64_t>(512, tiles / 8));
            for (int64_t S = 1; S <= maxS; S++) {
                int64_t tps = tcCeilDiv(tiles, S);
                int64_t units = qPairs * tcCeilDiv(tiles, tps);
                int64_t waves = tcCeilDiv(units, sms);
                double cost = (double)waves * (double)(tps + 6); // +6: per-unit fixed overhead
                if (cost < bestCost * 0.999) {
                    bestCost = cost;
                    bestS = (int)S;
                }
            }
            int64_t tps = tcCeilDiv(tiles, bestS);
            int S = (int)tcCeilDiv(tiles, tps);
            int cap;
            if (streaming) {
                // a thread emits ~ln(columns it sees) running maxima plus the near-ties of the maximum
                cap = 64;
            } else if (seen == 0) {
                cap = (int)(tps * (kTileN / kParts)); // everything passes in round 0
            } else {
                double expect = 1.5 * k * ((double)tps / (double)seen) / kParts;
                cap = tcNextPow2((int)std::min<double>(1 << 20, 4.0 * expect + 32.0));
                cap = std::max(cap, 32);
            }
            out.rounds.push_back({(int)seen, (int)end, S, (int)tps, cap});
            const size_t segs = (size_t)qPairs * S * kSegsPerUnit;
            out.arenaBytes = std::max(out.arenaBytes, segs * (size_t)cap * 8);
            out.countBytes = std::max(out.countBytes, segs * sizeof(int));
            seen = end;
        }
        return out;
    }
};

// n database rows, k results per query, sms SMs.  shardRanks = 0: a plain search; otherwise a sharded search over
// shardRanks ranks whose largest shard holds shardMaxTiles tiles.  int8: the scores come from the int8 tensor cores,
// whose certificate margin is about twice the fp16 one: more entries lie within 2 eps of the k-th best, so the base list
// holds 4k entries instead of 2k.
inline FlatTcSchedule planFlatTcSchedule(int64_t n, int k, int sms, int shardRanks = 0, int64_t shardMaxTiles = 0,
                                         bool int8 = false) {
    FlatTcSchedule s;
    s.k = k;
    s.sms = sms;
    s.T = tcCeilDiv(n, kTileN);
    // Sharded search: every rank runs the SAME number of rounds (one all-reduce per round), so the schedule
    // is laid out over the largest shard's tile count and clamped to this shard's.  Thresholds are pooled
    // across ranks after every round, i.e. a round over t local tiles is worth S*t tiles of evidence: the first
    // round shrinks by S and the rounds grow faster (fewer launches for a 1/S-size shard).
    const bool sharded = shardRanks > 0;
    s.nShards = sharded ? shardRanks : 1;
    s.Tsched = sharded ? std::max<int64_t>(s.T, shardMaxTiles) : s.T;
    s.kFrac = (k + s.nShards - 1) / s.nShards;
    s.LIST = std::max(128, tcNextPow2((int8 ? 4 : 2) * k));
    s.KL = std::max(64, tcNextPow2(k));

    // tile permutation: multiplicative hash with a multiplier coprime to T
    unsigned long long A = (unsigned long long)((double)s.T * 0.6180339887498949);
    if (A < 1)
        A = 1;
    while (std::gcd(A, (unsigned long long)s.T) != 1)
        A++;
    s.permA = A;
    s.permB = (unsigned long long)(s.T / 3);

    // first round: ~40 k rows (16 tiles at k = 100).  Every score of round 0 becomes a candidate, so a
    // fixed 16 tiles would make small-k searches (k-means assignment: k = 1, millions of queries) pay 4096
    // candidates per query for nothing.
    int r0Tiles = std::max(std::max(1, (40 * k + kTileN - 1) / kTileN), (k + 127) / 128 * 2);
    if (s.nShards > 1) // pooled evidence: nShards * r0Tiles tiles; a shard must still be able to vouch for kFrac rows
        r0Tiles = std::max<int>((r0Tiles + s.nShards - 1) / s.nShards, std::max(2, (2 * s.kFrac + kTileN - 1) / kTileN));
    // threshold selection by bisection (no sorted lists) holds kSelCap entries per query and round: the all-pass first
    // round is sized to 3/4 of that
    s.useBisect = int8 ? k <= 128 : s.LIST <= 256;
    if (s.useBisect)
        r0Tiles = std::min(r0Tiles, std::max(2, kSelCap * 3 / 4 / kTileN));
    s.r0Tiles = r0Tiles;
    // queries per pass: bounds the candidate arena, whose largest user is the all-pass round 0
    // (2 KB per query and tile) -- 16384 queries at k = 100, up to 131072 for small k
    // k = 1 (k-means assignment, the coarse quantiser of an add): streaming mode -- one pass over all tiles with
    // self-tightening per-thread thresholds (flat_tc_kernel SELF) and a fused select + exact re-rank
    // (tc_argmin_finish_kernel); no rounds, no all-pass first round, no per-query sorted lists.
    s.streaming = k == 1 && !sharded;
    // streaming: a batch is a whole number of waves of the persistent grid (one 128-query unit per CTA and wave)
    // (large k: the all-pass round covers 40 k rows, so the floor drops to keep the arena near 1 GiB)
    const int64_t kQFloor = r0Tiles > 64 ? 2048 : 16384;
    s.qBatch = s.streaming ? (int64_t)sms * kUnitM * 4
                           : std::min<int64_t>(131072, std::max<int64_t>(kQFloor, (int64_t)262144 / r0Tiles));
    return s;
}

} // namespace tc
} // namespace fb200
