// Runs the REFERENCE's own drivers over the faiss_b200 adapter (needs a GPU; built by tests/adapter/build_adapter.py
// where the reference's headers are available, executed by tests/test_adapter_gpu.py):
//   1. index_cpu_to_b200(IndexFlatL2) answers like the CPU index (integer data: identical ids and distances)
//   2. faiss::Clustering::train(n, x, adapter) == faiss::Clustering::train(n, x, IndexFlatL2)  (faiss/Clustering.cpp:254-356)
//   3. faiss::IndexShards over adapter sub-indexes == CPU IndexFlat                              (faiss/IndexShards.cpp:197-264)
//   4. IVFPQ / IVFFlat: CPU-trained index -> index_cpu_to_b200 -> search ~ CPU search; index_b200_to_cpu returns
//      byte-identical inverted lists (testIVFEquality, faiss/gpu/test/TestUtils.h:95-127)
//   5. per-call faiss::SearchParametersIVF through faiss::Index::search
#include <faiss/Clustering.h>
#include <faiss/IndexFlat.h>
#include <faiss/IndexIVFFlat.h>
#include <faiss/IndexIVFPQ.h>
#include <faiss/IndexShards.h>
#include <faiss/invlists/InvertedLists.h>
#include <faiss/utils/random.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "faiss_b200_adapter.h"

using namespace faiss_b200_adapter;
using faiss::idx_t;

static int failures = 0;
#define CHECK(cond, ...)                          \
    do {                                          \
        if (!(cond)) {                            \
            failures++;                           \
            printf("FAIL %s:%d: ", __FILE__, __LINE__); \
            printf(__VA_ARGS__);                  \
            printf("\n");                         \
        }                                         \
    } while (0)

static std::vector<float> rand_int(size_t n, int64_t seed, float scale) {
    std::vector<float> x(n);
    faiss::float_rand(x.data(), n, seed);
    for (auto& v : x)
        v = std::floor(v * scale);
    return x;
}

int main() {
    B200Resources res;
    const int d = 64;

    // ---- 1. Flat clone, integer regime
    {
        const idx_t N = 60000, nq = 50, k = 20;
        auto xb = rand_int(N * d, 1, 16), xq = rand_int(nq * d, 2, 16);
        faiss::IndexFlatL2 cpu(d);
        cpu.add(N, xb.data());
        std::unique_ptr<faiss::Index> gpu(index_cpu_to_b200(&res, 0, &cpu));
        CHECK(gpu->ntotal == N, "ntotal %ld", (long)gpu->ntotal);
        std::vector<float> D0(nq * k), D1(nq * k);
        std::vector<idx_t> I0(nq * k), I1(nq * k);
        cpu.search(nq, xq.data(), k, D0.data(), I0.data());
        gpu->search(nq, xq.data(), k, D1.data(), I1.data());
        CHECK(D0 == D1, "flat distances differ");
        size_t diff = 0;
        for (size_t i = 0; i < I0.size(); i++)
            diff += I0[i] != I1[i];
        // ties at the rank-k boundary may be cut differently by the CPU heap; inside the list (d, id) order is shared
        CHECK(diff <= I0.size() / 50, "flat ids differ in %zu places", diff);
        std::unique_ptr<faiss::Index> back(index_b200_to_cpu(gpu.get()));
        auto* bf = dynamic_cast<faiss::IndexFlat*>(back.get());
        CHECK(bf && bf->ntotal == N && memcmp(bf->get_xb(), xb.data(), sizeof(float) * N * d) == 0, "flat round trip");
        printf("1 flat clone ok (id differences at tie boundaries: %zu)\n", diff);
    }

    // ---- 2. the reference's Clustering driving the adapter
    {
        const idx_t n = 20000;
        const int k = 64;
        std::vector<float> x(n * d);
        faiss::float_rand(x.data(), x.size(), 5);
        faiss::ClusteringParameters cp;
        cp.niter = 6;
        cp.seed = 77;
        faiss::Clustering c0(d, k, cp), c1(d, k, cp);
        faiss::IndexFlatL2 cpu(d);
        B200IndexFlat gpu(&res, d, faiss::METRIC_L2);
        c0.train(n, x.data(), cpu);
        c1.train(n, x.data(), gpu);
        double maxdiff = 0;
        for (size_t i = 0; i < c0.centroids.size(); i++)
            maxdiff = std::max(maxdiff, (double)std::fabs(c0.centroids[i] - c1.centroids[i]));
        CHECK(maxdiff < 1e-3, "clustering centroids differ by %g", maxdiff);
        CHECK(std::fabs(c0.iteration_stats.back().obj - c1.iteration_stats.back().obj) <= 1e-4 * c0.iteration_stats.back().obj, "objective");
        CHECK(gpu.ntotal == k, "index holds the final centroids");
        printf("2 faiss::Clustering over the adapter ok (max centroid diff %.2e)\n", maxdiff);
    }

    // ---- 3. the reference's IndexShards over adapter sub-indexes
    {
        const idx_t N = 80000, nq = 40, k = 10;
        auto xb = rand_int(N * d, 11, 16), xq = rand_int(nq * d, 12, 16);
        B200IndexFlat a(&res, d, faiss::METRIC_L2), b(&res, d, faiss::METRIC_L2);
        faiss::IndexShards shards(d, /*threaded=*/true, /*successive_ids=*/true);
        shards.add_shard(&a);
        shards.add_shard(&b);
        shards.add(N, xb.data());
        CHECK(shards.ntotal == N && a.ntotal == N / 2, "shard sizes");
        faiss::IndexFlatL2 cpu(d);
        cpu.add(N, xb.data());
        std::vector<float> D0(nq * k), D1(nq * k);
        std::vector<idx_t> I0(nq * k), I1(nq * k);
        cpu.search(nq, xq.data(), k, D0.data(), I0.data());
        shards.search(nq, xq.data(), k, D1.data(), I1.data());
        CHECK(D0 == D1, "shards distances differ");
        size_t diff = 0;
        for (size_t i = 0; i < I0.size(); i++)
            diff += I0[i] != I1[i];
        CHECK(diff <= I0.size() / 50, "shards ids differ in %zu places", diff);
        printf("3 faiss::IndexShards over the adapter ok\n");
    }

    // ---- 4. IVF clones
    {
        const idx_t N = 30000, nq = 60, k = 10;
        const size_t nlist = 32, M = 8;
        const int d2 = 32;
        std::vector<float> xb(N * d2), xq(nq * d2);
        faiss::float_rand(xb.data(), xb.size(), 21);
        faiss::float_rand(xq.data(), xq.size(), 22);
        faiss::IndexFlatL2 q1(d2), q2(d2);
        faiss::IndexIVFPQ cpupq(&q1, d2, nlist, M, 8);
        cpupq.cp.niter = 5;
        cpupq.pq.cp.niter = 5;
        cpupq.train(N, xb.data());
        cpupq.add(N, xb.data());
        cpupq.nprobe = 4;
        std::unique_ptr<faiss::Index> gpu(index_cpu_to_b200(&res, 0, &cpupq));
        std::vector<float> D0(nq * k), D1(nq * k);
        std::vector<idx_t> I0(nq * k), I1(nq * k);
        cpupq.search(nq, xq.data(), k, D0.data(), I0.data());
        gpu->search(nq, xq.data(), k, D1.data(), I1.data());
        size_t same = 0;
        double maxrel = 0;
        for (size_t i = 0; i < I0.size(); i++) {
            same += I0[i] == I1[i];
            if (I0[i] == I1[i])
                maxrel = std::max(maxrel, (double)std::fabs(D0[i] - D1[i]) / std::max(1e-20, (double)std::fabs(D0[i])));
        }
        CHECK(same >= I0.size() * 97 / 100, "ivfpq ids equal %zu of %zu", same, I0.size());
        CHECK(maxrel <= 2e-4, "ivfpq distance rel err %g", maxrel);
        // 5. per-call SearchParametersIVF == setting nprobe
        faiss::SearchParametersIVF sp;
        sp.nprobe = 8;
        std::vector<float> D2(nq * k), D3(nq * k);
        std::vector<idx_t> I2(nq * k), I3(nq * k);
        gpu->search(nq, xq.data(), k, D2.data(), I2.data(), &sp);
        dynamic_cast<B200IndexIVF*>(gpu.get())->nprobe = 8;
        gpu->search(nq, xq.data(), k, D3.data(), I3.data());
        CHECK(I2 == I3 && D2 == D3, "SearchParametersIVF override");
        // round trip: byte-identical lists
        std::unique_ptr<faiss::Index> back(index_b200_to_cpu(gpu.get()));
        auto* bpq = dynamic_cast<faiss::IndexIVFPQ*>(back.get());
        CHECK(bpq && bpq->ntotal == N, "ivfpq back ntotal");
        bool eq = bpq != nullptr;
        for (size_t l = 0; l < nlist && eq; l++) {
            eq = bpq->invlists->list_size(l) == cpupq.invlists->list_size(l);
            if (!eq)
                break;
            faiss::InvertedLists::ScopedCodes c0(cpupq.invlists, l), c1(bpq->invlists, l);
            faiss::InvertedLists::ScopedIds i0(cpupq.invlists, l), i1(bpq->invlists, l);
            const size_t n = cpupq.invlists->list_size(l);
            eq = memcmp(c0.get(), c1.get(), n * M) == 0 && memcmp(i0.get(), i1.get(), n * sizeof(idx_t)) == 0;
        }
        CHECK(eq, "ivfpq lists not byte-identical after copyFrom/copyTo");
        // IVFFlat: train + add ON the adapter, compare with the CPU index it clones to
        B200IndexIVFFlat gfl(&res, d2, nlist, faiss::METRIC_L2);
        gfl.train(N, xb.data());
        gfl.add(N, xb.data());
        gfl.nprobe = 4;
        std::unique_ptr<faiss::Index> cfl(index_b200_to_cpu(&gfl));
        dynamic_cast<faiss::IndexIVFFlat*>(cfl.get())->nprobe = 4;
        cfl->search(nq, xq.data(), k, D0.data(), I0.data());
        gfl.search(nq, xq.data(), k, D1.data(), I1.data());
        same = 0;
        for (size_t i = 0; i < I0.size(); i++)
            same += I0[i] == I1[i];
        CHECK(same >= I0.size() * 99 / 100, "ivfflat ids equal %zu of %zu", same, I0.size());
        printf("4/5 IVF clones, SearchParametersIVF, byte-exact round trip ok\n");
    }
    if (failures == 0)
        printf("ADAPTER_OK\n");
    return failures == 0 ? 0 : 1;
}
