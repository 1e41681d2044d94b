// search_and_reconstruct / reconstruct_batch through the faiss_b200 adapter (needs a GPU; built by
// tests/adapter/build_adapter.py where the reference's headers are available, executed by
// tests/test_adapter_gpu.py).  faiss::Index::search_and_reconstruct on adapter clones of IndexFlatL2,
// IndexIVFFlat and IndexIVFPQ whose ids are stored twice with different vectors, against the CPU indexes:
//   * D and I equal the adapter's search;
//   * R is the entry the search scored: one of the CPU's entries under that id, and (exact integer data) its
//     distance to the query is D -- faiss::Index's per-label default would return one fixed entry per id;
//   * D equals the CPU IndexIVF::search_and_reconstruct's row by row;
//   * reconstruct_batch equals the CPU's reconstruct_n (the entry last in (list, offset) order).
#include <faiss/IndexFlat.h>
#include <faiss/IndexIVFFlat.h>
#include <faiss/IndexIVFPQ.h>
#include <faiss/utils/random.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <vector>

#include "faiss_b200_adapter.h"

using namespace faiss_b200_adapter;
using faiss::idx_t;

static int failures = 0;
#define CHECK(cond, ...)                                \
    do {                                                \
        if (!(cond)) {                                  \
            failures++;                                 \
            printf("FAIL %s:%d: ", __FILE__, __LINE__); \
            printf(__VA_ARGS__);                        \
            printf("\n");                               \
        }                                               \
    } while (0)

static std::vector<float> rand_int(size_t n, int64_t seed, float scale) {
    std::vector<float> x(n);
    faiss::float_rand(x.data(), n, seed);
    for (auto& v : x)
        v = std::floor(v * scale);
    return x;
}

// every (id -> decoded entries) of a CPU IVF index, in (list, offset) order
static std::map<idx_t, std::vector<std::vector<float>>> entries(const faiss::IndexIVF& ivf) {
    std::map<idx_t, std::vector<std::vector<float>>> out;
    for (size_t l = 0; l < ivf.nlist; l++) {
        const size_t len = ivf.invlists->list_size(l);
        const idx_t* ids = ivf.invlists->get_ids(l);
        for (size_t off = 0; off < len; off++) {
            std::vector<float> v(ivf.d);
            ivf.reconstruct_from_offset(l, off, v.data());
            out[ids[off]].push_back(v);
        }
        ivf.invlists->release_ids(l, ids);
    }
    return out;
}

static bool sameBits(const float* a, const float* b, int d) {
    return std::memcmp(a, b, sizeof(float) * d) == 0;
}

static void checkIvf(const char* what, const faiss::IndexIVF& cpu, B200IndexIVF& gpu, const std::vector<float>& xq, int nq,
                     int k, bool exactDistances) {
    const int d = cpu.d;
    std::vector<float> D0(nq * k), D(nq * k), R((size_t)nq * k * d), Dc(nq * k), Rc((size_t)nq * k * d);
    std::vector<idx_t> I0(nq * k), I(nq * k), Ic(nq * k);
    gpu.search(nq, xq.data(), k, D0.data(), I0.data());
    faiss::Index& base = gpu; // through the faiss::Index virtual
    base.search_and_reconstruct(nq, xq.data(), k, D.data(), I.data(), R.data());
    CHECK(D == D0 && I == I0, "%s: search_and_reconstruct D / I differ from search", what);
    auto all = entries(cpu);
    int notStored = 0, wrongDistance = 0, dupHits = 0;
    for (int q = 0; q < nq; q++)
        for (int j = 0; j < k; j++) {
            const idx_t id = I[q * k + j];
            const float* r = R.data() + ((size_t)q * k + j) * d;
            if (id < 0)
                continue;
            const auto& cands = all[id];
            dupHits += cands.size() > 1;
            bool found = false;
            for (const auto& v : cands)
                found |= sameBits(r, v.data(), d);
            notStored += !found;
            if (exactDistances) {
                double s = 0;
                for (int i = 0; i < d; i++)
                    s += ((double)xq[q * d + i] - r[i]) * ((double)xq[q * d + i] - r[i]);
                wrongDistance += (float)s != D[q * k + j];
            }
        }
    CHECK(notStored == 0, "%s: %d results are not a stored entry of their id", what, notStored);
    CHECK(wrongDistance == 0, "%s: %d reconstructions are not the scored entry", what, wrongDistance);
    CHECK(dupHits > 0, "%s: no result hit a duplicated id (the test data must exercise them)", what);
    if (exactDistances) {
        faiss::SearchParametersIVF p;
        p.nprobe = gpu.nprobe;
        cpu.search_and_reconstruct(nq, xq.data(), k, Dc.data(), Ic.data(), Rc.data(), &p);
        CHECK(Dc == D, "%s: distances differ from the CPU IndexIVF::search_and_reconstruct", what);
    }
    // reconstruct_batch == the CPU's reconstruct_n rows (last in (list, offset) order)
    std::vector<idx_t> keys;
    for (auto& kv : all)
        if (keys.size() < 300)
            keys.push_back(kv.first);
    std::vector<float> rb(keys.size() * d), want(keys.size() * d);
    base.reconstruct_batch((idx_t)keys.size(), keys.data(), rb.data());
    for (size_t i = 0; i < keys.size(); i++)
        std::memcpy(want.data() + i * d, all[keys[i]].back().data(), sizeof(float) * d);
    CHECK(rb == want, "%s: reconstruct_batch differs from the last entry in (list, offset) order", what);
    printf("%s: ok (%d results on duplicated ids)\n", what, dupHits);
}

int main() {
    B200Resources res;
    const int nb = 4000, dup = 600, nq = 64, k = 20;
    // ids: 0 .. nb-dup-1 once, then the first `dup` ids again with other vectors
    std::vector<idx_t> ids(nb);
    for (int i = 0; i < nb; i++)
        ids[i] = i < nb - dup ? i : i - (nb - dup);
    {
        const int d = 16, nlist = 32;
        auto xb = rand_int((size_t)nb * d, 1, 8.f);
        auto xq = rand_int((size_t)nq * d, 2, 8.f);
        faiss::IndexFlatL2 q(d);
        faiss::IndexIVFFlat cpu(&q, d, nlist);
        cpu.cp.niter = 5;
        cpu.train(nb, xb.data());
        cpu.add_with_ids(nb, xb.data(), ids.data());
        cpu.nprobe = 8;
        std::unique_ptr<faiss::Index> g(index_cpu_to_b200(&res, 0, &cpu));
        auto* gpu = dynamic_cast<B200IndexIVF*>(g.get());
        CHECK(gpu != nullptr, "IVFFlat clone is not a B200IndexIVF");
        gpu->nprobe = 8;
        checkIvf("IVFFlat", cpu, *gpu, xq, nq, k, true);
    }
    {
        const int d = 32, nlist = 16;
        auto xb = rand_int((size_t)nb * d, 3, 8.f);
        auto xq = rand_int((size_t)nq * d, 4, 8.f);
        faiss::IndexFlatL2 q(d);
        faiss::IndexIVFPQ cpu(&q, d, nlist, 8, 8);
        cpu.cp.niter = 5;
        cpu.pq.cp.niter = 5;
        cpu.train(nb, xb.data());
        cpu.add_with_ids(nb, xb.data(), ids.data());
        std::unique_ptr<faiss::Index> g(index_cpu_to_b200(&res, 0, &cpu));
        auto* gpu = dynamic_cast<B200IndexIVF*>(g.get());
        CHECK(gpu != nullptr, "IVFPQ clone is not a B200IndexIVF");
        gpu->nprobe = 6;
        checkIvf("IVFPQ", cpu, *gpu, xq, nq, k, false);
    }
    {
        const int d = 24;
        auto xb = rand_int((size_t)nb * d, 5, 8.f);
        auto xq = rand_int((size_t)nq * d, 6, 8.f);
        faiss::IndexFlatL2 cpu(d);
        cpu.add(nb, xb.data());
        std::unique_ptr<faiss::Index> g(index_cpu_to_b200(&res, 0, &cpu));
        std::vector<float> D(nq * k), R((size_t)nq * k * d), Dc(nq * k), Rc((size_t)nq * k * d);
        std::vector<idx_t> I(nq * k), Ic(nq * k);
        g->search_and_reconstruct(nq, xq.data(), k, D.data(), I.data(), R.data());
        cpu.search_and_reconstruct(nq, xq.data(), k, Dc.data(), Ic.data(), Rc.data());
        CHECK(D == Dc, "Flat: distances differ from the CPU");
        int bad = 0;
        for (int e = 0; e < nq * k; e++)
            bad += !sameBits(R.data() + (size_t)e * d, xb.data() + (size_t)I[e] * d, d);
        CHECK(bad == 0, "Flat: %d reconstructions are not the returned row", bad);
        printf("Flat: ok\n");
    }
    if (failures == 0)
        printf("ADAPTER_RECONS_OK\n");
    return failures == 0 ? 0 : 1;
}
