// Filtered search through the faiss_b200 adapter (needs a GPU; built by tests/adapter/build_adapter.py where the
// reference's headers are available, executed by tests/test_adapter_gpu.py).  faiss::Index::search(..., params)
// with the reference's own IDSelectorRange / IDSelectorBatch / IDSelectorNot / IDSelectorAnd, a user IDSelector
// subclass (the callback path), on an adapter
// clone of IndexFlatL2 and of IndexIVFFlat (add_with_ids ids with negative and >= 2^40 values), compared with the
// CPU index searched with the same parameters.
#include <faiss/IndexFlat.h>
#include <faiss/IndexIVFFlat.h>
#include <faiss/impl/IDSelector.h>
#include <faiss/utils/random.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "faiss_b200_adapter.h"

using namespace faiss_b200_adapter;
using faiss::idx_t;

static int failures = 0;
#define CHECK(cond, ...)                                        \
    do {                                                        \
        if (!(cond)) {                                          \
            failures++;                                         \
            printf("FAIL %s:%d: ", __FILE__, __LINE__);         \
            printf(__VA_ARGS__);                                \
            printf("\n");                                       \
        }                                                       \
    } while (0)

// a selector the library cannot see into
struct Mod7Selector : faiss::IDSelector {
    bool is_member(idx_t id) const override {
        return ((id % 7) + 7) % 7 == 3;
    }
};

static std::vector<float> rand_int(size_t n, int64_t seed, float scale) {
    std::vector<float> x(n);
    faiss::float_rand(x.data(), n, seed);
    for (auto& v : x)
        v = std::floor(v * scale);
    return x;
}

// the same distances row by row, and every returned id selected
static void compare(const char* what, const faiss::IDSelector& sel, int nq, int k, const std::vector<float>& D0,
                    const std::vector<idx_t>& I0, const std::vector<float>& D1, const std::vector<idx_t>& I1, bool sameIds) {
    int bad = 0, unselected = 0;
    for (int q = 0; q < nq; q++) {
        std::vector<float> a(D0.begin() + q * k, D0.begin() + (q + 1) * k), b(D1.begin() + q * k, D1.begin() + (q + 1) * k);
        std::sort(a.begin(), a.end());
        std::sort(b.begin(), b.end());
        bad += a != b;
        for (int j = 0; j < k; j++) {
            const idx_t id = I1[q * k + j];
            if (D1[q * k + j] < 1e30f && !sel.is_member(id))
                unselected++;
            if (sameIds && id != I0[q * k + j])
                bad++;
        }
    }
    CHECK(bad == 0 && unselected == 0, "%s: %d rows differ from the CPU index, %d unselected ids", what, bad, unselected);
    printf("%s: ok\n", what);
}

int main() {
    B200Resources res;
    const int d = 64;
    const int nq = 50, k = 20;
    auto xq = rand_int(nq * d, 2, 16);

    // ---- Flat (50 queries: the tensor-core path), integer data: identical ids and distances
    {
        const idx_t N = 40000;
        auto xb = rand_int(N * d, 1, 16);
        faiss::IndexFlatL2 cpu(d);
        cpu.add(N, xb.data());
        std::unique_ptr<faiss::Index> gpu(index_cpu_to_b200(&res, 0, &cpu));
        std::vector<idx_t> batch;
        for (idx_t i = 1; i < N; i += 5)
            batch.push_back(i);
        faiss::IDSelectorRange range(N / 5, N * 4 / 5);
        faiss::IDSelectorBatch bsel(batch.size(), batch.data());
        faiss::IDSelectorNot nsel(&range);
        Mod7Selector mod7;
        faiss::IDSelectorAnd both(&range, &mod7);
        const std::pair<const char*, const faiss::IDSelector*> sels[] = {
                {"flat Range", &range}, {"flat Batch", &bsel}, {"flat Not", &nsel}, {"flat callback", &mod7},
                {"flat And(Range, callback)", &both}};
        for (auto& s : sels) {
            faiss::SearchParameters p;
            p.sel = const_cast<faiss::IDSelector*>(s.second);
            std::vector<float> D0(nq * k), D1(nq * k);
            std::vector<idx_t> I0(nq * k), I1(nq * k);
            cpu.search(nq, xq.data(), k, D0.data(), I0.data(), &p);
            gpu->search(nq, xq.data(), k, D1.data(), I1.data(), &p);
            compare(s.first, *s.second, nq, k, D0, I0, D1, I1, true);
        }
    }

    // ---- IVF-Flat with add_with_ids ids (negative, >= 2^40), per-call nprobe
    {
        const idx_t N = 30000;
        const size_t nlist = 64;
        auto xb = rand_int(N * d, 3, 16);
        std::vector<idx_t> ids(N);
        for (idx_t i = 0; i < N; i++)
            ids[i] = i % 7 == 0 ? (idx_t(1) << 40) + i : i % 11 == 3 ? -i - 2 : i;
        faiss::IndexFlatL2 q(d);
        faiss::IndexIVFFlat cpu(&q, d, nlist);
        cpu.cp.niter = 4;
        cpu.train(N, xb.data());
        cpu.add_with_ids(N, xb.data(), ids.data());
        std::unique_ptr<faiss::Index> gpu(index_cpu_to_b200(&res, 0, &cpu));
        std::vector<idx_t> batch;
        for (idx_t i = 0; i < N; i += 10)
            batch.push_back(ids[i]);
        faiss::IDSelectorRange range(-10000, 20000);
        faiss::IDSelectorBatch bsel(batch.size(), batch.data());
        faiss::IDSelectorNot nsel(&range);
        Mod7Selector mod7;
        const std::pair<const char*, const faiss::IDSelector*> sels[] = {
                {"ivf Range", &range}, {"ivf Batch", &bsel}, {"ivf Not", &nsel}, {"ivf callback", &mod7}};
        for (auto& s : sels) {
            faiss::SearchParametersIVF p;
            p.sel = const_cast<faiss::IDSelector*>(s.second);
            p.nprobe = 8;
            std::vector<float> D0(nq * k), D1(nq * k);
            std::vector<idx_t> I0(nq * k), I1(nq * k);
            cpu.search(nq, xq.data(), k, D0.data(), I0.data(), &p);
            gpu->search(nq, xq.data(), k, D1.data(), I1.data(), &p);
            compare(s.first, *s.second, nq, k, D0, I0, D1, I1, false);
        }
    }
    if (failures == 0)
        printf("ADAPTER_SEL_OK\n");
    return failures == 0 ? 0 : 1;
}
