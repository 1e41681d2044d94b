// TEST DRIVER: the reference's LocalSearchQuantizer with B200IcmEncoderFactory as its icm_encoder_factory, against the
// same quantizer with the CPU encoder (faiss/impl/LocalSearchQuantizer.cpp).  Built by
// tests/adapter/build_adapter_lsq.py, run by tests/test_adapter_lsq_gpu.py; prints ADAPTER_LSQ_OK on success.
//   1. integer codebooks and vectors (every fp32 sum exact): compute_codes gives the CPU's codes byte for byte, over
//      several chunks, and icm_encode leaves the caller's std::mt19937 where the CPU leaves it (its next output);
//   2. LocalSearchQuantizer::train through the factory reaches an encode error within 1.05x of the CPU-trained one.
#include <faiss/impl/LocalSearchQuantizer.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "faiss_b200_adapter.h"

using faiss::LocalSearchQuantizer;
using faiss_b200_adapter::B200IcmEncoderFactory;

static int g_fail = 0;
#define CHECK(c)                                                   \
    do {                                                           \
        if (!(c)) {                                                \
            printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c);    \
            g_fail++;                                              \
        }                                                          \
    } while (0)

static std::vector<float> int_values(std::mt19937& rs, size_t count) {
    std::uniform_int_distribution<int> v(-8, 8);
    std::vector<float> out(count);
    for (auto& f : out)
        f = (float)v(rs);
    return out;
}

// faiss.contrib.datasets.SyntheticDataset's shape of data: a 10-dim ellipsoid bent by sin into d dimensions
static std::vector<float> synthetic(size_t n, size_t d, unsigned seed) {
    std::mt19937 rs(seed);
    std::normal_distribution<double> nd;
    std::uniform_real_distribution<double> ud;
    std::vector<double> proj(10 * d), scale(d);
    for (auto& p : proj)
        p = ud(rs);
    for (auto& s : scale)
        s = ud(rs) * 4 + 0.1;
    std::vector<float> x(n * d);
    for (size_t i = 0; i < n; i++) {
        double z[10];
        for (auto& v : z)
            v = nd(rs);
        for (size_t j = 0; j < d; j++) {
            double a = 0;
            for (int t = 0; t < 10; t++)
                a += z[t] * proj[t * d + j];
            x[i * d + j] = (float)std::sin(a * scale[j]);
        }
    }
    return x;
}

static double encode_error(const LocalSearchQuantizer& q, const std::vector<float>& x, size_t n) {
    std::vector<uint8_t> codes(q.code_size * n);
    q.compute_codes(x.data(), codes.data(), n);
    std::vector<float> dec(n * q.d);
    q.decode(codes.data(), dec.data(), n);
    double err = 0;
    for (size_t i = 0; i < n * q.d; i++)
        err += double(x[i] - dec[i]) * double(x[i] - dec[i]);
    return err;
}

int main() {
    // 1. integer data: codes byte for byte, generator state
    for (auto [M, nbits, d] : {std::tuple<int, int, int>{4, 4, 32}, {8, 8, 64}, {3, 10, 20}}) {
        const size_t n = 1000;
        std::mt19937 rs(M * 100 + nbits);
        LocalSearchQuantizer cpu(d, M, nbits), gpu(d, M, nbits);
        auto cb = int_values(rs, cpu.M * cpu.K * cpu.d); // the constructor leaves codebooks empty
        auto x = int_values(rs, n * d);
        for (auto* q : {&cpu, &gpu}) {
            q->codebooks = cb;
            q->is_trained = true;
            q->chunk_size = 300; // four chunks: the draws are made chunk by chunk
            q->encode_ils_iters = 6;
            q->nperts = std::min(4, M); // the CPU requires nperts <= M
        }
        gpu.icm_encoder_factory = new B200IcmEncoderFactory(1); // owned and deleted by gpu
        std::vector<uint8_t> cc(cpu.code_size * n), gc(gpu.code_size * n);
        cpu.compute_codes(x.data(), cc.data(), n);
        gpu.compute_codes(x.data(), gc.data(), n);
        CHECK(cc == gc);
        std::vector<int32_t> c0(n * M);
        std::uniform_int_distribution<int32_t> kd(0, cpu.K - 1);
        for (auto& c : c0)
            c = kd(rs);
        auto c1 = c0, c2 = c0;
        std::mt19937 g1(2024), g2(2024);
        cpu.icm_encode(c1.data(), x.data(), n, 5, g1);
        gpu.icm_encode(c2.data(), x.data(), n, 5, g2);
        CHECK(c1 == c2);
        CHECK(g1() == g2());
        printf("integer M=%d nbits=%d d=%d: codes %s\n", M, nbits, d, cc == gc && c1 == c2 ? "identical" : "DIFFER");
    }

    // 2. train through the factory (float data)
    {
        const size_t d = 32, nt = 2000, nb = 2000;
        auto xt = synthetic(nt, d, 1);
        auto xb = synthetic(nb, d, 2);
        LocalSearchQuantizer cpu(d, 4, 8), gpu(d, 4, 8);
        for (auto* q : {&cpu, &gpu})
            q->train_iters = 8;
        gpu.icm_encoder_factory = new B200IcmEncoderFactory(1);
        cpu.train(nt, xt.data());
        gpu.train(nt, xt.data());
        const double ec = encode_error(cpu, xb, nb), eg = encode_error(gpu, xb, nb);
        printf("train: encode error cpu %.4f gpu %.4f ratio %.5f\n", ec, eg, eg / ec);
        CHECK(eg <= 1.05 * ec);
    }

    if (g_fail == 0)
        printf("ADAPTER_LSQ_OK\n");
    return g_fail == 0 ? 0 : 1;
}
