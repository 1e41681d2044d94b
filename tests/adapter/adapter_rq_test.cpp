// TEST DRIVER: the reference's ResidualQuantizer through the adapter, against the same quantizer on the CPU
// (faiss/impl/ResidualQuantizer.cpp).  Built by tests/adapter/build_adapter_rq.py, run by tests/test_adapter_rq_gpu.py;
// prints ADAPTER_RQ_OK on success.
//   1. integer codebooks and vectors (every fp32 sum exact): B200ResidualQuantizer::compute_codes gives the CPU's bytes
//      in both modes, for the search types the device packs and for two the adapter packs on the host, with and
//      without centroids;
//   2. the reference's TestGpuResidualQuantizer check with B200ProgressiveDimIndexFactory as a plain
//      ResidualQuantizer's assign_index_factory: ncall grows in train and again in compute_codes, and the encode error
//      is within 0.9x - 1.1x of the CPU-trained quantizer's;
//   3. a B200ResidualQuantizer trained through the factory (with Train_refine_codebook, whose compute_codes runs on the
//      device) encodes within 1e-3 of the CPU encoder's error with the same codebooks, in both modes.
#include <faiss/impl/ResidualQuantizer.h>

#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "faiss_b200_adapter.h"

using faiss::AdditiveQuantizer;
using faiss::ResidualQuantizer;
using faiss_b200_adapter::B200ProgressiveDimIndexFactory;
using faiss_b200_adapter::B200Resources;
using faiss_b200_adapter::B200ResidualQuantizer;

static int g_fail = 0;
#define CHECK(c)                                                \
    do {                                                        \
        if (!(c)) {                                             \
            printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); \
            g_fail++;                                           \
        }                                                       \
    } while (0)

static std::vector<float> int_values(std::mt19937& rs, size_t count, int lim) {
    std::uniform_int_distribution<int> v(-lim, lim);
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

static double encode_error(const ResidualQuantizer& q, const std::vector<float>& x, size_t n) {
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
    B200Resources res;

    // 1. integer data: the CPU's bytes
    struct Shape {
        size_t d;
        std::vector<size_t> nbits;
        int beam;
    };
    for (const Shape& s : {Shape{32, {6, 6, 6, 6}, 5}, Shape{24, {4, 8, 5}, 16}}) {
        const size_t n = 300;
        std::mt19937 rs(s.d);
        size_t tk = 0;
        for (auto b : s.nbits)
            tk += size_t(1) << b;
        auto cb = int_values(rs, tk * s.d, 8);
        auto x = int_values(rs, n * s.d, 16);
        auto cent = int_values(rs, n * s.d, 3);
        std::vector<float> norms(n);
        for (size_t i = 0; i < n; i++)
            norms[i] = (float)(200 + 5 * i);
        int same = 0, total = 0;
        for (int st : {0, 1, 2, 3, 4, 5, 6, 7}) {
            auto type = (AdditiveQuantizer::Search_type_t)st;
            for (int lut : {0, 1}) {
                ResidualQuantizer cpu(s.d, s.nbits, type);
                B200ResidualQuantizer gpu(&res, s.d, s.nbits, type);
                for (ResidualQuantizer* q : {&cpu, (ResidualQuantizer*)&gpu}) {
                    q->codebooks = cb;
                    q->is_trained = true;
                    q->compute_codebook_tables();
                    q->max_beam_size = s.beam;
                    q->use_beam_LUT = lut;
                    q->train_norm(n, norms.data()); // norm_min / norm_max, and the qnorm table of the cqint types
                }
                for (const float* c : {(const float*)nullptr, (const float*)cent.data()}) {
                    std::vector<uint8_t> cc(cpu.code_size * n), gc(gpu.code_size * n);
                    cpu.compute_codes_add_centroids(x.data(), cc.data(), n, c);
                    gpu.compute_codes_add_centroids(x.data(), gc.data(), n, c);
                    CHECK(cc == gc);
                    same += cc == gc;
                    total++;
                }
            }
        }
        printf("integer d=%zu M=%zu beam=%d: %d / %d (search type, mode, centroids) identical\n", s.d, s.nbits.size(),
               s.beam, same, total);
    }

    // 2. TestGpuResidualQuantizer.TestNcall with the factory
    {
        const size_t d = 32, nt = 3000, nb = 1000;
        std::mt19937 rs(100);
        std::uniform_real_distribution<float> u;
        std::vector<float> xt(nt * d), xb(nb * d);
        for (auto& v : xt)
            v = u(rs);
        for (auto& v : xb)
            v = u(rs);
        ResidualQuantizer rq0(d, 4, 6), rq1(d, 4, 6);
        rq0.train(nt, xt.data());
        const double err0 = encode_error(rq0, xb, nb);
        B200ProgressiveDimIndexFactory fac(0);
        rq1.assign_index_factory = &fac;
        rq1.train(nt, xt.data());
        const int ncall_train = fac.ncall;
        CHECK(ncall_train > 0);
        const double err1 = encode_error(rq1, xb, nb);
        CHECK(fac.ncall > ncall_train);
        printf("factory: ncall train %d, after compute_codes %d; error cpu %.4f factory %.4f ratio %.4f\n", ncall_train,
               fac.ncall, err0, err1, err1 / err0);
        CHECK(0.9 * err0 < err1 && err1 < 1.1 * err0);
        rq1.assign_index_factory = nullptr;
    }

    // 3. B200ResidualQuantizer trained through the factory, against the CPU encoder on its codebooks
    {
        const size_t d = 32, nt = 4000, nb = 2000;
        auto xt = synthetic(nt, d, 1);
        auto xb = synthetic(nb, d, 2);
        B200ProgressiveDimIndexFactory fac(0);
        B200ResidualQuantizer gpu(&res, d, 4, 8);
        gpu.assign_index_factory = &fac;
        gpu.train_type = ResidualQuantizer::Train_progressive_dim | ResidualQuantizer::Train_refine_codebook;
        gpu.cp.niter = 10;
        gpu.train(nt, xt.data());
        gpu.assign_index_factory = nullptr;
        CHECK(fac.ncall > 0);
        for (int lut : {0, 1}) {
            ResidualQuantizer cpu(d, 4, 8);
            cpu.codebooks = gpu.codebooks;
            cpu.is_trained = true;
            cpu.compute_codebook_tables();
            cpu.use_beam_LUT = gpu.use_beam_LUT = lut;
            const double ec = encode_error(cpu, xb, nb), eg = encode_error(gpu, xb, nb);
            printf("trained through the factory, use_beam_LUT=%d: encode error cpu %.5f device %.5f\n", lut, ec, eg);
            CHECK(std::fabs(eg - ec) <= 1e-3 * ec);
        }
    }

    if (g_fail == 0)
        printf("ADAPTER_RQ_OK\n");
    return g_fail == 0 ? 0 : 1;
}
