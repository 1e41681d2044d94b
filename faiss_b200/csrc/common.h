// faiss_b200 -- common host-side definitions: error model, ids, metric enum.
//
// Error convention mirrors the reference: user errors throw a FaissException-like C++
// exception (faiss/impl/FaissAssert.h:71-100, FaissException.h:21-40) which the C ABI turns
// into an int status + thread-local message (c_api/error_c.h:19-35, c_api/macros_impl.h:22-36).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <exception>
#include <stdexcept>
#include <string>
#include <type_traits>

namespace fb200 {

using idx_t = int64_t; // faiss/MetricType.h:52

// faiss/MetricType.h:29-49 (same values).  Every index takes L2 and inner product; GpuIndexFlat and bfKnn also take
// the others, which run on the exact SIMT kernel.  METRIC_NaNEuclidean is declared but not implemented.
enum MetricType : int {
    METRIC_INNER_PRODUCT = 0,
    METRIC_L2 = 1,
    METRIC_L1 = 2,
    METRIC_Linf = 3,
    METRIC_Lp = 4, // sum |a-b|^p, p = metric_arg, no root
    METRIC_Canberra = 20,
    METRIC_BrayCurtis = 21,
    METRIC_JensenShannon = 22,
    METRIC_Jaccard = 23,
    METRIC_NaNEuclidean = 24,
    METRIC_GOWER = 25,
};

// faiss/MetricType.h:56-58: larger is better for these two; every other metric is a distance
inline bool is_similarity_metric(MetricType m) {
    return m == METRIC_INNER_PRODUCT || m == METRIC_Jaccard;
}

// the metrics the exact kernel implements (all of the above but METRIC_NaNEuclidean)
inline bool is_implemented_metric(MetricType m) {
    switch (m) {
        case METRIC_INNER_PRODUCT:
        case METRIC_L2:
        case METRIC_L1:
        case METRIC_Linf:
        case METRIC_Lp:
        case METRIC_Canberra:
        case METRIC_BrayCurtis:
        case METRIC_JensenShannon:
        case METRIC_Jaccard:
        case METRIC_GOWER:
            return true;
        default:
            return false;
    }
}

// limits preserved from the reference (faiss/gpu/utils/DeviceDefs.cuh:61-68, impl/IndexUtils.cu:21-43)
constexpr int kMaxK = 2048;
constexpr int kMaxNprobe = 2048;

class FaissException : public std::exception {
   public:
    explicit FaissException(const std::string& m) : msg(m) {}
    FaissException(const std::string& m, const char* func, const char* file, int line) {
        char buf[512];
        snprintf(buf, sizeof(buf), "Error in %s at %s:%d: ", func, file, line);
        msg = std::string(buf) + m;
    }
    const char* what() const noexcept override {
        return msg.c_str();
    }
    std::string msg;
};

#define FB_THROW_MSG(MSG) throw ::fb200::FaissException(MSG, __PRETTY_FUNCTION__, __FILE__, __LINE__)

#define FB_THROW_FMT(FMT, ...)                              \
    do {                                                    \
        char __buf[1024];                                   \
        snprintf(__buf, sizeof(__buf), FMT, __VA_ARGS__);   \
        FB_THROW_MSG(std::string(__buf));                   \
    } while (0)

#define FB_THROW_IF_NOT(X)                                  \
    do {                                                    \
        if (!(X)) {                                         \
            FB_THROW_FMT("Error: '%s' failed", #X);         \
        }                                                   \
    } while (0)

#define FB_THROW_IF_NOT_MSG(X, MSG)                         \
    do {                                                    \
        if (!(X)) {                                         \
            FB_THROW_FMT("Error: '%s' failed: " MSG, #X);   \
        }                                                   \
    } while (0)

#define FB_THROW_IF_NOT_FMT(X, FMT, ...)                            \
    do {                                                            \
        if (!(X)) {                                                 \
            FB_THROW_FMT("Error: '%s' failed: " FMT, #X, __VA_ARGS__); \
        }                                                           \
    } while (0)

// CUDA errors are internal failures: surface them as exceptions carrying the CUDA string
// (the reference asserts, faiss/gpu/utils/DeviceUtils.h:143-155; an exception is kinder to a
// host process and still non-ignorable).
#define CUDA_VERIFY(X)                                                              \
    do {                                                                            \
        cudaError_t __e = (X);                                                      \
        if (__e != cudaSuccess) {                                                   \
            FB_THROW_FMT("CUDA error %d: %s (%s)", (int)__e, cudaGetErrorString(__e), #X); \
        }                                                                           \
    } while (0)

// every kernel launch site is followed by CUDA_CHECK_LAST(): it also feeds the launch counter that
// bench.py reports as "gpu_launches"
long long& kernelLaunchCounter();
#define CUDA_CHECK_LAST()                        \
    do {                                         \
        ::fb200::kernelLaunchCounter()++;        \
        CUDA_VERIFY(cudaGetLastError());         \
    } while (0)

// optional per-kernel device timing (CUDA events on the launching stream), used by bench.py for
// the roofline line; off by default
struct KernelTiming {
    static void enable(bool on);
    static bool enabled();
    static void begin(const char* name, cudaStream_t stream);
    static void end(const char* name, cudaStream_t stream);
    // synchronises, sums and clears: total milliseconds and number of launches for `name`
    static void collect(const char* name, double* ms, int* launches);
};

#ifdef __CUDACC__
#define FB_HD __host__ __device__
#else
#define FB_HD
#endif

FB_HD inline int64_t ceil_div(int64_t a, int64_t b) {
    return (a + b - 1) / b;
}
FB_HD inline int64_t round_up(int64_t a, int64_t b) {
    return ceil_div(a, b) * b;
}
inline int next_pow2(int v) {
    int p = 1;
    while (p < v)
        p <<= 1;
    return p;
}

// runtime value -> compile-time constant for a launcher's kernel template: f(std::true_type{}) or f(std::false_type{})
template <typename F>
void withBool(bool b, F&& f) {
    if (b)
        f(std::true_type{});
    else
        f(std::false_type{});
}

} // namespace fb200
