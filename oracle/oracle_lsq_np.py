"""Numpy restatement of LocalSearchQuantizer's ICM encoding (the CPU lsq::IcmEncoder) and of the random draws it makes.

    icm_encode_impl      faiss/impl/LocalSearchQuantizer.cpp:539-592
    icm_encode_step      :594-672   (argmin: HeapWithBucketsCMaxFloat<16, 1>::addn, faiss/impl/approx_topk/)
    perturb_codes        :673-688
    compute_binary_terms :690-711
    compute_unary_terms  :713-758
    evaluate             :760-795
    compute_codes        :294-321   (random_int32, :138-147, then icm_encode in chunks of chunk_size, :501-537)

The draws are those of libstdc++: std::mt19937 raw words, and std::uniform_int_distribution<T>(0, r - 1) over them,
which for a 32-bit engine and r <= 2^32 is Lemire's nearly-divisionless downscaling (uniform_int_distribution::
operator() -> _S_nd<uint64_t> in bits/uniform_int_dist.h): p = word * r as 64 bits; when the low 32 bits of p are
below (2^32 - r) mod r, draw again; the result is p >> 32.  The distribution's integer type (size_t for m, int32_t
for k) does not change this path.

fp32 arithmetic follows the CPU where it is exact: every product and sum of the fixtures and tests that compare codes
byte for byte is an integer below 2^24.  The inner products here are float64 rounded to fp32, which is what any
summation order gives in that regime.

Only tests/, tests/golden/ and bench_icm.py import this module.
"""
import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)


# ------------------------------------------------------------------------------------------
# std::mt19937 (libstdc++ bits/random.tcc: seed, _M_gen_rand, operator())
# ------------------------------------------------------------------------------------------
class MT19937:
    N, MM = 624, 397

    def __init__(self, seed):
        mt = np.zeros(624, np.uint64)
        mt[0] = seed & 0xFFFFFFFF
        for i in range(1, 624):
            p = int(mt[i - 1])
            mt[i] = (1812433253 * (p ^ (p >> 30)) + i) & 0xFFFFFFFF
        self.mt = mt.astype(np.uint32)
        self.buf = np.zeros(0, np.uint32)  # tempered words not handed out yet

    def _twist(self):
        mt = self.mt.astype(np.uint64)

        def seg(lo, hi, nxt, far):
            y = (mt[lo:hi] & 0x80000000) | (nxt & 0x7FFFFFFF)
            mt[lo:hi] = far ^ (y >> 1) ^ np.where(y & 1, 0x9908B0DF, 0).astype(np.uint64)

        # entry i reads entries i + 1 and i + 397 (mod 624); the ones below i are already new
        seg(0, 227, mt[1:228].copy(), mt[397:624].copy())
        seg(227, 454, mt[228:455].copy(), mt[0:227].copy())
        seg(454, 623, mt[455:624].copy(), mt[227:396].copy())
        seg(623, 624, mt[0:1].copy(), mt[396:397].copy())
        self.mt = mt.astype(np.uint32)
        y = mt.copy()
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        return (y & 0xFFFFFFFF).astype(np.uint32)

    def words(self, count):
        """the next `count` raw outputs"""
        parts = [self.buf]
        have = self.buf.size
        while have < count:
            w = self._twist()
            parts.append(w)
            have += w.size
        allw = np.concatenate(parts)
        self.buf = allw[count:]
        return allw[:count].astype(np.uint64)


def uniform_ints(gen, ranges):
    """std::uniform_int_distribution(0, r - 1)(gen) for each r of `ranges` in order (1 <= r < 2^32)"""
    ranges = np.asarray(ranges, np.uint64)
    out = np.empty(ranges.size, np.uint64)
    pos = 0
    while pos < ranges.size:
        r = ranges[pos:]
        w = gen.words(r.size)
        p = w * r
        thr = (np.uint64(1 << 32) - r) % r
        rej = np.nonzero((p & 0xFFFFFFFF) < thr)[0]
        if rej.size == 0:
            out[pos:] = p >> 32
            break
        # draw j is rejected: it takes words until one passes; the words after it go back to the generator
        j = int(rej[0])
        out[pos:pos + j] = p[:j] >> 32
        gen.buf = np.concatenate([w[j + 1:].astype(np.uint32), gen.buf])
        rj = int(r[j])
        while True:
            q = int(gen.words(1)[0]) * rj
            if (q & 0xFFFFFFFF) >= ((1 << 32) - rj) % rj:
                break
        out[pos + j] = q >> 32
        pos += j + 1
    return out.astype(np.int64)


def draws(gen, M, K, nperts, n, ils_iters):
    """perturb_codes' draws over ils_iters iterations: [ils_iters, n, nperts, 2] int32 (m, k)"""
    cnt = ils_iters * n * nperts
    ranges = np.empty(2 * cnt, np.uint64)
    ranges[0::2] = M
    ranges[1::2] = K
    return uniform_ints(gen, ranges).astype(np.int32).reshape(ils_iters, n, nperts, 2)


# ------------------------------------------------------------------------------------------
# the encoder
# ------------------------------------------------------------------------------------------
def argmin_buckets(obj):
    """HeapWithBucketsCMaxFloat<16, 1>::addn(K, obj, 1, &best (= HUGE_VALF), &code (= 0)) per row of obj [n, K].
    Bucket j holds positions j, j + 16, ... below K // 16 * 16 and keeps the first of equal values (AVX2
    cmplt_min_max_fast keeps the current entry when current <= candidate); the buckets are merged on (value, index)
    (CMax::cmp2); the K % 16 leftovers replace the best only when strictly smaller (CMax::cmp)."""
    n, K = obj.shape
    best_v = np.full(n, np.inf, np.float32)
    best_i = np.zeros(n, np.int64)
    nb = K // 16 * 16
    if nb:
        bv = np.full((n, 16), FLT_MAX, np.float32)
        bi = np.tile(np.arange(16, dtype=np.int64), (n, 1))
        for g in range(0, nb, 16):
            v = obj[:, g:g + 16]
            take = v < bv
            bv = np.where(take, v, bv)
            bi = np.where(take, g + np.arange(16), bi)
        for j in range(16):
            take = (bv[:, j] < best_v) | ((bv[:, j] == best_v) & (bi[:, j] < best_i))
            best_v = np.where(take, bv[:, j], best_v)
            best_i = np.where(take, bi[:, j], best_i)
    for k in range(nb, K):
        take = obj[:, k] < best_v
        best_v = np.where(take, obj[:, k], best_v)
        best_i = np.where(take, k, best_i)
    return best_i.astype(np.int32)


def _ip32(a, b):
    return (a.astype(np.float64) @ b.astype(np.float64).T).astype(np.float32)


def unary_terms(cb, x):
    """compute_unary_terms: u [n, M, K] = (-2 * <x_i, C_m[k]>) + |C_m[k]|^2, one fp32 rounding per step"""
    M, K, d = cb.shape
    ip = _ip32(x, cb.reshape(M * K, d)).reshape(-1, M, K)
    norms = (cb.astype(np.float64) ** 2).sum(-1).astype(np.float32)
    return (np.float32(-2) * ip) + norms[None]


def binary_terms(cb):
    """compute_binary_terms: b [M, M, K, K] = 2 * <C_m1[k1], C_m2[k2]>"""
    M, K, d = cb.shape
    ip = _ip32(cb.reshape(M * K, d), cb.reshape(M * K, d)).reshape(M, K, M, K)
    return np.float32(2) * ip.transpose(0, 2, 1, 3)


def evaluate(cb, codes, x):
    """evaluate: decode 0 + C_0[c_0] + C_1[c_1] + ... in m order, then the squared L2 error per row"""
    M = cb.shape[0]
    dec = np.zeros(x.shape, np.float32)
    for m in range(M):
        dec = dec + cb[m][codes[:, m]]
    return ((x - dec) ** 2).sum(1, dtype=np.float32)


def icm_step(codes, u, b, icm_iters):
    M = codes.shape[1]
    for _ in range(icm_iters):
        for m in range(M):
            obj = u[:, m, :].copy()
            for m2 in range(M):
                if m2 != m:
                    obj = obj + b[m2, m][codes[:, m2]]
            codes[:, m] = argmin_buckets(obj)


def icm_encode(cb, codes, x, perts, icm_iters):
    """icm_encode_impl on codes [n, M] with the draws perts [ils_iters, n, nperts, 2]: the best codes"""
    cb = np.ascontiguousarray(cb, np.float32)
    x = np.ascontiguousarray(x, np.float32)
    M = cb.shape[0]
    codes = np.array(codes, np.int32)
    assert perts.shape[2] <= M, "nperts <= M"
    u = unary_terms(cb, x)
    b = binary_terms(cb)
    best = codes.copy()
    best_err = evaluate(cb, codes, x)
    rows = np.arange(codes.shape[0])
    for it in range(perts.shape[0]):
        for j in range(perts.shape[2]):
            codes[rows, perts[it, :, j, 0]] = perts[it, :, j, 1]
        icm_step(codes, u, b, icm_iters)
        err = evaluate(cb, codes, x)
        better = err < best_err
        best_err = np.where(better, err, best_err)
        best[better] = codes[better]
        codes = best.copy()
    return best


def encode_seeded(cb, codes, x, ils_iters, nperts, icm_iters, seed):
    """lsq::IcmEncoder::encode with std::mt19937(seed): (codes, the generator's next output afterwards)"""
    M, K, _ = cb.shape
    gen = MT19937(seed)
    p = draws(gen, M, K, nperts, x.shape[0], ils_iters)
    out = icm_encode(cb, codes, x, p, icm_iters)
    return out, int(gen.words(1)[0])


def compute_codes(cb, x, ils_iters, nperts, icm_iters, seed, chunk_size=10000):
    """LocalSearchQuantizer::compute_codes, unpacked to int32 [n, M]"""
    M, K, _ = cb.shape
    n = x.shape[0]
    gen = MT19937(seed)
    codes = uniform_ints(gen, np.full(n * M, K, np.uint64)).astype(np.int32).reshape(n, M)
    for i0 in range(0, n, chunk_size):
        i1 = min(n, i0 + chunk_size)
        p = draws(gen, M, K, nperts, i1 - i0, ils_iters)
        codes[i0:i1] = icm_encode(cb, codes[i0:i1], x[i0:i1], p, icm_iters)
    return codes
