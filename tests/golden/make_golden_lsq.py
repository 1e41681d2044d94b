"""Mint tests/golden/lsq.npz from the reference CPU library (oracle/_ref): lsq::IcmEncoder::encode and
LocalSearchQuantizer::compute_codes on integer-valued codebooks and vectors (|v| <= 8, so every unary, binary and
evaluate sum is exact in fp32), with the perturbation draws of std::mt19937 + std::uniform_int_distribution.

Cases cover K = 4 (every entry a leftover of the 16-bucket argmin), K = 16 / 32 / 256 (whole buckets), nperts = 0,
nperts = M, and a forced-tie case: codebooks with few distinct rows, so most argmins are exact ties decided by the
tie rule.

    python -m tests.golden.make_golden_lsq
"""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lsq.npz")

# name, M, K, d, n, ils_iters, nperts, icm_iters, seed, distinct codebook rows (0: all random)
CASES = [
    ("m4k16", 4, 16, 32, 60, 8, 4, 4, 1234, 0),
    ("m3k4", 3, 4, 8, 50, 5, 2, 3, 7, 0),
    ("m8k256", 8, 256, 24, 40, 3, 4, 2, 99, 0),
    ("nperts0", 4, 16, 16, 40, 3, 0, 4, 5, 0),
    ("ties_k32", 4, 32, 12, 80, 6, 3, 4, 2024, 3),
    ("ties_k16", 3, 16, 6, 80, 6, 3, 4, 77, 2),
]
# compute_codes: name, M, K, d, n, encode_ils_iters, nperts, icm_iters, random_seed
CC_CASES = [("cc_m4k16", 4, 16, 16, 70, 4, 4, 4, 0x12345)]


def int_data(rs, M, K, d, n, distinct):
    if distinct:
        rows = rs.randint(-8, 9, (M, distinct, d)).astype(np.float32)
        cb = rows[:, rs.randint(0, distinct, K)]
    else:
        cb = rs.randint(-8, 9, (M, K, d)).astype(np.float32)
    x = rs.randint(-8, 9, (n, d)).astype(np.float32)
    return np.ascontiguousarray(cb), x


def load():
    return dict(np.load(PATH))


def main():
    from oracle import ref_lsq

    out = {}
    rs = np.random.RandomState(0)
    for name, M, K, d, n, ils, nperts, icm, seed, distinct in CASES:
        cb, x = int_data(rs, M, K, d, n, distinct)
        codes0 = rs.randint(0, K, (n, M)).astype(np.int32)
        q = ref_lsq.LSQ(cb, nperts=nperts, icm_iters=icm)
        codes, nxt = q.icm_encode(codes0, x, ils, seed)
        perts, nxt_d = ref_lsq.draws(M, K, nperts, n, ils, seed)
        assert nxt_d == nxt
        out.update({name + "/cb": cb, name + "/x": x, name + "/codes0": codes0, name + "/codes": codes,
                    name + "/perts": perts, name + "/next": np.uint32(nxt)})
    for name, M, K, d, n, ils, nperts, icm, seed in CC_CASES:
        cb, x = int_data(rs, M, K, d, n, 0)
        q = ref_lsq.LSQ(cb, nperts=nperts, icm_iters=icm, encode_ils_iters=ils, random_seed=seed)
        out.update({name + "/cb": cb, name + "/x": x, name + "/codes": q.compute_codes(x)})
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
