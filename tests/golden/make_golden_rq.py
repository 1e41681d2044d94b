"""Mint tests/golden/rq.npz from the reference CPU library (oracle/_ref): ResidualQuantizer::refine_beam,
refine_beam_LUT (on the CPU's own query norms and x·Cᵀ) and compute_codes_add_centroids on integer-valued codebooks
and vectors, so every dot product, norm and partial sum is exact in fp32 and only the order of the roundings that
remain, and the selection's tie rule, decide the result.

Cases cover:
  - beams 1, 5 and 32;
  - mixed nbits, with steps where K < 32 (the scalar tail of the AVX2 LUT build) and K >= 32;
  - M = 10, where the LUT accumulation runs in chunks of 8;
  - codebooks with repeated rows, so whole groups of candidates tie;
  - compute_codes in both modes for every search type the device packs, with and without centroids.

    python -m tests.golden.make_golden_rq
"""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rq.npz")

# name, d, nbits, beam, n, repeated codebook rows
CASES = [
    ("m4b5", 16, [6, 6, 6, 6], 5, 120, False),
    ("ties_b5", 8, [5, 5, 5], 5, 120, True),
    ("mixed_b32", 12, [4, 8, 3, 6, 5], 32, 60, False),
    ("m10_b5", 10, [4, 6, 3, 5, 4, 6, 3, 5, 5, 6], 5, 60, False),
    ("b1", 8, [8, 8, 4], 1, 80, False),
]
SEARCH_TYPES = range(6)  # ST_decompress .. ST_norm_qint4: the types the device packs
NORM_RANGE = (200.0, 900.0)  # norm_min / norm_max of the qint types: some norms fall outside and are clamped


def int_data(rs, d, nbits, n, repeated):
    tk = sum(1 << b for b in nbits)
    cb = rs.randint(-8, 9, (tk, d)).astype(np.float32)
    if repeated:
        cb[1::2] = cb[0::2]  # every codeword twice: candidates (b, 2k) and (b, 2k + 1) tie
    x = rs.randint(-16, 17, (n, d)).astype(np.float32)
    cent = rs.randint(-3, 4, (n, d)).astype(np.float32)
    return cb, x, cent


def load():
    return dict(np.load(PATH))


def case(gd, name):
    return {k.split("/", 1)[1]: v for k, v in gd.items() if k.startswith(name + "/")}


def main():
    from oracle import ref_rq

    out = {}
    rs = np.random.RandomState(0)
    for name, d, nbits, beam, n, repeated in CASES:
        cb, x, cent = int_data(rs, d, nbits, n, repeated)
        q = ref_rq.RQ(d, nbits, cb)
        c0, r0, d0 = q.refine_beam(x[:, None], 1, beam)
        c1, d1 = q.refine_beam_lut(x, beam)
        e = {"cb": cb, "x": x, "cent": cent, "codes0": c0, "resid0": r0, "dis0": d0, "codes1": c1, "dis1": d1}
        for lut in (0, 1):
            for st in SEARCH_TYPES:
                qs = ref_rq.RQ(d, nbits, cb, search_type=st, max_beam_size=beam, use_beam_LUT=lut,
                               norm_min=NORM_RANGE[0], norm_max=NORM_RANGE[1])
                e["packed%d_%d" % (lut, st)] = qs.compute_codes(x)
                e["packed%d_%d_cent" % (lut, st)] = qs.compute_codes(x, cent)
        out.update({name + "/" + k: v for k, v in e.items()})
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
