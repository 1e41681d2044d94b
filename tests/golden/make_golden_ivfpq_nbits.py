"""Mint tests/golden/ivfpq_nbits.npz from the reference CPU library (oracle/_ref, oracle/ref_pq.py).

    python tests/golden/make_golden_ivfpq_nbits.py

One case per (nbits, d, M, metric) of CASES: IndexIVFPQ with 4-, 5- and 6-bit codes.  Inputs are regenerated
from the case seeds with float_rand by case_data(), so the file only holds what the reference computed: the
coarse centroids, the PQ centroids IndexIVFPQ::train produces with that coarse quantizer preset, every inverted
list (packed code bytes + ids), ProductQuantizer::compute_codes of a probe set, and the search results.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ivfpq_nbits.npz")
NLIST, NB, NQ, NPC, K, NPROBE, NITER = 16, 3000, 20, 64, 10, 4, 5

# (nbits, d, M, metric); metric 1 = L2, 0 = IP.  The 4-bit cases with M in {32, 64} take the interleaved
# nibble-pair scan, every other case the packed vector-major scan.
CASES = [
    (4, 64, 32, 1),
    (4, 64, 32, 0),
    (4, 128, 64, 1),
    (4, 64, 16, 0),
    (4, 40, 5, 1),
    (5, 64, 16, 1),
    (5, 64, 16, 0),
    (6, 48, 12, 1),
    (6, 64, 32, 0),
]


def case_data(i, d):
    """database rows (also the training set), queries and the compute_codes probe set of case i"""
    from oracle import oracle_np as o

    s = 100 * (i + 1)
    xb = o.float_rand(NB * d, s + 1).reshape(NB, d)
    xq = o.float_rand(NQ * d, s + 2).reshape(NQ, d)
    xp = o.float_rand(NPC * d, s + 3).reshape(NPC, d)
    return xb, xq, xp


def main():
    from oracle import ref_pq

    out = {"cases": np.array(CASES, dtype=np.int64)}
    for i, (nbits, d, M, metric) in enumerate(CASES):
        xb, xq, xp = case_data(i, d)
        # the coarse quantizer first, then IndexIVFPQ::train with it preset (only the PQ is trained)
        coarse = ref_pq.IndexIVFPQ(d, NLIST, M, nbits, metric)
        coarse.set_cp(niter=NITER)
        coarse.set_pq_cp(niter=NITER)
        coarse.train(xb)
        idx = ref_pq.IndexIVFPQ(d, NLIST, M, nbits, metric)
        idx.set_pq_cp(niter=NITER)
        idx.set_centroids(coarse.centroids())
        idx.train(xb)
        idx.add(xb)
        idx.set_nprobe(NPROBE)
        D, I = idx.search(xq, K)
        codes, ids, lens = [], [], []
        for l in range(NLIST):
            c, a = idx.get_list(l)
            codes.append(c)
            ids.append(a)
            lens.append(a.size)
        p = "c%d_" % i
        out[p + "centroids"] = idx.centroids()
        out[p + "pq"] = idx.pq_centroids()
        out[p + "codes"] = np.concatenate(codes)
        out[p + "ids"] = np.concatenate(ids)
        out[p + "lens"] = np.array(lens, dtype=np.int64)
        out[p + "probe_codes"] = idx.pq_compute_codes(xp)
        out[p + "D"] = D
        out[p + "I"] = I
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


def load():
    """[(case dict)] with the lists split back per inverted list"""
    z = np.load(OUT)
    cases = []
    for i, (nbits, d, M, metric) in enumerate(z["cases"]):
        p = "c%d_" % i
        nbits, d, M = int(nbits), int(d), int(M)
        cs = (M * nbits + 7) // 8
        lens = z[p + "lens"]
        off = np.concatenate([[0], np.cumsum(lens)])
        codes = [z[p + "codes"][off[l] * cs : off[l + 1] * cs] for l in range(NLIST)]
        ids = [z[p + "ids"][off[l] : off[l + 1]] for l in range(NLIST)]
        xb, xq, xp = case_data(i, d)
        cases.append(dict(
            i=i, nbits=nbits, d=d, M=M, metric=int(metric), code_size=cs, xb=xb, xq=xq, xp=xp,
            centroids=z[p + "centroids"], pq=z[p + "pq"], codes=codes, ids=ids, probe_codes=z[p + "probe_codes"],
            D=z[p + "D"], I=z[p + "I"],
        ))
    return cases


if __name__ == "__main__":
    main()
