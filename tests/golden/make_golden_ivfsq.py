"""Mint tests/golden/ivfsq.npz from the reference CPU library (oracle/_ref, oracle/ref_sq.py).

    python tests/golden/make_golden_ivfsq.py

One case per (qtype, d, metric, by_residual) of CASES.  Inputs are regenerated from the case seed by
case_data(), so the file only holds what the reference computed: the coarse centroids, the trained
ScalarQuantizer parameters, every inverted list (codes + ids) and the search results.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ivfsq.npz")
NLIST, NB, NQ, K, NPROBE = 8, 200, 8, 10, 3

# (qtype, d, metric, by_residual); metric 1 = L2, 0 = IP
CASES = []
for _qt in range(7):
    CASES += [(_qt, 40, 1, True), (_qt, 40, 0, False), (_qt, 128, 0, True), (_qt, 128, 1, False)]


def case_data(i, qtype, d):
    """training rows, database rows, queries of case i (8bit_direct: integers in [0, 256))"""
    rs = np.random.RandomState(1000 + i)
    if qtype == 5:
        gen = lambda n: np.floor(rs.rand(n, d) * 256).astype(np.float32)  # noqa: E731
    else:
        gen = lambda n: (rs.rand(n, d) * 4).astype(np.float32)  # noqa: E731
    return gen(NB), gen(NB), gen(NQ)


def main():
    from oracle import ref_sq

    out = {"cases": np.array(CASES, dtype=np.int64)}
    for i, (qt, d, metric, res) in enumerate(CASES):
        xt, xb, xq = case_data(i, qt, d)
        idx = ref_sq.IndexIVFScalarQuantizer(d, NLIST, qt, metric, res)
        idx.set_cp(niter=5)
        idx.train(xt)
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
        out[p + "trained"] = idx.trained()
        out[p + "codes"] = np.concatenate(codes)
        out[p + "ids"] = np.concatenate(ids)
        out[p + "lens"] = np.array(lens, dtype=np.int64)
        out[p + "D"] = D
        out[p + "I"] = I
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


def load():
    """[(case dict)] with lists split back per inverted list"""
    z = np.load(OUT)
    cases = []
    for i, (qt, d, metric, res) in enumerate(z["cases"]):
        p = "c%d_" % i
        lens = z[p + "lens"]
        off = np.concatenate([[0], np.cumsum(lens)])
        cs = z[p + "codes"].size // max(1, int(lens.sum()))
        codes = [z[p + "codes"][off[l] * cs : off[l + 1] * cs] for l in range(NLIST)]
        ids = [z[p + "ids"][off[l] : off[l + 1]] for l in range(NLIST)]
        xt, xb, xq = case_data(i, int(qt), int(d))
        cases.append(dict(
            i=i, qtype=int(qt), d=int(d), metric=int(metric), by_residual=bool(res), xt=xt, xb=xb, xq=xq,
            centroids=z[p + "centroids"], trained=z[p + "trained"], codes=codes, ids=ids, D=z[p + "D"], I=z[p + "I"],
        ))
    return cases


if __name__ == "__main__":
    main()
