"""Mint tests/golden/reconstruct.npz from the reference CPU library (oracle/_ref): IndexIVF::reconstruct_n of CPU
IVF indexes whose lists hold random codes, for every stored layout of the GPU decoder -- every scalar-quantiser type
at d = 40 and d = 36 with and without a residual, PQ with 8-bit (M = 8 / 16 / 32), 4-bit (M = 8 / 32 / 64), 5- and
6-bit codes, and IVF-Flat.  Every id in [0, N) is stored, some twice, so the last-in-(list, offset) rule shows.
Plus one IndexIVF::search_and_return_codes case with include_listno at nlist = 300 (2-byte list numbers), with
search_and_reconstruct on the same index.

    python -m tests.golden.make_golden_reconstruct
"""
import os

import numpy as np

from oracle import oracle_recons_np as rn
from oracle import oracle_sq_np as so

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reconstruct.npz")
NLIST, N, DUP = 8, 40, 12
CODES_NLIST, CODES_N, CODES_D, CODES_NQ, CODES_K, CODES_NPROBE = 300, 2000, 8, 6, 5, 300

CASES = [("flat", rn.FLAT, {"d": 16})]
CASES += [("pq%d_m%d" % (nb, m), rn.PQ, {"d": 64, "M": m, "nbits": nb})
          for nb, m in ((8, 8), (8, 16), (8, 32), (4, 8), (4, 32), (4, 64), (5, 8), (6, 8))]
CASES += [("sq%d_%s_d%d" % (q, "res" if r else "nores", d), rn.SQ, {"d": d, "qtype": q, "by_residual": r})
          for q in range(7) for r in (True, False) for d in (40, 36)]


def _lists(rs, kind, p):
    d = p["d"]
    ids = np.concatenate([rs.permutation(N), rs.choice(N, DUP)]).astype(np.int64)
    n = ids.size
    if kind == rn.FLAT:
        codes = (rs.rand(n, d) * 4).astype(np.float32).view(np.uint8).reshape(n, -1)
    elif kind == rn.PQ:
        codes = rs.randint(0, 256, (n, (p["M"] * p["nbits"] + 7) // 8)).astype(np.uint8)
    elif p["qtype"] == so.QT_fp16:
        codes = (rs.rand(n, d) * 8 - 4).astype(np.float16).view(np.uint8).reshape(n, -1)
    else:
        codes = rs.randint(0, 256, (n, so.code_size(p["qtype"], d))).astype(np.uint8)
    assign = rs.randint(0, NLIST, n)
    return [codes[assign == l] for l in range(NLIST)], [ids[assign == l] for l in range(NLIST)]


def make():
    from oracle import ref, ref_sq

    rs = np.random.RandomState(2026)
    out = {}
    for name, kind, p in CASES:
        d = p["d"]
        lc, li = _lists(rs, kind, p)
        cent = (rs.rand(NLIST, d) * 2 - 1).astype(np.float32)
        if kind == rn.FLAT:
            cpu = ref.IndexIVFFlat(d, NLIST)
        elif kind == rn.PQ:
            cpu = ref.IndexIVFPQ(d, NLIST, p["M"], p["nbits"])
            pq = (rs.rand(p["M"], 1 << p["nbits"], d // p["M"]) * 2 - 1).astype(np.float32)
            cpu.set_pq_centroids(pq)
            out[name + "/pq"] = pq
        else:
            cpu = ref_sq.IndexIVFScalarQuantizer(d, NLIST, p["qtype"], 1, p["by_residual"])
            t = so.train_minmax((rs.rand(50, d) * 6 - 3).astype(np.float32), p["qtype"])
            cpu.set_trained(t)
            out[name + "/trained"] = t
        cpu.set_centroids(cent)
        for l in range(NLIST):
            if li[l].size:
                cpu.add_entries(l, li[l], lc[l])
        cpu.set_is_trained(True)
        out[name + "/centroids"] = cent
        for l in range(NLIST):
            out["%s/codes%d" % (name, l)] = lc[l].reshape(-1)
            out["%s/ids%d" % (name, l)] = li[l]
        out[name + "/recons"] = cpu.reconstruct_n(0, N, d)
    # search_and_return_codes with list numbers: IVF-Flat over 300 lists, integer data, unique ids
    from oracle import ref_recons

    cpu = ref.IndexIVFFlat(CODES_D, CODES_NLIST)
    cent = np.floor(rs.rand(CODES_NLIST, CODES_D) * 16).astype(np.float32)
    xb = np.floor(rs.rand(CODES_N, CODES_D) * 16).astype(np.float32)
    ids = (rs.permutation(CODES_N) * 3 + 5).astype(np.int64)
    assign = rs.randint(0, CODES_NLIST, CODES_N)
    cpu.set_centroids(cent)
    for l in range(CODES_NLIST):
        if (assign == l).any():
            cpu.add_entries(l, ids[assign == l], xb[assign == l].view(np.uint8))
    cpu.set_is_trained(True)
    xq = np.floor(rs.rand(CODES_NQ, CODES_D) * 16).astype(np.float32)
    D, I, C = ref_recons.search_and_return_codes(cpu, xq, CODES_K, CODES_NPROBE, include_listno=True)
    _, _, R = ref_recons.search_and_reconstruct(cpu, xq, CODES_K, CODES_NPROBE)
    out.update({"codes/centroids": cent, "codes/xb": xb, "codes/ids": ids, "codes/assign": assign, "codes/xq": xq,
                "codes/D": D, "codes/I": I, "codes/codes": C, "codes/R": R})
    np.savez_compressed(PATH, **out)


def load():
    return dict(np.load(PATH))


if __name__ == "__main__":
    make()
    print("wrote", PATH)
