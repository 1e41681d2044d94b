"""Mints tests/golden/idselector.npz from the reference CPU library (oracle/_ref, oracle/ref_sel.py): IndexFlat
(L2, IP) and IndexIVFFlat (L2, IP, add_with_ids ids with negative and >= 2^40 values) searched with
SearchParameters::sel for the eight selectors of the reference GPU tests (faiss/gpu/test/TestUtils.cpp:433-475).

    python tests/golden/make_golden_idselector.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import oracle_sel_np as osel  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "idselector.npz")
NF, NI, D, NQ, K, NLIST, NPROBE = 2000, 3000, 32, 20, 15, 16, 4
METRICS = {"l2": 1, "ip": 0}


def data():
    rs = np.random.RandomState(123)
    xf = np.floor(rs.rand(NF, D) * 16).astype(np.float32)
    xi = np.floor(rs.rand(NI, D) * 16).astype(np.float32)
    xq = np.floor(rs.rand(NQ, D) * 16).astype(np.float32)
    return xf, xi, xq, osel.ivf_ids(NI)


def reference_results():
    from oracle import ref, ref_sel

    xf, xi, xq, ids = data()
    out = {"xf": xf, "xi": xi, "xq": xq, "ivf_ids": ids}
    for mname, metric in METRICS.items():
        flat = ref.IndexFlat(D, metric)
        flat.add(xf)
        for sname, spec in osel.reference_selectors(NF).items():
            out["flat_%s_%s_D" % (mname, sname)], out["flat_%s_%s_I" % (mname, sname)] = ref_sel.search(flat, xq, K, spec)
        ivf = ref.IndexIVFFlat(D, NLIST, metric)
        ivf.set_cp(niter=4)
        ivf.train(xi)
        ivf.add_with_ids(xi, ids)
        out["ivf_%s_centroids" % mname] = ivf.centroids()
        out["ivf_%s_assign" % mname] = ivf.quantizer_search(xi, 1)[1][:, 0]
        for sname, spec in osel.ivf_selectors(ids).items():
            out["ivf_%s_%s_D" % (mname, sname)], out["ivf_%s_%s_I" % (mname, sname)] = ref_sel.search(
                ivf, xq, K, spec, nprobe=NPROBE)
    return out


if __name__ == "__main__":
    np.savez_compressed(OUT, **reference_results())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
