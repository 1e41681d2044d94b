"""Mint tests/golden/pairwise.npz: all-pairs distance matrices of the CPU, per metric.

    python tests/golden/make_golden_pairwise.py

For every metric of CASES, two cases, each stored with its inputs (small):
  int     integer-valued data (floor(16 u) + 1; Gower: mixed columns): every partial sum is exact for L2, IP, L1, Linf,
          BrayCurtis and Jaccard, so those matrices are the exact values
  float   random floats of the metric's domain; for Canberra and JensenShannon one query row and one database row
          carry a zero component, so that some entries are NaN, as the CPU computes them
The matrices come from the reference CPU library (oracle/ref_pairwise.py) where it is built, else from the numpy
restatements (oracle_np.pairwise, oracle_metrics_np.pairwise_extra); test_pairwise_oracle.py checks that both agree.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import oracle_metrics_np as m  # noqa: E402
from oracle import oracle_np as o  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pairwise.npz")
NB, NQ, D = 50, 6, 19

# (name, metric, metric_arg)
CASES = [
    ("L2", m.METRIC_L2, 0.0),
    ("IP", m.METRIC_INNER_PRODUCT, 0.0),
    ("L1", m.METRIC_L1, 0.0),
    ("Linf", m.METRIC_Linf, 0.0),
    ("Lp1", m.METRIC_Lp, 1.0),
    ("Lp2", m.METRIC_Lp, 2.0),
    ("Lp0.5", m.METRIC_Lp, 0.5),
    ("Lp3", m.METRIC_Lp, 3.0),
    ("Canberra", m.METRIC_Canberra, 0.0),
    ("BrayCurtis", m.METRIC_BrayCurtis, 0.0),
    ("JensenShannon", m.METRIC_JensenShannon, 0.0),
    ("Jaccard", m.METRIC_Jaccard, 0.0),
    ("Gower", m.METRIC_GOWER, 0.0),
]


def case_data(i, metric, kind):
    rs = np.random.RandomState(3000 + 2 * i + (kind == "int"))
    integer = kind == "int"
    xb = m.metric_data(metric, rs, NB, D, integer)
    xq = m.metric_data(metric, rs, NQ, D, integer)
    if kind == "float" and metric in (m.METRIC_Canberra, m.METRIC_JensenShannon):
        xq[1, 4] = 0.0
        xb[[3, 4], 4] = 0.0
    return xq, xb


def numpy_pairwise(xq, xb, metric, arg):
    """the CPU's values restated in numpy"""
    if metric == m.METRIC_Lp and arg in (1.0, 2.0):
        metric, arg = (m.METRIC_L1 if arg == 1.0 else m.METRIC_L2), 0.0
    if metric in (m.METRIC_L2, m.METRIC_INNER_PRODUCT):
        return o.pairwise(xq, xb, metric)
    return m.pairwise_extra(xq, xb, metric, arg)


def main():
    from oracle import ref_pairwise

    live = ref_pairwise.available()
    out = {}
    for i, (name, metric, arg) in enumerate(CASES):
        for kind in ("int", "float"):
            xq, xb = case_data(i, metric, kind)
            dis = ref_pairwise.pairwise(xq, xb, metric, arg) if live else numpy_pairwise(xq, xb, metric, arg)
            key = "%s_%s" % (name, kind)
            out[key + "_xq"], out[key + "_xb"], out[key + "_D"] = xq, xb, dis
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "from", "the reference library" if live else "the numpy restatements")


if __name__ == "__main__":
    main()
