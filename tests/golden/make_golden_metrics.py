"""Mint tests/golden/metrics.npz from the reference CPU library (oracle/_ref, oracle/ref_metrics.py).

    python tests/golden/make_golden_metrics.py

One case per (metric, metric_arg, d, data kind) of CASES.  Inputs are regenerated from the case seed by
case_data(), so the file only holds what the reference's knn_extra_metrics returned: D and I per case.

Data kinds:
  float   random floats of the metric's domain (positive for Canberra / JensenShannon / Jaccard, mixed
          numeric / categorical columns for Gower)
  int     floor(16 u) + 1 (Gower: numeric columns in quarters)
  nan     a third of the rows give a NaN distance (zero components for Canberra / JensenShannon, out-of-range
          or mixed values for Gower)
  pad     all but 6 rows give a NaN distance, k = 20: every query has fewer valid rows than k
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import oracle_metrics_np as m  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "metrics.npz")
NB, NQ, K, K_PAD = 300, 8, 10, 20

KINDS = ["float", "int", "nan", "pad"]
# (metric, metric_arg, d, kind)
CASES = []
for _mt, _arg in [(m.METRIC_L1, 0.0), (m.METRIC_Linf, 0.0), (m.METRIC_Lp, 0.5), (m.METRIC_Lp, 3.0),
                  (m.METRIC_Canberra, 0.0), (m.METRIC_BrayCurtis, 0.0), (m.METRIC_JensenShannon, 0.0),
                  (m.METRIC_Jaccard, 0.0), (m.METRIC_GOWER, 0.0)]:
    CASES += [(_mt, _arg, 17, "float"), (_mt, _arg, 40, "int")]
for _mt in (m.METRIC_Canberra, m.METRIC_JensenShannon, m.METRIC_GOWER):
    CASES += [(_mt, 0.0, 17, "nan"), (_mt, 0.0, 40, "pad")]


def _spoil(metric, rs, xb, xq, rows):
    """make the distance of `rows` NaN against every query"""
    if metric == m.METRIC_Canberra:  # a = b = 0 in one component: 0/0
        xq[:, 0] = 0
        xb[rows, 0] = 0
    elif metric == m.METRIC_JensenShannon:  # a zero component: 0 * log(m / 0)
        xb[rows, rs.randint(0, xb.shape[1], rows.size)] = 0
    elif metric == m.METRIC_GOWER:  # alternately an out-of-range numeric value and a numeric value in a categorical column
        xb[rows[0::2], 0] = 1.5
        xb[rows[1::2], 1] = 0.5
    else:
        raise ValueError(metric)


def case_data(i, metric, d, kind):
    """database rows, queries of case i"""
    rs = np.random.RandomState(2000 + i)
    integer = kind == "int"
    xb = m.metric_data(metric, rs, NB, d, integer)
    xq = m.metric_data(metric, rs, NQ, d, integer)
    if integer and metric == m.METRIC_GOWER:
        for x in (xb, xq):
            x[:, 0::2] = np.floor(x[:, 0::2] * 4) / 4
    if kind == "nan":
        _spoil(metric, rs, xb, xq, rs.permutation(NB)[: NB // 3])
    elif kind == "pad":
        _spoil(metric, rs, xb, xq, rs.permutation(NB)[: NB - 6])
    return xb, xq


def case_k(kind):
    return K_PAD if kind == "pad" else K


def main():
    from oracle import ref_metrics

    out = {
        "cases": np.array([(mt, d, KINDS.index(kind)) for mt, _, d, kind in CASES], dtype=np.int64),
        "args": np.array([a for _, a, _, _ in CASES], dtype=np.float32),
    }
    for i, (mt, arg, d, kind) in enumerate(CASES):
        xb, xq = case_data(i, mt, d, kind)
        D, I = ref_metrics.knn_extra_metrics(xq, xb, case_k(kind), mt, arg)
        out["c%d_D" % i] = D
        out["c%d_I" % i] = I
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


def load():
    """[(case dict)]"""
    z = np.load(OUT)
    cases = []
    for i, ((mt, d, kind), arg) in enumerate(zip(z["cases"], z["args"])):
        kind = KINDS[int(kind)]
        xb, xq = case_data(i, int(mt), int(d), kind)
        cases.append(dict(i=i, metric=int(mt), arg=float(arg), d=int(d), kind=kind, k=case_k(kind), xb=xb, xq=xq,
                          D=z["c%d_D" % i], I=z["c%d_I" % i]))
    return cases


if __name__ == "__main__":
    main()
