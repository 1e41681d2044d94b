"""CPU model of the tensor-core Flat path's rounding certificate (DESIGN.md 3.1, `tc_prepare_queries_kernel`):
fp16 inputs after power-of-two scaling, fp32 accumulation, fp32 bias, one FMA -- against the bound
eps_q = c1*|q|*max|y| + c2*(|q| + max|y|)^2 that the kernel uses to set thresholds.  The test restates the
arithmetic in numpy (it does not call the product) and checks, over norm ratios from 1e-3 to 1e3, that
  |approx score - real score| + |exact-kernel fp32 distance - real distance| / 2  <=  eps_q
which is the inequality the proof of exactness needs."""
import numpy as np
import pytest


def _pow2_scale(m):
    # max|x| * s in [2^13, 2^14)   (tc_query_scale_kernel / FlatTcDatabase::prepare)
    if m <= 0:
        return 1.0
    e = np.frexp(np.float32(m))[1]
    return float(np.ldexp(1.0, 14 - int(e)))


def _seq_sum32(terms):
    acc = np.float32(0)
    for t in terms:
        acc = np.float32(acc + np.float32(t))
    return acc


@pytest.mark.parametrize("d", [24, 64, 128])
@pytest.mark.parametrize("qscale,yscale", [(1.0, 1.0), (1e-3, 1.0), (1.0, 1e-3), (1.0, 300.0), (30.0, 0.02)])
def test_certificate_bound_holds(d, qscale, yscale):
    rs = np.random.RandomState(d + int(1000 * qscale) + int(7 * yscale))
    dpad = (d + 63) // 64 * 64
    nq, n = 6, 40
    Q = (rs.randn(nq, d) * qscale).astype(np.float32)
    Y = (rs.rand(n, d) * yscale).astype(np.float32)
    sq, sy = _pow2_scale(np.abs(Q).max()), _pow2_scale(np.abs(Y).max())
    Q16 = (Q * np.float32(sq)).astype(np.float16)
    Y16 = (Y * np.float32(sy)).astype(np.float16)
    inv = np.float32(1.0 / (sq * sy))
    ynorm2 = np.array([_seq_sum32(np.float32(v) * np.float32(v) for v in row) for row in Y], dtype=np.float32)
    bias = np.float32(-0.5) * ynorm2
    ymax = np.float32(np.sqrt(ynorm2.max()) * 1.0001)
    c1 = np.float32(1.01 * (2.0 ** -10 + dpad * 2.0 ** -22))
    c2 = np.float32((dpad + 16) * 2.0 ** -24)
    for qi in range(nq):
        qn = np.float32(np.sqrt(_seq_sum32(np.float32(v) * np.float32(v) for v in Q[qi])) * 1.0001)
        eps = float(c1 * qn * ymax + c2 * (qn + ymax) * (qn + ymax))
        for j in range(n):
            prods = Q16[qi].astype(np.float32) * Y16[j].astype(np.float32)  # exact in fp32
            acc = _seq_sum32(prods)  # one plausible fp32 accumulation order
            approx = float(np.float32(np.float64(acc) * np.float64(inv) + np.float64(bias[j])))  # fma, one rounding
            real_s = float(np.dot(Q[qi].astype(np.float64), Y[j].astype(np.float64)) - 0.5 * np.dot(Y[j].astype(np.float64), Y[j].astype(np.float64)))
            # exact kernel: sequential fp32 FMA of (q - y)^2 in dimension order
            dk = np.float32(0)
            for a, b in zip(Q[qi], Y[j]):
                df = np.float32(a - b)
                dk = np.float32(np.float64(df) * np.float64(df) + np.float64(dk))
            real_d = float(((Q[qi].astype(np.float64) - Y[j].astype(np.float64)) ** 2).sum())
            lhs = abs(approx - real_s) + abs(float(dk) - real_d) / 2
            assert lhs <= eps, (lhs, eps, qi, j)
