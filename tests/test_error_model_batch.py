"""CPU model of the fp16 tensor-core Flat path's certificate with ONE query scale for the whole batch
(`tc_query_scale_kernel`, `tc_prepare_queries_kernel`; DESIGN.md 3.1 (i)).  The batch's largest coordinate sets the
power-of-two scale s_q, so next to one large query the elements of every other query land in fp16's subnormal range,
where rounding is off by up to 2^-25 / s_q in absolute terms instead of 2^-11 relative; rows far below the database's
largest meet the same under s_y.  The test restates the arithmetic in numpy (it does not call the product) over batches
with one query 2^20 to 2^40 times an ordinary one (and one 2^-30 times), against rows whose norms spread over 2^20,
and checks for every query
  |approx score - real score| + |exact-kernel fp32 distance - real distance| / 2  <=  eps_q
(for IP the distance is the score and the second term is not halved), the inequality the proof of exactness needs, with
  eps_q = c1 |q| max|y| + c2 (|q| + max|y|)^2 + 1.01 (u_q max|y| + u_y |q| + u_q u_y),   u = sqrt(dpad) 2^-25 / s.
Without the last group (the bound as it was before) the check fails at 2^34."""
import numpy as np
import pytest

F = np.float32
L2, IP = 1, 0


def _pow2_scale(m):
    # max|x| * s in [2^13, 2^14)   (tc_query_scale_kernel / FlatTcDatabase::prepareFp16)
    if m <= 0:
        return 1.0
    e = np.frexp(F(m))[1]
    return float(np.ldexp(1.0, 14 - int(e)))


def _fp16(X, s):
    # __float2half_rn(v * s): np.float16 rounds to nearest even, subnormals included
    return (X * F(s)).astype(np.float16).astype(F)


def _sq_norms(X):
    # a plausible fp32 order: sequential FMA; the constants carry a 1.0001 margin for any order
    acc = np.zeros(X.shape[0], F)
    for i in range(X.shape[1]):
        acc = F(X[:, i].astype(np.float64) ** 2 + acc)
    return acc


def _model(Q, Y, metric):
    """per query: (the left-hand side over all rows, eps with the underflow term, eps without it)"""
    d = Q.shape[1]
    dpad = (d + 63) // 64 * 64
    sq, sy = _pow2_scale(np.abs(Q).max()), _pow2_scale(np.abs(Y).max())
    Q16, Y16 = _fp16(Q, sq), _fp16(Y, sy)
    inv = F(1.0 / (sq * sy))
    yn2 = _sq_norms(Y)
    bias = F(-0.5) * yn2 if metric == L2 else np.zeros_like(yn2)
    # tensor cores: fp16 products are exact in fp32; one plausible accumulation order
    acc = np.zeros((Q.shape[0], Y.shape[0]), F)
    for i in range(d):
        acc = F(acc + np.outer(Q16[:, i], Y16[:, i]))
    approx = F(acc.astype(np.float64) * np.float64(inv) + bias.astype(np.float64))  # fma, one rounding
    # exact kernel: sequential fp32 FMA in dimension order
    dk = np.zeros_like(acc)
    for i in range(d):
        if metric == L2:
            df = F(Q[:, i][:, None] - Y[:, i][None, :]).astype(np.float64)
            dk = F(df * df + dk)
        else:
            dk = F(np.outer(Q[:, i].astype(np.float64), Y[:, i].astype(np.float64)) + dk)
    q64, y64 = Q.astype(np.float64), Y.astype(np.float64)
    dot = q64 @ y64.T
    if metric == L2:
        real_s = dot - 0.5 * (y64 * y64).sum(1)[None, :]
        real_d = (q64 * q64).sum(1)[:, None] + (y64 * y64).sum(1)[None, :] - 2 * dot
        lhs = np.abs(approx - real_s) + np.abs(dk - real_d) / 2
    else:
        lhs = np.abs(approx - dot) + np.abs(dk - dot)
    # the bound, in fp32 as the kernel computes it
    c1 = F(1.01 * (2.0 ** -10 + dpad * 2.0 ** -22))
    c2 = F((dpad + 16) * 2.0 ** -24)
    ymax = F(np.sqrt(yn2.max()) * F(1.0001))
    uq = F(np.sqrt(F(dpad)) * F(2.0 ** -25) / F(sq))
    uy = F(np.sqrt(F(dpad)) * F(2.0 ** -25) / F(sy))
    qn = F(np.sqrt(_sq_norms(Q)) * F(1.0001))
    s = F(qn + ymax)
    old = F(c1 * qn * ymax + c2 * s * s)
    new = F(old + F(1.01) * F(uq * ymax + uy * qn + uq * uy))
    return lhs, new, old


def _data(d, ratio, tiny, seed):
    rs = np.random.RandomState(seed)
    Y = rs.rand(48, d).astype(F)
    Y[::2] *= F(2.0 ** -20)  # half of the rows far below max|y|: their elements underflow under s_y
    Q = rs.randn(8 if tiny else 7, d).astype(F)
    Q[6] *= F(ratio)  # the companion that sets the batch scale
    if tiny:
        Q[7] *= F(2.0 ** -30)
    return Q, Y


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d", [24, 64, 200])
@pytest.mark.parametrize("ratio", [1.0, 2.0 ** 20, 2.0 ** 30, 2.0 ** 34, 2.0 ** 40])
@pytest.mark.parametrize("tiny", [False, True])
def test_batch_scale_certificate_holds(metric, d, ratio, tiny):
    Q, Y = _data(d, ratio, tiny, d + int(np.log2(ratio)) + 100 * tiny + 1000 * metric)
    lhs, eps, _ = _model(Q, Y, metric)
    for qi in range(Q.shape[0]):
        assert (lhs[qi] <= eps[qi]).all(), (qi, lhs[qi].max(), eps[qi])


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d", [24, 64, 200])
def test_bound_without_underflow_term_fails_at_2_34(metric, d):
    """the bound before the underflow term: an ordinary query next to one 2^34 times larger breaks it"""
    Q, Y = _data(d, 2.0 ** 34, False, d + 34 + 1000 * metric)
    lhs, eps, old = _model(Q, Y, metric)
    ordinary = slice(0, 6)
    assert (lhs[ordinary] > old[ordinary, None]).any()
    assert (lhs[ordinary] <= eps[ordinary, None]).all()
