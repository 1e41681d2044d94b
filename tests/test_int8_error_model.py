"""CPU model of the int8 certificate of the tensor-core Flat L2 search (DESIGN.md 3.1, `tc_prepare_rows8_kernel`,
`tc_prepare_queries8_kernel`): the rows and queries are centred on the per-dimension midrange c, quantised to int8 with
one database scale and one scale per query, multiplied exactly in int32 and scored as fma(acc, inv, -|y - c|^2 / 2).
The test restates that arithmetic in numpy (it does not call the product) and checks
  |approx score - real centred score| + |exact-kernel fp32 distance - real distance| / 2  <=  eps_q
which is the inequality the proof of exactness needs, over dimensions 113 to 128, spreads of query and row scales,
data far from the origin and values that sit on rounding half-steps."""
import numpy as np
import pytest

F = np.float32


def _q8(v, s):
    return np.clip(np.rint(F(v * F(s))), -127, 127).astype(np.int64)


def _norm(v):
    # a plausible fp32 order: sequential FMA; the constants carry a 1.0001 margin for any order
    acc = F(0)
    for x in v:
        acc = F(np.float64(x) * np.float64(x) + np.float64(acc))
    return acc


def _model(Y, Q):
    n, d = Y.shape
    lo, hi = Y.min(0), Y.max(0)
    c = F(F(0.5) * lo) + F(F(0.5) * hi)
    Yc = F(Y - c)
    sy = F(F(127) / np.abs(Yc).max())
    Y8 = _q8(Yc, sy)
    yc2 = np.array([_norm(r) for r in Yc], dtype=F)
    bias = F(-0.5) * yc2
    maxYhat = F(np.sqrt(F((Y8 * Y8).sum(1).max())) / sy * F(1.0001))
    Ry = F(Yc - F(Y8.astype(F) / sy))
    maxRy = F(np.sqrt(max(_norm(r) for r in Ry)) * F(1.0001))
    maxYc = F(np.sqrt(yc2.max()) * F(1.0001))
    c2 = F((128 + 16) * 2.0 ** -24)
    out = []
    for q in Q:
        qc = F(q - c)
        sq = F(F(127) / np.abs(qc).max())
        Q8 = _q8(qc, sq)
        qh = F(F(np.sqrt(F((Q8 * Q8).sum()))) / sq * F(1.0001))
        rq = F(np.sqrt(_norm(F(qc - F(Q8.astype(F) / sq)))) * F(1.0001))
        qcn = F(np.sqrt(_norm(qc)) * F(1.0001))
        s = F(qcn + maxYc)
        eps = float(F(F(qh * maxRy + rq * maxYhat + rq * maxRy) * F(1.0001)) + F(2.0 ** -20) * qh * maxYhat + c2 * s * s)
        inv = F(F(1) / F(sq * sy))
        acc = Y8 @ Q8  # exact, |acc| < 2^24
        approx = F(acc.astype(np.float64) * np.float64(inv) + bias.astype(np.float64))  # fma, one rounding
        q64, y64, c64 = q.astype(np.float64), Y.astype(np.float64), c.astype(np.float64)
        real_s = (y64 - c64) @ (q64 - c64) - 0.5 * ((y64 - c64) ** 2).sum(1)
        # exact kernel: sequential fp32 FMA of (q - y)^2 in dimension order
        dk = np.zeros(n, dtype=F)
        for i in range(d):
            df = F(q[i] - Y[:, i])
            dk = F(df.astype(np.float64) * df + dk.astype(np.float64))
        real_d = ((q64 - y64) ** 2).sum(1)
        lhs = np.abs(approx.astype(np.float64) - real_s) + np.abs(dk.astype(np.float64) - real_d) / 2
        out.append((lhs, eps))
    return out


@pytest.mark.parametrize("d", [113, 120, 128])
@pytest.mark.parametrize("qscale,yscale", [(1.0, 1.0), (1e-3, 1.0), (1.0, 1e-3), (1.0, 300.0), (30.0, 0.02)])
def test_int8_certificate_holds(d, qscale, yscale):
    rs = np.random.RandomState(d + int(1000 * qscale) + int(7 * yscale))
    Y = (rs.rand(48, d) * yscale).astype(F)
    Q = (rs.randn(6, d) * qscale).astype(F)
    for lhs, eps in _model(Y, Q):
        assert (lhs <= eps).all(), (lhs.max(), eps)


@pytest.mark.parametrize("d", [113, 120, 128])
def test_int8_certificate_holds_far_from_origin(d):
    rs = np.random.RandomState(d)
    Y = (1000.0 + rs.rand(48, d)).astype(F)
    Q = (1000.0 + rs.rand(6, d)).astype(F)
    for lhs, eps in _model(Y, Q):
        assert (lhs <= eps).all(), (lhs.max(), eps)


@pytest.mark.parametrize("d", [113, 120, 128])
def test_int8_certificate_holds_on_half_steps(d):
    # every dimension spans [-63.5, 63.5]: c = 0 and s_y = 2 exactly, and y * s_y lands on m + 0.5
    rs = np.random.RandomState(d + 1)
    Y = ((rs.randint(-127, 127, size=(48, d)) + 0.5) / 2).astype(F)
    Y[0, :], Y[1, :] = -63.5, 63.5
    Q = ((rs.randint(-127, 127, size=(6, d)) + 0.5) / 2).astype(F)
    Q[:, 0] = 63.5  # s_q = 2 as well
    for lhs, eps in _model(Y, Q):
        assert (lhs <= eps).all(), (lhs.max(), eps)
