"""CPU self-test of the IVF-SQ inner-product bound (oracle_bound_np.sq_ip_truth).

Accept: a float32 emulation of ivfsq_scan.cu's IP evaluation -- the host's folded decode m = fl(vmin + b / 2),
b = fl(vdiff / s), w_i = fl(q_i b_i), K = sum q_i m_i (fma chains per thread, a 32-lane butterfly, then the 4
warps in order), acc = fma chain sum w_i c_i, value acc + (K + cd) -- stays within the bound against the exact
decode vmin + vdiff (c + 1/2) / s, for every qtype, with cancellation, large |vmin|, uniform and per-dimension
ranges, d up to 300 (two components per thread in K).
Reject: the same emulation with one term dropped (the coarse term, one component) or the level count s a few
ulps off is caught.
"""
import numpy as np
import pytest

from oracle import oracle_bound_np as ob
from oracle import oracle_ivf_check_np as oc
from oracle import oracle_sq_np as osq

f32 = np.float32
THREADS = 128  # 4 warps


def _fma(a, b, c):
    """fl(a * b + c) for float32 arrays: the product of two fp32 values is exact in float64"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def _nudge(x, ulps):
    x = f32(x)
    for _ in range(abs(ulps)):
        x = np.nextafter(x, f32(np.inf) if ulps > 0 else f32(-np.inf))
    return x


def emulate_ip(q, C, vmin, vdiff, s, cd, direct, drop_coarse=False, drop_comp=None, s_ulps=0):
    """the kernel's fp32 value acc + (K + cd) for code values C [n, d] (levels; fp16 / 8bit_direct: the stored
    value).  cd: the coarse term as handed to the kernel (fp32)."""
    q = q.astype(f32)
    n, d = C.shape
    if direct:
        b, m = np.ones(d, f32), np.zeros(d, f32)
    else:
        b = (vdiff.astype(f32) / _nudge(s, s_ulps)).astype(f32)
        m = (vmin.astype(f32) + f32(0.5) * b).astype(f32)
    w = (q * b).astype(f32)
    acc = np.zeros(n, f32)
    for i in range(d):
        if i != drop_comp:
            acc = _fma(w[i], C[:, i].astype(f32), acc)
    part = np.zeros(THREADS, f32)
    for i in range(d):
        part[i % THREADS] = _fma(q[i], m[i], part[i % THREADS])
    warps = part.reshape(4, 32)
    for o in (16, 8, 4, 2, 1):
        warps = (warps + warps[:, np.arange(32) ^ o]).astype(f32)
    K = f32(0)
    for r in warps[:, 0]:
        K = f32(K + r)
    Kp = K if drop_coarse else f32(K + f32(cd))
    return (acc + Kp).astype(f32)


def _case(qtype, d, kind, seed, n=300):
    """(q, C, X exact, vmin, vdiff, s, qc): codes, ranges and a query built to stress the bound"""
    rs = np.random.RandomState(seed)
    s = oc.sq_levels(qtype)
    direct = qtype in (osq.QT_fp16, osq.QT_8bit_direct)
    q = rs.randn(d).astype(f32)
    if kind == "big_vmin":
        q = (np.abs(q) + 0.1).astype(f32)  # same sign everywhere: the m terms add up
    if direct:
        vmin = vdiff = np.zeros(d)
        if qtype == osq.QT_fp16:
            C = (rs.randn(n, d) * (1e3 if kind == "big_vmin" else 1.0)).astype(np.float16).astype(f32)
        else:
            C = rs.randint(0, 256, (n, d)).astype(f32)
        if kind == "cancel":  # pairs of components that cancel: q_{2j+1} = -q_{2j}, equal values
            q[1::2] = -q[: d // 2 * 2 : 2][: d // 2]
            C[:, 1::2] = C[:, : d // 2 * 2 : 2][:, : d // 2]
        X = C.astype(np.float64)
    else:
        uniform = qtype in osq.UNIFORM
        lo = rs.randn(1 if uniform else d) * (1e4 if kind == "big_vmin" else 3.0)
        span = np.abs(rs.randn(1 if uniform else d)) * (0.5 if kind == "big_vmin" else 4.0) + 1e-3
        vmin = np.broadcast_to(lo, (d,)).astype(f32).astype(np.float64)
        vdiff = np.broadcast_to(span, (d,)).astype(f32).astype(np.float64)
        C = rs.randint(0, s + 1, (n, d)).astype(f32)  # levels 0 .. s: 8-bit codes reach 255 = s
        if kind == "cancel":  # q . vmin ~ 0: the large m terms cancel, the truth is small against the bound
            vmin = np.abs(vmin) + 100.0
            q[1::2] = -q[: d // 2 * 2 : 2][: d // 2] * f32(1 + 1e-3)
        X = vmin[None, :] + vdiff[None, :] * (C.astype(np.float64) + 0.5) / s
    qc = float(rs.randn() * (1e3 if kind == "big_vmin" else 10.0))
    return q, C, X, vmin, vdiff, s, qc


QTYPES = [osq.QT_8bit, osq.QT_4bit, osq.QT_8bit_uniform, osq.QT_4bit_uniform, osq.QT_fp16, osq.QT_8bit_direct,
          osq.QT_6bit]


@pytest.mark.parametrize("qtype", QTYPES)
@pytest.mark.parametrize("d", [1, 3, 17, 128, 300])
@pytest.mark.parametrize("kind", ["plain", "big_vmin", "cancel"])
@pytest.mark.parametrize("residual", [False, True])
def test_sq_ip_bound_holds(qtype, d, kind, residual):
    q, C, X, vmin, vdiff, s, qc = _case(qtype, d, kind, seed=qtype * 1000 + d * 7 + len(kind) + residual)
    qc = qc if residual else 0.0
    direct = qtype in (osq.QT_fp16, osq.QT_8bit_direct)
    V = emulate_ip(q, C, vmin, vdiff, s, f32(qc), direct)
    t, beta = ob.sq_ip_truth(q, X, vmin, vdiff, s, qc)
    err = np.abs(V.astype(np.float64) - t)
    assert np.all(err <= beta), "max |err| / bound %.3f" % float((err / beta).max())


@pytest.mark.parametrize("qtype", [osq.QT_8bit, osq.QT_4bit, osq.QT_6bit, osq.QT_fp16])
def test_sq_ip_bound_catches_dropped_coarse_term(qtype):
    q, C, X, vmin, vdiff, s, qc = _case(qtype, 64, "plain", seed=qtype)
    V = emulate_ip(q, C, vmin, vdiff, s, f32(qc), qtype == osq.QT_fp16, drop_coarse=True)
    t, beta = ob.sq_ip_truth(q, X, vmin, vdiff, s, qc)
    assert np.all(np.abs(V - t) > beta)


@pytest.mark.parametrize("qtype", [osq.QT_8bit, osq.QT_4bit_uniform, osq.QT_6bit, osq.QT_8bit_direct])
def test_sq_ip_bound_catches_dropped_component(qtype):
    q, C, X, vmin, vdiff, s, qc = _case(qtype, 32, "plain", seed=qtype + 50)
    q[5] = f32(50.0)  # the dropped component weighs more than the bound
    C[:, 5] = np.maximum(C[:, 5], f32(1))
    if qtype != osq.QT_8bit_direct:
        X = vmin[None, :] + vdiff[None, :] * (C.astype(np.float64) + 0.5) / s
    else:
        X = C.astype(np.float64)
    V = emulate_ip(q, C, vmin, vdiff, s, f32(qc), qtype == osq.QT_8bit_direct, drop_comp=5)
    t, beta = ob.sq_ip_truth(q, X, vmin, vdiff, s, qc)
    assert np.all(np.abs(V - t) > beta)


@pytest.mark.parametrize("qtype", [osq.QT_8bit, osq.QT_4bit, osq.QT_6bit])
def test_sq_ip_bound_catches_levels_a_few_ulps_off(qtype):
    """one decode constant off: every b_i = vdiff_i / s moves by ~16 ulps, each term q_i b_i c_i with it.  At d = 1
    with the top levels and vmin = 0 the bound is about 7 ulps of the value."""
    s = oc.sq_levels(qtype)
    rs = np.random.RandomState(qtype)
    n = 200
    q = (np.abs(rs.randn(n, 1)) + 0.5).astype(f32)
    vmin, vdiff = np.zeros(1), np.array([f32(3.7)], np.float64)
    C = np.full((n, 1), s - 1, f32)
    X = vmin[None, :] + vdiff[None, :] * (C.astype(np.float64) + 0.5) / s
    for qi in range(4):
        ok = emulate_ip(q[qi], C, vmin, vdiff, s, f32(0), False)
        off = emulate_ip(q[qi], C, vmin, vdiff, s, f32(0), False, s_ulps=-16)
        t, beta = ob.sq_ip_truth(q[qi], X, vmin, vdiff, s)
        assert np.all(np.abs(ok - t) <= beta)
        assert np.all(np.abs(off - t) > beta), "ratio %.2f" % float((np.abs(off - t) / beta).min())
