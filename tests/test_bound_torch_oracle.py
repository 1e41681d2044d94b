"""Self-test of the device certifier (oracle/oracle_bound_torch.certify_knn) against the numpy checker it scales up
(oracle/oracle_bound_np.check_knn, with exact_topk for exact mode).

Both must accept correct results -- fp32 distances in the (key, id) order, as the kernels return them -- on L2 and
inner-product cases, with query blocks and row chunks of 1, 7 and everything, so that block edges fall everywhere.
Both must reject every planted defect.  The CPU cases run on torch CPU tensors; one GPU case repeats the agreement
with CUDA tensors, so that the cuBLAS DGEMM truth is under the same test.
"""
import itertools

import numpy as np
import pytest

from oracle import oracle_bound_np as ob
from oracle import oracle_bound_torch as obt

L2, IP = ob.METRIC_L2, ob.METRIC_INNER_PRODUCT
f32 = np.float32
N, NQ, DIM, K = 300, 24, 24, 16


def _data(kind, metric, seed, n=N, nq=NQ, d=DIM):
    rs = np.random.RandomState(seed)
    if kind == "int":  # few values in few dimensions: tie groups everywhere, rank k included
        xb = rs.randint(-2, 3, (n, 4)).astype(f32)
        xq = rs.randint(-2, 3, (nq, 4)).astype(f32)
        return xb, xq
    if kind == "gauss" or metric == IP:
        return rs.randn(n, d).astype(f32), rs.randn(nq, d).astype(f32)
    return rs.rand(n, d).astype(f32), rs.rand(nq, d).astype(f32)


def _result(xq, xb, k, metric, mask=None):
    """fp32 distances (one rounding per product and per addition), the top k of each query in the (key, id) order,
    padded with -1 and the sentinel"""
    if metric == L2:
        Dall = ((xq[:, None, :] - xb[None, :, :]) ** 2).sum(-1, dtype=f32)
    else:
        Dall = (xq @ xb.T).astype(f32)
    ids = np.arange(xb.shape[0]) if mask is None else np.nonzero(mask)[0]
    D = np.full((xq.shape[0], k), ob.FLT_MAX if metric == L2 else -ob.FLT_MAX, f32)
    I = np.full((xq.shape[0], k), -1, np.int64)
    for qi in range(xq.shape[0]):
        key = Dall[qi, ids] if metric == L2 else -Dall[qi, ids]
        o = np.lexsort((ids, key))[:k]
        D[qi, : o.size] = Dall[qi, ids[o]]
        I[qi, : o.size] = ids[o]
    return D, I


def _truth(xq, xb, metric):
    return ob.l2_truth_many(xq, xb) if metric == L2 else ob.ip_truth_many(xq, xb)


def np_verdict(D, I, xq, xb, k, metric, mask=None, exact=False):
    """None if check_knn (and, exact, exact_topk) accept, else the message"""
    ids = np.arange(xb.shape[0]) if mask is None else np.nonzero(mask)[0]
    T, B = _truth(xq, xb[ids], metric)
    if exact:
        B = np.zeros_like(T)
    try:
        ob.check_knn(D, I, ids, T, B, k, metric)
        if exact:
            for qi in range(xq.shape[0]):
                eD, eI = ob.exact_topk(T[qi], ids, k, metric)
                if not (np.array_equal(D[qi], eD) and np.array_equal(I[qi], eI)):
                    raise ob.CertificateError("query %d is not the exact top-k" % qi)
    except ob.CertificateError as e:
        return str(e)
    return None


def torch_verdict(D, I, xq, xb, k, metric, mask=None, exact=False, qb=None, rc=None, device="cpu"):
    import torch

    Y = torch.from_numpy(xb).to(device)
    Q = torch.from_numpy(xq).to(device)
    m = None if mask is None else torch.from_numpy(mask).to(device)
    try:
        obt.certify_knn(torch.from_numpy(D).to(device), torch.from_numpy(I).to(device), Q, Y, k, metric, candidates=m,
                        exact=exact, q_block=qb or xq.shape[0], row_chunk=rc or xb.shape[0])
    except ob.CertificateError as e:
        return str(e)
    return None


# ------------------------------------------------------------------ accept
BLOCKS = [1, 7, None]  # None: the whole query set / database in one block


@pytest.mark.parametrize("qb,rc", list(itertools.product(BLOCKS, BLOCKS)))
@pytest.mark.parametrize("metric,kind", [(L2, "uniform"), (IP, "gauss"), (L2, "int"), (IP, "int")])
def test_both_accept_correct_results(metric, kind, qb, rc):
    xb, xq = _data(kind, metric, seed=3 + metric)
    D, I = _result(xq, xb, K, metric)
    exact = kind == "int"
    assert np_verdict(D, I, xq, xb, K, metric, exact=exact) is None
    assert torch_verdict(D, I, xq, xb, K, metric, exact=exact, qb=qb, rc=rc) is None


@pytest.mark.parametrize("metric", [L2, IP])
def test_both_accept_masked_and_padded_results(metric):
    xb, xq = _data("uniform", metric, seed=11)
    rs = np.random.RandomState(5)
    for sel in (150, K, 10, 0):  # more than k, exactly k, fewer than k (-1 padding), none
        mask = np.zeros(N, bool)
        mask[rs.choice(N, sel, replace=False)] = True
        D, I = _result(xq, xb, K, metric, mask)
        assert np_verdict(D, I, xq, xb, K, metric, mask) is None, sel
        for qb, rc in ((7, 7), (None, None)):
            assert torch_verdict(D, I, xq, xb, K, metric, mask, qb=qb, rc=rc) is None, sel


def test_exact_mode_refuses_data_outside_its_regime():
    import torch

    xb, xq = _data("uniform", L2, seed=2)
    D, I = _result(xq, xb, K, L2)
    with pytest.raises(ValueError, match="integer"):
        obt.certify_knn(D, I, torch.from_numpy(xq), torch.from_numpy(xb), K, L2, exact=True)
    big = np.rint(xb * 2000).astype(f32)  # integers whose squared sums pass 2^24
    D, I = _result(xq * 0, big, K, L2)
    with pytest.raises(ValueError, match="2\\^24"):
        obt.certify_knn(D, I, torch.from_numpy(xq * 0), torch.from_numpy(big), K, L2, exact=True)


# ------------------------------------------------------------------ reject
def _sorted_truth(xq, xb, metric, qi):
    """(float64 truth, ids) of query qi in the (key, id) order"""
    T, _ = _truth(xq[qi:qi + 1], xb, metric)
    t = T[0]
    key = t if metric == L2 else -t
    o = np.lexsort((np.arange(t.size), key))
    return t[o], o


def _swap_member(D, I, xq, xb, metric):
    """the query whose ranks k and k+1 are farthest apart: its k-th member replaced by the (k+1)-th"""
    gaps = []
    for qi in range(xq.shape[0]):
        t, _ = _sorted_truth(xq, xb, metric, qi)
        gaps.append(abs(t[K] - t[K - 1]))
    qi = int(np.argmax(gaps))
    t, o = _sorted_truth(xq, xb, metric, qi)
    I[qi, K - 1] = o[K]
    D[qi, K - 1] = f32(t[K])


def _swap_two(D, I, xq, xb, metric):
    qi = 5
    j = int(np.nonzero(D[qi, 1:] != D[qi, :-1])[0][0])
    D[qi, [j, j + 1]] = D[qi, [j + 1, j]]
    I[qi, [j, j + 1]] = I[qi, [j + 1, j]]


def _past_bound(D, I, xq, xb, metric):
    """the last entry's distance moved to the first float32 beyond its bound (away from the others: the order holds)"""
    qi = 9
    T, B = _truth(xq[qi:qi + 1], xb[I[qi, K - 1]][None, :], metric)
    t, b = float(T[0, 0]), float(B[0, 0])
    if metric == L2:
        v = f32(t + 1.01 * b)
        while float(v) <= t + 1.01 * b:
            v = np.nextafter(v, f32(np.inf))
    else:
        v = f32(t - 1.01 * b)
        while float(v) >= t - 1.01 * b:
            v = np.nextafter(v, f32(-np.inf))
    D[qi, K - 1] = v


def _duplicate(D, I, xq, xb, metric):
    I[2, 1] = I[2, 0]


def _minus_one(D, I, xq, xb, metric):
    I[4, 3] = -1


def _bad_padding(D, I, xq, xb, metric):
    assert I[6, K - 1] == -1
    D[6, K - 1] = np.inf if metric == L2 else -np.inf


def _tie_descending(D, I, xq, xb, metric):
    for qi in range(xq.shape[0]):
        j = np.nonzero(D[qi, 1:] == D[qi, :-1])[0]
        if j.size:
            j = int(j[0])
            I[qi, [j, j + 1]] = I[qi, [j + 1, j]]
            return
    raise AssertionError("no tie to plant the defect in")


def _outside_mask(D, I, xq, xb, metric, mask):
    I[7, K - 2] = int(np.nonzero(~mask)[0][0])


def _wrong_tie_member(D, I, xq, xb, metric):
    """a query whose rank-k tie group runs past k: its last entry replaced by a larger id of the same group"""
    for qi in range(xq.shape[0]):
        t, o = _sorted_truth(xq, xb, metric, qi)
        if t[K - 1] == t[K]:
            assert I[qi, K - 1] == o[K - 1]
            I[qi, K - 1] = o[K]
            return
    raise AssertionError("no tie group at rank k")


# (name, metric, data, mask rows selected (None: no mask), exact, defect)
DEFECTS = [
    ("swap_member", L2, "uniform", None, False, _swap_member),
    ("swap_member", IP, "gauss", None, False, _swap_member),
    ("swap_two", L2, "uniform", None, False, _swap_two),
    ("swap_two", IP, "gauss", None, False, _swap_two),
    ("past_bound", L2, "uniform", None, False, _past_bound),
    ("past_bound", IP, "gauss", None, False, _past_bound),
    ("duplicate", L2, "uniform", None, False, _duplicate),
    ("minus_one", IP, "gauss", None, False, _minus_one),
    ("bad_padding", L2, "uniform", 10, False, _bad_padding),
    ("bad_padding", IP, "gauss", 10, False, _bad_padding),
    ("tie_descending", L2, "int", None, True, _tie_descending),
    ("tie_descending", L2, "int", None, False, _tie_descending),
    ("outside_mask", L2, "uniform", 150, False, _outside_mask),
    ("outside_mask", IP, "gauss", 150, False, _outside_mask),
    ("wrong_tie_member", L2, "int", None, True, _wrong_tie_member),
    ("wrong_tie_member", IP, "int", None, True, _wrong_tie_member),
]


def _planted(metric, kind, sel, exact, defect):
    xb, xq = _data(kind, metric, seed=17 + metric)
    mask = None
    if sel is not None:
        mask = np.zeros(N, bool)
        mask[np.random.RandomState(1).choice(N, sel, replace=False)] = True
    D, I = _result(xq, xb, K, metric, mask)
    assert np_verdict(D, I, xq, xb, K, metric, mask, exact) is None  # correct before the defect
    if defect is _outside_mask:
        defect(D, I, xq, xb, metric, mask)
    else:
        defect(D, I, xq, xb, metric)
    return D, I, xq, xb, mask


@pytest.mark.parametrize("name,metric,kind,sel,exact,defect", DEFECTS,
                         ids=["%s-%s%s" % (c[0], "l2" if c[1] == L2 else "ip", "-exact" if c[4] else "") for c in DEFECTS])
def test_both_reject_planted_defects(name, metric, kind, sel, exact, defect):
    D, I, xq, xb, mask = _planted(metric, kind, sel, exact, defect)
    assert np_verdict(D, I, xq, xb, K, metric, mask, exact) is not None, "numpy checker accepted %s" % name
    for qb, rc in ((1, 1), (7, 7), (None, None), (7, None)):
        v = torch_verdict(D, I, xq, xb, K, metric, mask, exact, qb, rc)
        assert v is not None, "certify_knn accepted %s (blocks %s x %s)" % (name, qb, rc)


def test_wrong_tie_member_passes_without_exact_mode():
    """the rank-k tie group's membership is free under a positive bound: only exact mode pins it"""
    D, I, xq, xb, mask = _planted(L2, "int", None, True, _wrong_tie_member)
    assert torch_verdict(D, I, xq, xb, K, L2, exact=False) is None
    assert torch_verdict(D, I, xq, xb, K, L2, exact=True) is not None


@pytest.mark.gpu
def test_agreement_on_cuda_tensors():
    """the same accept and reject cases with the truth on the device (cuBLAS DGEMM)"""
    for metric, kind in ((L2, "uniform"), (IP, "gauss"), (L2, "int")):
        xb, xq = _data(kind, metric, seed=3 + metric)
        D, I = _result(xq, xb, K, metric)
        for qb, rc in ((7, 7), (None, None)):
            assert torch_verdict(D, I, xq, xb, K, metric, exact=kind == "int", qb=qb, rc=rc, device="cuda") is None
    for name, metric, kind, sel, exact, defect in DEFECTS:
        D, I, xq, xb, mask = _planted(metric, kind, sel, exact, defect)
        assert np_verdict(D, I, xq, xb, K, metric, mask, exact) is not None, name
        for qb, rc in ((7, 7), (None, None)):
            assert torch_verdict(D, I, xq, xb, K, metric, mask, exact, qb, rc, device="cuda") is not None, name
