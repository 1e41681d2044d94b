"""The tensor-core Flat search at hostile magnitudes (DESIGN.md 3.1, *Certificate*).

The fp16 path scales a whole query batch by one power of two, taken from the batch's largest coordinate, so one
large query pushes the elements of every other query of the batch towards fp16's subnormal range.  The certificate
eps_q must cover that, or an ordinary query loses a true top-k member without any overflow flagging it.  Here:
  * a query's (D, I) must be the same whether it is searched alone or next to a hostile companion (2^34, 2^40,
    2^-30 times an ordinary query, or the zero vector), and the whole batch must equal the exact kernel's result;
  * on hostile databases (far from the origin, rounding half-steps, scale spreads, a constant column, a query on the
    int8 centre, identical rows, inf and NaN), both the fp16 and the int8 path must equal the exact kernel, and the
    fitness test must pick the expected operand width;
  * an IVF `add` next to a vector of 1e10s or 1e12s must still put every other vector in its exact nearest list.
Every case asserts that it ran on the tensor cores, so none quietly tests only the exact kernel."""
import numpy as np
import pytest

from oracle import oracle_bound_np as ob

pytestmark = pytest.mark.gpu

L2, IP = 1, 0
N, NQ = 50000, 64

# name: (d, metric, k, fp16 storage, database rows, operand bits)
CONFIGS = {
    "fp16_l2": (64, L2, 10, False, N, 16),
    "fp16_ip": (64, IP, 10, False, N, 16),
    "ksplit": (200, L2, 100, False, N, 16),
    "large_k": (96, L2, 1024, False, N, 16),
    "streaming": (64, L2, 1, False, 4096, 16),
    "fp16_storage": (64, L2, 10, True, N, 16),
    "int8": (128, L2, 100, False, N, 8),
}
# the companion query: a scale of an ordinary query, or 0 for the zero vector
COMPANIONS = [2.0 ** 34, 2.0 ** 40, 2.0 ** -30, 0.0]
# fp16 storage keeps the companion within fp16 range: 6e4 against queries at 1e-3
STORAGE_QSCALE, STORAGE_COMPANIONS = 1e-3, [6e4, 2.0 ** -30, 0.0]

@pytest.fixture(scope="module")
def indexes():
    """each config's index and its data, built once and freed with the module"""
    return {}


def _index(res, indexes, name):
    if name not in indexes:
        import faiss_b200 as fb

        d, metric, k, fp16, n, bits = CONFIGS[name]
        rs = np.random.RandomState(d + k + 7 * fp16)
        xb = rs.rand(n, d).astype(np.float32)
        idx = fb.GpuIndexFlat(res, d, metric, use_float16=fp16)
        idx.add(xb)
        if fp16:
            xb = xb.astype(np.float16).astype(np.float32)  # what the index stores
        xq = rs.rand(NQ, d).astype(np.float32) * np.float32(STORAGE_QSCALE if fp16 else 1.0)
        indexes[name] = (idx, xb, xq)
    return indexes[name]


def _tc_search(idx, xq, k, bits):
    D, I = idx.search(xq, k)
    info = idx.lastSearchInfo()
    assert info["tensor_cores"] == 1, info
    assert idx.lastSearchOperandBits() == bits
    return D, I, info


def _exact(idx, xq, k):
    idx.setUseTensorCores(False)
    try:
        D, I = idx.search(xq, k)
        assert idx.lastSearchInfo()["tensor_cores"] == 0
        assert idx.lastSearchOperandBits() == 0
    finally:
        idx.setUseTensorCores(True)
    return D, I


def _assert_same(D, I, De, Ie, what=""):
    assert np.array_equal(I, Ie), "%s: ids differ in queries %s" % (what, np.nonzero((I != Ie).any(1))[0][:10])
    assert np.array_equal(D, De, equal_nan=True), "%s: distances differ in queries %s" % (
        what, np.nonzero((D != De).any(1))[0][:10])


def _params():
    out = []
    for name, cfg in CONFIGS.items():
        for comp in (STORAGE_COMPANIONS if cfg[3] else COMPANIONS):
            out.append(pytest.param(name, comp, id="%s-%s" % (name, "zero" if comp == 0 else "2^%g" % np.log2(comp))))
    return out


@pytest.mark.parametrize("name", list(CONFIGS))
def test_alone_is_certified_against_float64(res, indexes, name):
    """the ordinary batch by itself: the exact kernel's result, certified against float64, with no fallback"""
    d, metric, k, fp16, n, bits = CONFIGS[name]
    idx, xb, xq = _index(res, indexes, name)
    D, I, info = _tc_search(idx, xq, k, bits)
    assert info["fallback_queries"] == 0, info
    _assert_same(D, I, *_exact(idx, xq, k), what=name)
    T, B = (ob.l2_truth_many if metric == L2 else ob.ip_truth_many)(xq, xb)
    ob.check_knn(D, I, np.arange(n), T, B, k, metric, what=name)


@pytest.mark.parametrize("name,comp", _params())
def test_companion_does_not_change_other_queries(res, indexes, name, comp):
    d, metric, k, fp16, n, bits = CONFIGS[name]
    idx, xb, xq = _index(res, indexes, name)
    D0, I0, _ = _tc_search(idx, xq, k, bits)
    rs = np.random.RandomState(11)
    c = (rs.rand(1, d) * comp).astype(np.float32)
    h = NQ // 2  # the companion sits inside the ordinary queries' 128-query tile
    batch = np.vstack([xq[:h], c, xq[h:]])
    D, I, _ = _tc_search(idx, batch, k, bits)
    rows = np.r_[0:h, h + 1:NQ + 1]
    _assert_same(D[rows], I[rows], D0, I0, what="%s next to %g" % (name, comp))
    _assert_same(D, I, *_exact(idx, batch, k), what="%s batch with %g" % (name, comp))


# ---------------------------------------------------------------------------------------------- hostile data
# path: (d, k, operand bits when the database is fit for int8)
PATHS = {"fp16": (64, 10), "int8": (128, 100)}
HN, HQ = 40000, 48


def _centre(xb):
    """the int8 layout's centre: the per-dimension midrange, rounded as the device rounds it"""
    f = np.float32
    return f(f(0.5) * xb.min(0)) + f(f(0.5) * xb.max(0))


def _half_steps(rs, d, frac):
    """values m / 2 with every dimension spanning [-63.5, 63.5] (the int8 scale is then 2 exactly); a fraction
    `frac` of the coordinates sit on m + 0.5 halves, where y * s_y lands on a rounding half-step"""
    xb = (rs.randint(-127, 128, size=(HN, d)) / 2).astype(np.float32)
    half = rs.rand(HN, d) < frac
    xb[half] = ((rs.randint(-127, 127, size=int(half.sum())) + 0.5) / 2).astype(np.float32)
    xb[0, :], xb[1, :] = -63.5, 63.5
    xq = ((rs.randint(-127, 127, size=(HQ, d)) + 0.5) / 2).astype(np.float32)
    xq[:, 0] = 63.5
    return xb, xq


def _hostile(case, d):
    """(rows, queries, fit for int8) of one hostile case"""
    rs = np.random.RandomState(d * 100 + len(case))
    u = lambda *s: rs.rand(*s).astype(np.float32)  # noqa: E731
    if case in ("far_1e3", "far_1e4"):
        off = np.float32(1e3 if case == "far_1e3" else 1e4)
        return off + u(HN, d), off + u(HQ, d), True
    if case == "half_steps":  # every coordinate on a half-step: max |r_y| fails the int8 fitness test
        return _half_steps(rs, d, 1.0) + (False,)
    if case == "some_half_steps":  # a tenth of them: fit
        return _half_steps(rs, d, 0.1) + (True,)
    if case == "q_1e-3":
        return u(HN, d), (rs.randn(HQ, d) * 1e-3).astype(np.float32), True
    if case == "y_300":
        return u(HN, d) * np.float32(300), rs.randn(HQ, d).astype(np.float32), True
    if case == "q_30_y_0.02":
        return u(HN, d) * np.float32(0.02), (rs.randn(HQ, d) * 30).astype(np.float32), True
    if case == "constant_column":
        xb = u(HN, d)
        xb[:, 5] = 0.7
        return xb, u(HQ, d), True
    if case == "query_on_centre":  # q - c = 0: the a == 0 branch of the int8 query preparation
        xb, xq = u(HN, d), u(HQ, d)
        xq[3] = _centre(xb)
        return xb, xq, True
    if case == "identical_rows":  # all scores tie: the certificate cannot separate them
        return np.repeat(u(1, d), HN, axis=0), u(HQ, d), True
    if case == "inf_row":
        xb = u(HN, d)
        xb[123, 7] = np.inf
        return xb, u(HQ, d), False
    if case == "nan_row":
        xb = u(HN, d)
        xb[4567, 0] = np.nan
        return xb, u(HQ, d), False
    if case == "nan_query":
        xq = u(HQ, d)
        xq[5, 9] = np.nan
        return u(HN, d), xq, True
    raise ValueError(case)


HOSTILE = ["far_1e3", "far_1e4", "half_steps", "some_half_steps", "q_1e-3", "y_300", "q_30_y_0.02",
           "constant_column", "query_on_centre", "identical_rows", "inf_row", "nan_row", "nan_query"]


@pytest.mark.parametrize("case", HOSTILE)
@pytest.mark.parametrize("path", list(PATHS))
def test_hostile_data_equals_exact(res, path, case):
    import faiss_b200 as fb

    d, k = PATHS[path]
    xb, xq, fit = _hostile(case, d)
    bits = 8 if path == "int8" and fit else 16
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    D, I, info = _tc_search(idx, xq, k, bits)
    _assert_same(D, I, *_exact(idx, xq, k), what="%s %s" % (path, case))
    if case == "identical_rows":
        assert info["fallback_queries"] > 0, info
        assert (I == np.arange(k)).all()
    if case == "nan_query":  # no distance to a NaN query is better than another: no result
        assert (I[5] == -1).all()
        assert (np.delete(I, 5, axis=0) >= 0).all()


@pytest.mark.parametrize("huge", [1e10, 1e12])
def test_ivf_add_next_to_a_huge_vector_assigns_exact_lists(res, huge):
    """the coarse assignment of `add` runs the k = 1 streaming search over 2048 centroids, all vectors of one `add`
    in one query batch: a vector of 1e10s (or 1e12s, about 2^38 times the others) in it must not move any other
    vector to a list that is not its nearest"""
    import faiss_b200 as fb

    rs = np.random.RandomState(3)
    d, nlist = 64, 2048
    centres = rs.rand(256, d).astype(np.float32) * 4
    clustered = lambda n: (centres[rs.randint(0, 256, n)] + 0.1 * rs.randn(n, d)).astype(np.float32)  # noqa: E731
    ivf = fb.GpuIndexIVFFlat(res, d, nlist)
    ivf.setClustering(niter=4)
    ivf.train(clustered(nlist * 40))
    xb = clustered(20000)
    ivf.add(np.vstack([np.full((1, d), huge, dtype=np.float32), xb]))  # ids 1 .. 20000 are the ordinary vectors
    got = np.full(xb.shape[0] + 1, -1, dtype=np.int64)
    for l in range(nlist):
        got[ivf.getListIndices(l)] = l
    assert (got >= 0).all()
    exact = fb.GpuIndexFlatL2(res, d, use_tensor_cores=False)
    exact.add(ivf.getCoarseCentroids())
    _, I = exact.search(xb, 1)
    wrong = np.nonzero(got[1:] != I[:, 0])[0]
    assert wrong.size == 0, "%d vectors in the wrong list, e.g. %s" % (wrong.size, wrong[:10])
