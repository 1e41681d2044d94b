"""CPU tests of the extra-metric restatement (oracle/oracle_metrics_np.py) against the fixture
(tests/golden/metrics.npz) and, where oracle/_ref was built, against the live reference."""
import numpy as np
import pytest

from oracle import oracle_metrics_np as m
from oracle import oracle_np as o
from tests.golden import make_golden_metrics as g


@pytest.fixture(scope="module")
def cases():
    return g.load()


@pytest.fixture(scope="module")
def ref_metrics():
    from oracle import ref_metrics as r

    if not r.available():
        pytest.skip("oracle/_ref/libfaiss_ref_metrics.so not built (needs /root/reference at build time)")
    return r


def _check(c, D, I):
    if c["kind"] == "int" and c["metric"] not in (m.METRIC_Lp, m.METRIC_Canberra, m.METRIC_JensenShannon):
        m.assert_same_knn(c["D"], c["I"], D, I)  # every partial sum is exact: bit for bit
    else:
        o.compare_lists(c["D"], c["I"], D, I, eps=1e-5, pct_max_diff1=0.0, pct_max_diffN=0.0)


def test_fixture_cases(cases):
    assert len(cases) == len(g.CASES)
    for c in cases:
        D, I = m.knn_extra(c["xq"], c["xb"], c["k"], c["metric"], c["arg"])
        _check(c, D, I)


def test_fixture_nan_rows_excluded(cases):
    """NaN rows never appear; fewer valid rows than k pads with (-1, FLT_MAX)"""
    for c in cases:
        if c["kind"] not in ("nan", "pad"):
            continue
        dis = m.pairwise_extra(c["xq"], c["xb"], c["metric"], c["arg"])
        bad = np.isnan(dis)
        assert bad.any(axis=1).all()
        for q in range(c["xq"].shape[0]):
            ids = c["I"][q][c["I"][q] >= 0]
            assert not bad[q, ids].any()
        if c["kind"] == "pad":
            assert (c["I"][:, 6:] == -1).all() and (c["D"][:, 6:] == m.FLT_MAX).all()


@pytest.mark.parametrize("metric,arg", [(m.METRIC_L1, 0.0), (m.METRIC_Linf, 0.0), (m.METRIC_Lp, 0.5), (m.METRIC_Lp, 3.0),
                                        (m.METRIC_Lp, -1.0), (m.METRIC_Canberra, 0.0), (m.METRIC_BrayCurtis, 0.0),
                                        (m.METRIC_JensenShannon, 0.0), (m.METRIC_Jaccard, 0.0), (m.METRIC_GOWER, 0.0)])
@pytest.mark.parametrize("kind", ["float", "int"])
def test_live_reference(ref_metrics, metric, arg, kind):
    """fresh seeds: knn_extra equals the reference's knn_extra_metrics and its IndexFlat of the same metric"""
    rs = np.random.RandomState(metric * 10 + int(arg * 2) + (kind == "int"))
    d = 33
    xb = m.metric_data(metric, rs, 700, d, kind == "int")
    xq = m.metric_data(metric, rs, 9, d, kind == "int")
    if kind == "int" and metric == m.METRIC_GOWER:
        for x in (xb, xq):
            x[:, 0::2] = np.floor(x[:, 0::2] * 4) / 4
    rD, rI = ref_metrics.knn_extra_metrics(xq, xb, 15, metric, arg)
    idx = ref_metrics.IndexFlat(d, metric, arg)
    idx.add(xb)
    fD, fI = idx.search(xq, 15)
    assert np.array_equal(rD, fD) and np.array_equal(rI, fI)
    D, I = m.knn_extra(xq, xb, 15, metric, arg)
    _check(dict(kind=kind, metric=metric, D=rD, I=rI), D, I)


def test_selection_rules():
    """(distance, id) order, larger first for Jaccard, sentinel-valued and NaN distances dropped"""
    dis = np.array([[3, 1, np.nan, 1, m.FLT_MAX, 2]], dtype=np.float32)
    D, I = m.select(dis, 6, m.METRIC_L1)
    assert I.tolist() == [[1, 3, 5, 0, -1, -1]]
    assert D[0, 4] == m.FLT_MAX
    D, I = m.select(dis, 3, m.METRIC_Jaccard)
    assert I.tolist() == [[4, 0, 5]]
    D, I = m.select(np.array([[-m.FLT_MAX, 0.5]], dtype=np.float32), 2, m.METRIC_Jaccard)
    assert I.tolist() == [[1, -1]] and D[0, 1] == -m.FLT_MAX
