"""The numpy restatement of filtered search (oracle/oracle_sel_np.py) against the reference CPU library: the fixture
tests/golden/idselector.npz (minted by tests/golden/make_golden_idselector.py) and, where oracle/_ref was built, the
live reference selectors and searches."""
import os

import numpy as np
import pytest

from oracle import oracle_np as o
from oracle import oracle_sel_np as osel
from tests.golden import make_golden_idselector as g

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "idselector.npz")


@pytest.fixture(scope="module")
def fix():
    return np.load(FIX)


@pytest.fixture(scope="module")
def ref_sel():
    from oracle import ref_sel as r

    if not r.available():
        pytest.skip("oracle/_ref/libfaiss_ref_sel.so not built (needs /root/reference at build time)")
    return r


def test_fixture_inputs_are_reproducible(fix):
    xf, xi, xq, ids = g.data()
    assert np.array_equal(fix["xf"], xf) and np.array_equal(fix["xi"], xi) and np.array_equal(fix["xq"], xq)
    assert np.array_equal(fix["ivf_ids"], ids)
    assert (ids < 0).any() and (ids >= 1 << 40).any()


@pytest.mark.parametrize("metric", list(g.METRICS))
@pytest.mark.parametrize("name", list(osel.reference_selectors(g.NF)))
def test_flat_matches_reference_fixture(fix, name, metric):
    spec = osel.reference_selectors(g.NF)[name]
    D, I = osel.knn_flat_sel(fix["xq"], fix["xf"], g.K, spec, g.METRICS[metric])
    rD, rI = fix["flat_%s_%s_D" % (metric, name)], fix["flat_%s_%s_I" % (metric, name)]
    if metric == "l2":
        assert np.array_equal(I, rI) and np.array_equal(D, rD)
    else:  # the CPU's inner-product heap puts a tie group in decreasing id order
        assert osel.equal_up_to_ties(D, I, rD, rI)


@pytest.mark.parametrize("metric", list(g.METRICS))
@pytest.mark.parametrize("name", list(osel.ivf_selectors(osel.ivf_ids(g.NI))))
def test_ivfflat_matches_reference_fixture(fix, name, metric):
    ids = fix["ivf_ids"]
    spec = osel.ivf_selectors(ids)[name]
    D, I = osel.ivfflat_search_sel(
        fix["xq"], g.K, g.NPROBE, fix["ivf_%s_centroids" % metric], fix["xi"], ids, fix["ivf_%s_assign" % metric], spec,
        g.METRICS[metric])
    rD, rI = fix["ivf_%s_%s_D" % (metric, name)], fix["ivf_%s_%s_I" % (metric, name)]
    assert osel.is_member(spec, rI[rI != -1]).all()
    if metric == "l2":  # integer data: exact distances, ties by id
        assert np.array_equal(I, rI) and np.array_equal(D, rD)
    else:
        assert osel.equal_up_to_ties(D, I, rD, rI)


@pytest.mark.parametrize("name", list(osel.reference_selectors(100)) + ["ivf_" + n for n in osel.ivf_selectors(osel.ivf_ids(300))])
def test_is_member_matches_live_reference(ref_sel, name):
    if name.startswith("ivf_"):
        ids = osel.ivf_ids(300)
        spec = osel.ivf_selectors(ids)[name[4:]]
        probe = np.concatenate([ids, ids + 1, ids - 1])
    else:
        spec = osel.reference_selectors(100)[name]
        probe = np.arange(-20, 130, dtype=np.int64)
    probe = np.concatenate([probe, np.array([-(2**63), -1, 2**40, 2**63 - 1], dtype=np.int64)])
    assert np.array_equal(ref_sel.Selector(spec).is_member(probe), osel.is_member(spec, probe))


def test_fixture_matches_live_reference(ref_sel, fix):
    live = g.reference_results()
    for key, v in live.items():
        assert np.array_equal(v, fix[key]), key
