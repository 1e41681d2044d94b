"""tests/golden/pairwise.npz against the CPU restatements in numpy (no GPU): oracle_np.pairwise and
oracle_metrics_np.pairwise_extra, and against the live reference CPU library where oracle/_ref is built."""
import os

import numpy as np
import pytest

from oracle import oracle_metrics_np as m
from tests.golden import make_golden_pairwise as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT_INT = ("L2", "IP", "L1", "Linf", "Lp1", "Lp2", "BrayCurtis", "Jaccard")


@pytest.fixture(scope="module")
def fixture():
    return np.load(os.path.join(ROOT, "tests", "golden", "pairwise.npz"))


def _close(got, want, what):
    nan = np.isnan(want)
    assert np.array_equal(nan, np.isnan(got)), what
    np.testing.assert_allclose(got[~nan], want[~nan], rtol=1e-5, atol=1e-6, err_msg=what)


@pytest.mark.parametrize("i,name,metric,arg", [(i,) + c for i, c in enumerate(g.CASES)], ids=[c[0] for c in g.CASES])
def test_fixture_matches_numpy(fixture, i, name, metric, arg):
    for kind in ("int", "float"):
        key = "%s_%s" % (name, kind)
        xq, xb = g.case_data(i, metric, kind)
        assert np.array_equal(fixture[key + "_xq"], xq) and np.array_equal(fixture[key + "_xb"], xb), key
        want = g.numpy_pairwise(xq, xb, metric, arg)
        if kind == "int" and name in EXACT_INT:
            assert np.array_equal(fixture[key + "_D"], want), key
        else:
            _close(fixture[key + "_D"], want, key)


def test_fixture_has_nan_entries(fixture):
    for name in ("Canberra", "JensenShannon"):
        assert np.isnan(fixture[name + "_float_D"]).any(), name


@pytest.mark.parametrize("i,name,metric,arg", [(i,) + c for i, c in enumerate(g.CASES)], ids=[c[0] for c in g.CASES])
def test_fixture_matches_reference(ref, fixture, i, name, metric, arg):
    from oracle import ref_pairwise

    if not ref_pairwise.available():
        pytest.skip("oracle/_ref/libfaiss_ref_pairwise.so not built")
    for kind in ("int", "float"):
        key = "%s_%s" % (name, kind)
        live = ref_pairwise.pairwise(fixture[key + "_xq"], fixture[key + "_xb"], metric, arg)
        if kind == "int" and name in EXACT_INT:
            assert np.array_equal(live, fixture[key + "_D"]), key
        else:
            _close(live, fixture[key + "_D"], key)

