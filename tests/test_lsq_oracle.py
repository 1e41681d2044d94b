"""The numpy restatement of LocalSearchQuantizer's ICM encoding and of its random draws (oracle/oracle_lsq_np.py)
against the reference CPU library, byte for byte: the results minted into tests/golden/lsq.npz, and the live shim
(oracle/ref_lsq.py) where it is built.  The GPU tests compare the device encoder with this restatement."""
import numpy as np
import pytest

from oracle import oracle_lsq_np as lo
from tests.golden import make_golden_lsq as g


@pytest.fixture(scope="module")
def golden():
    return g.load()


def _case(golden, name):
    return {k.split("/", 1)[1]: v for k, v in golden.items() if k.startswith(name + "/")}


@pytest.mark.parametrize("case", g.CASES, ids=[c[0] for c in g.CASES])
def test_draws_match_reference(golden, case):
    name, M, K, d, n, ils, nperts, icm, seed, _ = case
    c = _case(golden, name)
    gen = lo.MT19937(seed)
    p = lo.draws(gen, M, K, nperts, n, ils)
    assert np.array_equal(p, c["perts"])
    assert int(gen.words(1)[0]) == int(c["next"])


@pytest.mark.parametrize("case", g.CASES, ids=[c[0] for c in g.CASES])
def test_icm_encode_matches_reference(golden, case):
    name, M, K, d, n, ils, nperts, icm, seed, _ = case
    c = _case(golden, name)
    codes, nxt = lo.encode_seeded(c["cb"], c["codes0"], c["x"], ils, nperts, icm, seed)
    assert np.array_equal(codes, c["codes"])
    assert nxt == int(c["next"])


def test_forced_ties_are_frequent(golden):
    # the tie cases only pin the tie rule if their argmins really tie: count rows of the first step that tie
    c = _case(golden, "ties_k32")
    u = lo.unary_terms(c["cb"], c["x"])
    ties = (u[:, 0, :] == u[:, 0, :].min(1, keepdims=True)).sum(1)
    assert (ties > 1).mean() > 0.5


@pytest.mark.parametrize("case", g.CC_CASES, ids=[c[0] for c in g.CC_CASES])
def test_compute_codes_matches_reference(golden, case):
    name, M, K, d, n, ils, nperts, icm, seed = case
    c = _case(golden, name)
    assert np.array_equal(lo.compute_codes(c["cb"], c["x"], ils, nperts, icm, seed), c["codes"])


def test_argmin_tie_rule():
    # equal minima: the smallest index wins, inside a bucket, across buckets and among the leftovers
    obj = np.full((4, 40), 5, np.float32)
    obj[0, [3, 19, 35]] = 1  # bucket 3 twice, then a leftover
    obj[1, [17, 2]] = 1  # bucket 1 (position 17) and bucket 2
    obj[2, [36, 38]] = 0  # leftovers only
    obj[3, :] = 2  # all equal
    assert list(lo.argmin_buckets(obj)) == [3, 2, 36, 0]


def test_live_reference(golden):
    from oracle import ref_lsq

    if not ref_lsq.available():
        pytest.skip("oracle/_ref/libfaiss_ref_lsq.so not built")
    rs = np.random.RandomState(5)
    for M, K, d, n, ils, nperts, icm, distinct in ((4, 16, 20, 100, 4, 4, 3, 0), (3, 64, 10, 100, 3, 2, 2, 4), (5, 8, 7, 60, 2, 0, 2, 0)):
        cb, x = g.int_data(rs, M, K, d, n, distinct)
        codes0 = rs.randint(0, K, (n, M)).astype(np.int32)
        want, want_next = ref_lsq.LSQ(cb, nperts=nperts, icm_iters=icm).icm_encode(codes0, x, ils, 31)
        got, got_next = lo.encode_seeded(cb, codes0, x, ils, nperts, icm, 31)
        assert np.array_equal(got, want) and got_next == want_next
        p, p_next = ref_lsq.draws(M, K, nperts, n, ils, 31)
        gen = lo.MT19937(31)
        assert np.array_equal(lo.draws(gen, M, K, nperts, n, ils), p) and int(gen.words(1)[0]) == p_next
