"""CPU tests of the packed PQ code restatement (oracle/oracle_pq_np.py) against the 4/5/6-bit IVF-PQ fixture
(tests/golden/ivfpq_nbits.npz)."""
import numpy as np
import pytest

from oracle import oracle_np as o
from oracle import oracle_pq_np as po
from tests.golden import make_golden_ivfpq_nbits as g


@pytest.fixture(scope="module")
def cases():
    return g.load()


def test_pack_unpack_round_trips_fixture_lists(cases):
    for c in cases:
        for l in range(g.NLIST):
            codes = po.pq_unpack_codes(c["codes"][l], c["M"], c["nbits"])
            assert codes.shape == (c["ids"][l].size, c["M"]) and (codes < (1 << c["nbits"])).all()
            assert np.array_equal(po.pq_pack_codes(codes, c["nbits"]).reshape(-1), c["codes"][l]), (c["i"], l)
        # ProductQuantizer::compute_codes of the probe set: the numpy encoder, packed, gives the same bytes
        assert np.array_equal(po.pq_pack_codes(o.pq_encode(c["xp"], c["pq"]), c["nbits"]), c["probe_codes"]), c["i"]


def test_numpy_search_reproduces_fixture(cases):
    for c in cases:
        D, I = po.ivfpq_search(c["xq"], g.K, g.NPROBE, c["centroids"], c["pq"], c["codes"], c["ids"], c["metric"], nbits=c["nbits"])
        o.compare_lists(c["D"], c["I"], D, I, eps=1e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)
