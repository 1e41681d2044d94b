"""The numpy restatement of ResidualQuantizer's beam search (oracle/oracle_rq_np.py) against the reference CPU library,
byte for byte: the results minted into tests/golden/rq.npz, and the live shim (oracle/ref_rq.py) where it is built.
The GPU tests compare the device encoder with this restatement."""
import numpy as np
import pytest

from oracle import oracle_rq_np as ro
from tests.golden import make_golden_rq as g


@pytest.fixture(scope="module")
def golden():
    return g.load()


def _ref():
    from oracle import ref_rq

    return ref_rq if ref_rq.available() else None


@pytest.mark.parametrize("case", g.CASES, ids=[c[0] for c in g.CASES])
def test_refine_beam_matches_reference(golden, case):
    name, d, nbits, beam, n, _ = case
    c = g.case(golden, name)
    codes, resid, dis = ro.refine_beam(c["cb"], nbits, c["x"][:, None], beam)
    assert np.array_equal(codes, c["codes0"])
    assert np.array_equal(resid, c["resid0"])
    assert np.array_equal(dis.view(np.uint32), c["dis0"].view(np.uint32))


@pytest.mark.parametrize("case", g.CASES, ids=[c[0] for c in g.CASES])
def test_refine_beam_lut_matches_reference(golden, case):
    name, d, nbits, beam, n, _ = case
    c = g.case(golden, name)
    codes, dis = ro.refine_beam_lut(c["cb"], nbits, c["x"], beam)
    assert np.array_equal(codes, c["codes1"])
    assert np.array_equal(dis.view(np.uint32), c["dis1"].view(np.uint32))


@pytest.mark.parametrize("case", g.CASES, ids=[c[0] for c in g.CASES])
@pytest.mark.parametrize("lut", [0, 1])
@pytest.mark.parametrize("st", list(g.SEARCH_TYPES))
def test_compute_codes_matches_reference(golden, case, lut, st):
    name, d, nbits, beam, n, _ = case
    c = g.case(golden, name)
    lo_, hi = g.NORM_RANGE
    assert np.array_equal(ro.compute_codes(c["cb"], nbits, c["x"], lut, beam, st, lo_, hi), c["packed%d_%d" % (lut, st)])
    got = ro.compute_codes(c["cb"], nbits, c["x"], lut, beam, st, lo_, hi, centroids=c["cent"])
    assert np.array_equal(got, c["packed%d_%d_cent" % (lut, st)])


def test_fixture_exercises_ties_and_clamping(golden):
    # the tie case decides most beams by the id order: count candidates tied with the last kept one
    c = g.case(golden, "ties_b5")
    assert (c["dis0"][:, :-1] == c["dis0"][:, 1:]).mean() > 0.3
    # the qint8 norms reach both clamps
    n8 = np.concatenate([golden[name + "/packed0_%d" % ro.ST_norm_qint8][:, -1] for name, *_ in g.CASES])
    assert (n8 == 0).any() and (n8 == 255).any() and ((n8 > 0) & (n8 < 255)).any()


def test_pack_codes_bit_layout():
    # LSB first, fields back to back: codes (5, 3) with nbits (3, 5) are bits 101 then 11000
    packed = ro.pack_codes(np.array([[5, 3]]), [3, 5])
    assert packed.tolist() == [[0b00011101]]
    packed = ro.pack_codes(np.array([[1]]), [4], ro.ST_norm_float, norms=np.array([1.0], np.float32))
    assert packed.tolist() == [[0x01, 0x00, 0x00, 0xF8, 0x03]]  # 1 | (1.0f = 0x3F800000) << 4


def test_encode_qint_edges():
    # (x - min) / (max - min) * 256, floored, clamped to [0, 255]; NaN and |x1| >= 2^31 convert to 0x80000000 -> 0
    q = ro._encode_qint(np.array([0.0, 10.0, 5.0, 9.99, 1e30, np.nan], np.float32), 0.0, 10.0, 256)
    assert q.tolist() == [0, 255, 128, 255, 0, 0]


def test_restatement_matches_live_reference():
    ref = _ref()
    if ref is None:
        pytest.skip("oracle/_ref/libfaiss_ref_rq.so not built")
    rs = np.random.RandomState(5)
    for d, nbits, beam in [(32, [6] * 4, 5), (40, [4, 8, 6, 8, 5, 8, 8, 3, 8, 8], 16), (20, [3, 12], 7), (12, [7, 2, 5], 3)]:
        cb, x, cent = g.int_data(rs, d, nbits, 40, False)
        q = ref.RQ(d, nbits, cb)
        _, norms, cross = q.tables()
        n2, cr2 = ro.tables(cb, nbits)
        assert np.array_equal(norms, n2) and np.array_equal(cross, np.concatenate([c.ravel() for c in cr2]))
        for got, want in zip(q.refine_beam(x[:, None], 1, beam), ro.refine_beam(cb, nbits, x[:, None], beam)):
            assert np.array_equal(got, want)
        # beam_in > 1 (the reference needs out_beam >= beam_in: its residual pool is sized by the out beams)
        xb = np.stack([x, x + 1, x - 2], 1)
        for got, want in zip(q.refine_beam(xb, 3, beam), ro.refine_beam(cb, nbits, xb, beam)):
            assert np.array_equal(got, want)
        for got, want in zip(q.refine_beam_lut(x, beam), ro.refine_beam_lut(cb, nbits, x, beam)):
            assert np.array_equal(got, want)
