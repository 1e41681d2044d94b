"""The numpy restatement of IndexIVF::reconstruct_n (oracle/oracle_recons_np.py) against the reference CPU library's
own results in tests/golden/reconstruct.npz, bit for bit: every scalar-quantiser type at d = 40 and 36 with and
without a residual, PQ at every code width and layout the GPU stores, IVF-Flat.  The GPU tests compare the device
decoder with this restatement."""
import numpy as np
import pytest

from oracle import oracle_recons_np as rn
from tests.golden import make_golden_reconstruct as g


@pytest.fixture(scope="module")
def golden():
    return g.load()


@pytest.mark.parametrize("name,kind,params", g.CASES, ids=[c[0] for c in g.CASES])
def test_reconstruct_n_matches_reference(golden, name, kind, params):
    d = params["d"]
    lc = [golden["%s/codes%d" % (name, l)] for l in range(g.NLIST)]
    li = [golden["%s/ids%d" % (name, l)] for l in range(g.NLIST)]
    kw = {}
    if kind == rn.PQ:
        kw = {"M": params["M"], "nbits": params["nbits"], "pq": golden[name + "/pq"]}
    elif kind == rn.SQ:
        kw = {"qtype": params["qtype"], "by_residual": params["by_residual"], "trained": golden[name + "/trained"]}
    out = np.full((g.N, d), np.nan, np.float32)
    rn.reconstruct_n(kind, lc, li, 0, g.N, d, out, golden[name + "/centroids"], **kw)
    want = golden[name + "/recons"]
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), name


def test_encode_listno():
    # IndexIVF::encode_listno: coarse_code_size() little-endian bytes
    assert rn.coarse_code_size(1) == 0 and rn.coarse_code_size(256) == 1 and rn.coarse_code_size(300) == 2
    assert list(rn.encode_listno(299, 300)) == [299 & 0xFF, 1]
    assert list(rn.encode_listno(5, 256)) == [5]


def test_search_and_return_codes_listno_matches_reference(golden):
    # the reference's search_and_return_codes(include_listno) at nlist = 300: every returned row is the 2-byte
    # encode_listno of the entry's list followed by its list bytes, and search_and_reconstruct returns its vector
    ids, assign, xb = golden["codes/ids"], golden["codes/assign"], golden["codes/xb"]
    where = {int(i): r for r, i in enumerate(ids)}
    I, C, R = golden["codes/I"], golden["codes/codes"], golden["codes/R"]
    assert rn.coarse_code_size(g.CODES_NLIST) == 2 and C.shape[2] == 2 + 4 * g.CODES_D
    assert (I >= 0).all()
    for q in range(I.shape[0]):
        for j in range(I.shape[1]):
            r = where[int(I[q, j])]
            want = np.concatenate([rn.encode_listno(int(assign[r]), g.CODES_NLIST), xb[r].view(np.uint8)])
            assert np.array_equal(C[q, j], want)
            assert np.array_equal(R[q, j].view(np.uint32), xb[r].view(np.uint32))
