"""GpuIndexIVFPQ with 4-, 5- and 6-bit codes (GpuIndexIVFPQConfig::interleavedLayout) against the reference
fixture (tests/golden/ivfpq_nbits.npz) and, where oracle/_ref was built, against the live reference.  The 4-bit
cases with M in {32, 64} run the interleaved nibble-pair scan, the others the packed vector-major scan."""
import numpy as np
import pytest

from oracle import oracle_np as o
from oracle import oracle_pq_np as po
from tests.golden import make_golden_ivfpq_nbits as g

pytestmark = pytest.mark.gpu

FAST = 0     # case 0: nbits 4, d 64, M 32, L2 (nibble-pair scan)
GENERIC = 5  # case 5: nbits 5, d 64, M 16, L2 (packed scan)


@pytest.fixture(scope="module")
def cases():
    return g.load()


def _payload(c):
    return {"d": c["d"], "nlist": g.NLIST, "metric": c["metric"], "centroids": c["centroids"], "pq": c["pq"],
            "codes": c["codes"], "ids": c["ids"]}


def _clone(res, c):
    from faiss_b200 import cloner

    idx = cloner.gpu_ivf_from_payload(res, _payload(c))
    idx.nprobe = g.NPROBE
    return idx


def _new(res, c, **kw):
    import faiss_b200 as fb

    return fb.GpuIndexIVFPQ(res, c["d"], g.NLIST, c["M"], c["nbits"], c["metric"], interleaved_layout=True, **kw)


def test_clone_search_and_lists(res, cases):
    for c in cases:
        idx = _clone(res, c)
        assert idx.is_trained and idx.ntotal == g.NB and idx._code_size() == c["code_size"]
        assert np.array_equal(idx.getPQCentroids(), c["pq"])
        for l in range(g.NLIST):
            assert np.array_equal(idx.getListVectorData(l), c["codes"][l]), (c["i"], l)
            assert np.array_equal(idx.getListIndices(l), c["ids"][l]), (c["i"], l)
        D, I = idx.search(c["xq"], g.K)
        o.compare_lists(c["D"], c["I"], D, I, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)


def test_add_reproduces_reference_lists(res, cases):
    for c in cases:
        idx = _new(res, c)
        idx.setCoarseCentroids(c["centroids"])
        idx.setPQCentroids(c["pq"])
        idx.setIsTrained(True)
        idx.add(c["xb"][:1000])
        idx.add(c["xb"][1000:])  # two batches: insertion order is kept
        assert idx.ntotal == g.NB
        cs, bad = c["code_size"], 0
        for l in range(g.NLIST):
            gi, gc = idx.getListIndices(l), idx.getListVectorData(l).reshape(-1, cs)
            if gi.size == c["ids"][l].size and np.array_equal(gi, c["ids"][l]):
                bad += int((gc != c["codes"][l].reshape(-1, cs)).any(axis=1).sum())
            else:  # an assignment flipped on an fp near-tie
                bad += len(set(gi.tolist()) ^ set(c["ids"][l].tolist()))
        assert bad <= g.NB * 0.002, (c["i"], bad)


def test_train_with_preset_coarse_matches_reference(res, cases):
    for c in cases:
        idx = _new(res, c)
        idx.setPQClustering(niter=g.NITER)
        idx.setCoarseCentroids(c["centroids"])
        idx.train(c["xb"])
        assert idx.is_trained
        pq = idx.getPQCentroids()
        assert pq.shape == c["pq"].shape
        assert np.allclose(pq, c["pq"], rtol=1e-3, atol=1e-4), c["i"]


def test_preassigned_params_and_precomputed_setting(res, cases):
    import faiss_b200 as fb

    for c in cases:
        idx = _clone(res, c)
        D, I = idx.search(c["xq"], g.K)
        flat = fb.GpuIndexFlat(res, c["d"], c["metric"])
        flat.add(c["centroids"])
        cD, cI = flat.search(c["xq"], g.NPROBE)
        D2, I2 = idx.search_preassigned(c["xq"], g.K, cI, cD)
        assert np.array_equal(D, D2) and np.array_equal(I, I2), c["i"]
        idx.nprobe = 1
        D3, I3 = idx.search(c["xq"], g.K, params=fb.SearchParametersIVF(nprobe=g.NPROBE))
        assert np.array_equal(D, D3) and np.array_equal(I, I3), c["i"]
        idx.nprobe = g.NPROBE
        # precomputed term-2 tables are not used below 8 bits: the setting does not change results
        idx.setPrecomputedCodes(True)
        D4, I4 = idx.search(c["xq"], g.K)
        assert np.array_equal(D, D4) and np.array_equal(I, I4), c["i"]


def _trained(res, c, n=40000, seed=11):
    rs = np.random.RandomState(seed)
    xb = rs.rand(n, c["d"]).astype(np.float32)
    idx = _new(res, c)
    idx.setClustering(niter=4)
    idx.setPQClustering(niter=4)
    idx.train(xb[:20000])
    idx.add(xb)
    return idx, rs


@pytest.mark.parametrize("case", [FAST, GENERIC])
def test_batch_size_invariance(res, cases, case):
    """as test_ivf_scan_batch_size_invariance: 3000-, 400- and 50-query batches agree bit for bit"""
    c = cases[case]
    idx, rs = _trained(res, c)
    xq = rs.rand(3000, c["d"]).astype(np.float32)
    idx.nprobe = 9
    D, I = idx.search(xq, 50)
    for bs in (400, 50):
        for q0 in (0, 1200, 3000 - bs):
            Db, Ib = idx.search(xq[q0 : q0 + bs], 50)
            assert np.array_equal(Db, D[q0 : q0 + bs])
            diff = Ib != I[q0 : q0 + bs]
            if diff.any():  # ids may only differ inside runs of exactly tied distances
                Dq = D[q0 : q0 + bs]
                tied = np.zeros_like(diff)
                tied[:, 1:] |= Dq[:, 1:] == Dq[:, :-1]
                tied[:, :-1] |= Dq[:, :-1] == Dq[:, 1:]
                assert not (diff & ~tied).any()


@pytest.mark.parametrize("case", [0, 1, 3, 4, 7])
def test_scan_vs_oracle_on_own_lists(res, cases, case):
    """k = 2048 (case 0) with every list probed, on the nibble-pair (0, 1) and packed (3, 4, 7) scans, against the
    numpy search over the index's own centroids and list bytes"""
    c = cases[case]
    idx, rs = _trained(res, c, n=12000, seed=case)
    xq = rs.rand(6, c["d"]).astype(np.float32)
    k = 2048 if case == 0 else 100
    nl = g.NLIST
    idx.nprobe = nl
    D, I = idx.search(xq, k)
    rD, rI = po.ivfpq_search(xq, k, nl, idx.getCoarseCentroids(), idx.getPQCentroids(),
                             [idx.getListVectorData(l) for l in range(nl)], [idx.getListIndices(l) for l in range(nl)],
                             c["metric"], nbits=c["nbits"])
    o.compare_lists(rD, rI, D, I, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)


def test_shards_equal_unsharded(res, cases):
    import torch

    import faiss_b200 as fb
    from faiss_b200 import cloner

    c = cases[FAST]
    idx = _clone(res, c)
    D, I = idx.search(c["xq"], g.K)
    devices = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    resources = [fb.StandardGpuResources() for _ in devices]
    sh = cloner.gpu_ivf_shards_from_payload(resources, _payload(c), shard_type=cloner.SHARD_BY_ID_MOD, devices=devices)
    assert sh.ntotal == idx.ntotal
    for i in range(len(devices)):
        sh.at(i).nprobe = g.NPROBE
    Ds, Is = sh.search(c["xq"], g.K)
    # the interleaved layout sums a vector's table entries in an order set by its position mod 32, which
    # re-sharding changes: distances agree to rounding (DESIGN §2), ids exactly
    assert np.array_equal(I, Is) and np.allclose(D, Ds, rtol=1e-6, atol=0)


def test_constraints(res):
    import faiss_b200 as fb

    with pytest.raises(fb.FaissError):
        fb.GpuIndexIVFPQ(res, 64, 16, 16, 4)  # 4 bits need interleavedLayout
    for nbits in (3, 7):
        with pytest.raises(fb.FaissError, match="Bits per code must be between 4, 5, 6 or 8"):
            fb.GpuIndexIVFPQ(res, 64, 16, 16, nbits, interleaved_layout=True)
    with pytest.raises(fb.FaissError):
        fb.GpuIndexIVFPQ(res, 60, 16, 16, 4, interleaved_layout=True)  # d % M != 0
    with pytest.raises(fb.FaissError, match="lookup table does not fit"):
        fb.GpuIndexIVFPQ(res, 1024, 16, 1024, 6, interleaved_layout=True)  # 4 * 1024 * 64 B > 160 KiB
    # nbits = 8 with the flag is the default index
    idx = fb.GpuIndexIVFPQ(res, 64, 16, 16, 8, interleaved_layout=True)
    assert idx._code_size() == 16


def test_live_reference_large(res, ref):
    """N = 200k, d = 128, M = 64, nbits = 4, nlist = 256 trained and filled on the GPU, cloned to the reference
    CPU index list by list (add_entries), both searched"""
    from oracle import ref_pq

    N, d, M, nbits, nlist, nq, k, nprobe = 200_000, 128, 64, 4, 256, 200, 50, 16
    rs = np.random.RandomState(7)
    xb = rs.rand(N, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    import faiss_b200 as fb

    gi = fb.GpuIndexIVFPQ(res, d, nlist, M, nbits, 1, interleaved_layout=True)
    gi.setClustering(niter=5)
    gi.setPQClustering(niter=5)
    gi.train(xb[:60000])
    gi.add(xb)
    gi.nprobe = nprobe
    D, I = gi.search(xq, k)
    r = ref_pq.IndexIVFPQ(d, nlist, M, nbits, 1)
    r.set_centroids(gi.getCoarseCentroids())
    r.set_pq_centroids(gi.getPQCentroids())
    for l in range(nlist):
        ids = gi.getListIndices(l)
        if ids.size:
            r.add_entries(l, ids, gi.getListVectorData(l))
    r.set_is_trained(True)
    assert r.ntotal == N
    r.set_nprobe(nprobe)
    rD, rI = r.search(xq, k)
    o.compare_lists(rD, rI, D, I, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)
