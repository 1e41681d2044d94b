"""GpuIndexIVFScalarQuantizer on the GPU against the CPU reference: the fixture tests/golden/ivfsq.npz and,
where oracle/_ref was built, the live reference (oracle/ref_sq.py)."""
import numpy as np
import pytest

from oracle import oracle_np as o
from oracle import oracle_sq_np as so
from tests.golden import make_golden_ivfsq as g

pytestmark = pytest.mark.gpu

# relative distance tolerance: the folded decode (DESIGN.md, IVF-SQ scan) differs from the CPU's decode-then-
# subtract by a few fp32 rounding steps per component, far below this for the data used here
EPS = 1e-4


@pytest.fixture(scope="module")
def ref_sq():
    from oracle import ref_sq as r

    if not r.available():
        pytest.skip("oracle/_ref/libfaiss_ref_sq.so not built (needs /root/reference at build time)")
    return r


@pytest.fixture(scope="module")
def cases():
    return g.load()


def _payload(d, nlist, metric, qtype, by_residual, centroids, trained, codes, ids):
    return {"d": d, "nlist": nlist, "metric": metric, "centroids": centroids, "codes": codes, "ids": ids,
            "sq": {"qtype": qtype, "by_residual": by_residual, "trained": trained}}


def _clone(res, p):
    from faiss_b200 import cloner

    return cloner.gpu_ivf_from_payload(res, p)


def _ref_payload(idx, d, nlist, metric):
    lists = [idx.get_list(l) for l in range(nlist)]
    return _payload(d, nlist, metric, idx.qtype, idx.by_residual, idx.centroids(), idx.trained(),
                    [c for c, _ in lists], [a for _, a in lists])


def _data(rs, n, d, qtype):
    if qtype == so.QT_8bit_direct:
        return np.floor(rs.rand(n, d) * 256).astype(np.float32)
    return (rs.rand(n, d) * 4).astype(np.float32)


def test_clone_search_fixture(res, cases):
    for c in cases:
        p = _payload(c["d"], g.NLIST, c["metric"], c["qtype"], c["by_residual"], c["centroids"], c["trained"],
                     c["codes"], c["ids"])
        idx = _clone(res, p)
        assert idx.is_trained and idx.ntotal == g.NB and idx.code_size == so.code_size(c["qtype"], c["d"])
        assert np.array_equal(idx.getTrained(), c["trained"])
        for l in range(g.NLIST):
            assert np.array_equal(idx.getListVectorData(l), c["codes"][l])
            assert np.array_equal(idx.getListIndices(l), c["ids"][l])
        idx.nprobe = g.NPROBE
        D, I = idx.search(c["xq"], g.K)
        o.compare_lists(c["D"], c["I"], D, I, eps=EPS, pct_max_diff1=0.02, pct_max_diffN=0.01)


@pytest.mark.parametrize("qtype", range(7))
@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize("by_residual", [True, False])
def test_clone_search_live(res, ref_sq, qtype, metric, by_residual):
    # d = 36: the generic scan path.  (8bit_direct: the avx2 CPU scanner only switches to byte arithmetic at
    # d % 16 == 0, so d = 36 keeps its float decode on both sides.)
    d, nlist, k = 36, 16, 20
    rs = np.random.RandomState(100 + 4 * qtype + 2 * metric + by_residual)
    idx = ref_sq.IndexIVFScalarQuantizer(d, nlist, qtype, metric, by_residual)
    idx.set_cp(niter=5)
    idx.train(_data(rs, 4000, d, qtype))
    idx.add(_data(rs, 5000, d, qtype))
    idx.set_nprobe(5)
    xq = _data(rs, 50, d, qtype)
    rD, rI = idx.search(xq, k)
    p = _ref_payload(idx, d, nlist, metric)
    gidx = _clone(res, p)
    gidx.nprobe = 5
    D, I = gidx.search(xq, k)
    o.compare_lists(rD, rI, D, I, eps=EPS, pct_max_diff1=0.02, pct_max_diffN=0.01)
    for l in range(nlist):
        assert np.array_equal(gidx.getListVectorData(l), p["codes"][l])


@pytest.mark.parametrize("qtype", [so.QT_8bit, so.QT_8bit_uniform, so.QT_4bit, so.QT_6bit])
def test_train_bit_exact(res, ref_sq, qtype):
    """same coarse centroids on both sides, then train: the trained parameters are bit-exact; 120000 rows
    take the 100000-row subsample path (fvecs_maybe_subsample, seed 1234)"""
    import faiss_b200 as fb

    d, nlist = 16, 8
    rs = np.random.RandomState(qtype)
    for n in (3000, 120000):
        xt = (rs.randn(n, d) * 2).astype(np.float32)
        r = ref_sq.IndexIVFScalarQuantizer(d, nlist, qtype, 1, True)
        r.set_cp(niter=3)
        r.train(xt)
        gi = fb.GpuIndexIVFScalarQuantizer(res, d, nlist, qtype)
        gi.setCoarseCentroids(r.centroids())
        gi.train(xt)
        assert gi.is_trained
        assert np.array_equal(gi.getTrained().view(np.uint32), r.trained().view(np.uint32)), n


@pytest.mark.parametrize("qtype", range(7))
def test_add_reproduces_reference_lists(res, ref_sq, qtype):
    import faiss_b200 as fb

    d, nlist = 40, 16
    rs = np.random.RandomState(50 + qtype)
    r = ref_sq.IndexIVFScalarQuantizer(d, nlist, qtype, 1, True)
    r.set_cp(niter=4)
    r.train(_data(rs, 3000, d, qtype))
    xb = _data(rs, 4000, d, qtype)
    r.add(xb)
    gi = fb.GpuIndexIVFScalarQuantizer(res, d, nlist, qtype)
    gi.setCoarseCentroids(r.centroids())
    gi.setTrained(r.trained())
    gi.setIsTrained(True)
    gi.add(xb)
    assert gi.ntotal == xb.shape[0]
    cs = gi.code_size
    ref_code, ref_list, gpu_code, gpu_list = {}, {}, {}, {}
    for l in range(nlist):
        c, a = r.get_list(l)
        for j, i in enumerate(a):
            ref_code[int(i)], ref_list[int(i)] = c[j * cs : (j + 1) * cs], l
        gc, ga = gi.getListVectorData(l), gi.getListIndices(l)
        for j, i in enumerate(ga):
            gpu_code[int(i)], gpu_list[int(i)] = gc[j * cs : (j + 1) * cs], l
        # lists keep insertion order
        assert np.all(np.diff(ga) > 0)
    flips = [i for i in ref_list if ref_list[i] != gpu_list[i]]
    assert len(flips) <= 4, flips  # near-tie coarse assignments
    for i in ref_code:
        if i not in flips:
            assert np.array_equal(ref_code[i], gpu_code[i]), i


def _trained_index(res, qtype, d, metric, by_residual, nlist=32, n=6000, seed=0):
    import faiss_b200 as fb

    rs = np.random.RandomState(seed)
    xb = _data(rs, n, d, qtype)
    idx = fb.GpuIndexIVFScalarQuantizer(res, d, nlist, qtype, metric, by_residual)
    idx.setClustering(niter=5)
    idx.train(xb)
    idx.add(xb)
    return idx, xb, _data(rs, 64, d, qtype)


def _oracle_search(idx, xq, k, nprobe, metric):
    nl = idx.nlist
    return so.ivfsq_search(xq, k, nprobe, idx.getCoarseCentroids(), idx.qtype, idx.getTrained(),
                           [idx.getListVectorData(l) for l in range(nl)], [idx.getListIndices(l) for l in range(nl)],
                           metric, idx.by_residual)


@pytest.mark.parametrize("qtype,d", [(so.QT_8bit, 128), (so.QT_8bit_uniform, 256), (so.QT_fp16, 64),
                                     (so.QT_fp16, 256), (so.QT_4bit, 256), (so.QT_4bit_uniform, 512),
                                     (so.QT_8bit, 40), (so.QT_6bit, 36), (so.QT_6bit, 128), (so.QT_4bit, 39),
                                     (so.QT_fp16, 100)])
@pytest.mark.parametrize("metric", [1, 0])
def test_scan_paths_vs_oracle(res, qtype, d, metric):
    """fast-path shapes (rows of whole 128-byte chunks) and generic shapes against the numpy restatement"""
    idx, xb, xq = _trained_index(res, qtype, d, metric, True, seed=d + qtype)
    idx.nprobe = 6
    D, I = idx.search(xq, 50)
    rD, rI = _oracle_search(idx, xq, 50, 6, metric)
    o.compare_lists(rD, rI, D, I, eps=EPS, pct_max_diff1=0.02, pct_max_diffN=0.01)


@pytest.mark.parametrize("metric", [1, 0])
def test_preassigned_batches_and_inputs(res, metric):
    import torch

    import faiss_b200 as fb

    idx, xb, xq = _trained_index(res, so.QT_8bit, 64, metric, True)
    idx.nprobe = 8
    D, I = idx.search(xq, 20)
    flat = fb.GpuIndexFlat(res, 64, metric)
    flat.add(idx.getCoarseCentroids())
    cD, cI = flat.search(xq, 8)
    D2, I2 = idx.search_preassigned(xq, 20, cI, cD)
    assert np.array_equal(D, D2) and np.array_equal(I, I2)
    # user-supplied centroid distances: IP with a residual adds them to every distance
    D3, I3 = idx.search_preassigned(xq, 20, cI, cD + 1.0)
    if metric == 0:
        assert np.array_equal(I3, I) and np.allclose(D3, D + 1.0, rtol=1e-6)
    else:
        assert np.array_equal(D3, D) and np.array_equal(I3, I)
    # query-batch-size invariance
    Db = np.concatenate([idx.search(xq[i : i + 7], 20)[0] for i in range(0, xq.shape[0], 7)])
    Ib = np.concatenate([idx.search(xq[i : i + 7], 20)[1] for i in range(0, xq.shape[0], 7)])
    assert np.array_equal(D, Db) and np.array_equal(I, Ib)
    # torch CUDA inputs give the same results
    Dt, It = idx.search(torch.from_numpy(xq).cuda(), 20)
    assert np.array_equal(Dt.cpu().numpy(), D) and np.array_equal(It.cpu().numpy(), I)


def test_edges(res):
    import faiss_b200 as fb

    d, nlist = 32, 64
    idx, xb, xq = _trained_index(res, so.QT_8bit, d, 1, True, nlist=nlist, n=3000)
    # k = 2048 against the oracle
    idx.nprobe = 64
    D, I = idx.search(xq[:4], 2048)
    rD, rI = _oracle_search(idx, xq[:4], 2048, 64, 1)
    o.compare_lists(rD, rI, D, I, eps=EPS, pct_max_diff1=0.02, pct_max_diffN=0.01)
    # nprobe above the limit
    idx.nprobe = 4096
    with pytest.raises(fb.FaissError):
        idx.search(xq, 5)
    idx.nprobe = 4
    # a NaN query gives -1 ids
    q = xq[:3].copy()
    q[1, 5] = np.nan
    D, I = idx.search(q, 5)
    assert (I[1] == -1).all() and (I[0] >= 0).all()
    # an empty list: clone with list 0 emptied
    lists = [(idx.getListVectorData(l), idx.getListIndices(l)) for l in range(nlist)]
    codes = [c for c, _ in lists]
    ids = [a for _, a in lists]
    codes[0], ids[0] = codes[0][:0], ids[0][:0]
    p = _payload(d, nlist, 1, so.QT_8bit, True, idx.getCoarseCentroids(), idx.getTrained(), codes, ids)
    e = _clone(res, p)
    e.nprobe = 4
    assert e.getListLength(0) == 0
    D, I = e.search(xq, 10)
    rD, rI = so.ivfsq_search(xq, 10, 4, p["centroids"], so.QT_8bit, p["sq"]["trained"], codes, ids, 1, True)
    o.compare_lists(rD, rI, D, I, eps=EPS, pct_max_diff1=0.02, pct_max_diffN=0.01)


def test_shards_equal_unsharded(res):
    import faiss_b200 as fb
    from faiss_b200 import cloner

    d, nlist = 48, 16
    idx, xb, xq = _trained_index(res, so.QT_4bit, d, 1, True, nlist=nlist, n=5000)
    idx.nprobe = 6
    D, I = idx.search(xq, 20)
    p = _payload(d, nlist, 1, so.QT_4bit, True, idx.getCoarseCentroids(), idx.getTrained(),
                 [idx.getListVectorData(l) for l in range(nlist)], [idx.getListIndices(l) for l in range(nlist)])
    resources = [fb.StandardGpuResources() for _ in range(3)]
    sh = cloner.gpu_ivf_shards_from_payload(resources, p, shard_type=cloner.SHARD_BY_ID_MOD)
    assert sh.ntotal == idx.ntotal
    for i in range(3):
        sh.at(i).nprobe = 6
    Ds, Is = sh.search(xq, 20)
    assert np.array_equal(I, Is) and np.array_equal(D, Ds)


def test_errors(res):
    import faiss_b200 as fb

    with pytest.raises(fb.FaissError, match="Unsupported scalar QuantizerType"):
        fb.GpuIndexIVFScalarQuantizer(res, 32, 8, fb.QT_bf16)
    rs = np.random.RandomState(0)
    xb = rs.rand(1000, 32).astype(np.float32)
    idx = fb.GpuIndexIVFScalarQuantizer(res, 32, 8, fb.QT_8bit)
    with pytest.raises(fb.FaissError):
        idx.add(xb)  # not trained
    idx.setRangeStat(fb.RS_meanstd, 1.0)
    with pytest.raises(fb.FaissError):
        idx.train(xb)
    with pytest.raises(fb.FaissError):
        idx.setTrained(np.zeros(3, np.float32))  # wrong length
