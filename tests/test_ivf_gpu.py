"""GPU parity tests for IVF-Flat / IVF-PQ, k-means and IndexShards, through the C ABI.

Model: faiss/gpu/test/TestGpuIndexIVFPQ.cpp:183-897, TestGpuIndexIVFFlat.cpp, test_gpu_index.py:124-196
(search == search_preassigned bit-exact), test_gpu_basics.py:117-133 (k-means objective),
test_multi_gpu.py:23-43 (sharded flat == unsharded)."""
import numpy as np
import pytest

from oracle import oracle_np as o

pytestmark = pytest.mark.gpu


def _lists_from_golden(golden, name, M):
    lens = golden["ivfpq_%s_lens" % name]
    codes_all, ids_all = golden["ivfpq_%s_codes" % name], golden["ivfpq_%s_ids" % name]
    codes, ids = [], []
    c0 = i0 = 0
    for n in lens:
        codes.append(codes_all[c0 : c0 + n * M])
        ids.append(ids_all[i0 : i0 + n])
        c0 += n * M
        i0 += n
    return codes, ids


@pytest.mark.parametrize("metric,name", [(1, "l2"), (0, "ip")])
def test_ivfpq_copyfrom_golden_search(res, golden, metric, name):
    """clone the reference-trained CPU index (centroids, PQ, ArrayInvertedLists bytes) and search:
    TestGpuIndexIVFPQ.cpp CopyFrom + Query, tolerance eps=1e-4 rel (reference test uses 0.035)"""
    import faiss_b200 as fb

    N, d, nlist, M, nq, k, nprobe = [int(v) for v in golden["ivfpq_shape"]]
    xq = o.float_rand(nq * d, 22).reshape(nq, d)
    codes, ids = _lists_from_golden(golden, name, M)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, metric)
    idx.setCoarseCentroids(golden["ivfpq_%s_centroids" % name])
    idx.setPQCentroids(golden["ivfpq_%s_pq" % name])
    for l in range(nlist):
        idx.setList(l, codes[l], ids[l])
    idx.setIsTrained(True)
    assert idx.ntotal == N
    idx.nprobe = nprobe
    D, I = idx.search(xq, k)
    o.compare_lists(golden["ivfpq_%s_D" % name], golden["ivfpq_%s_I" % name], D, I, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)
    # copyTo: byte-exact inverted lists (testIVFEquality, faiss/gpu/test/TestUtils.h:95-127)
    for l in range(nlist):
        assert np.array_equal(idx.getListVectorData(l), codes[l])
        assert np.array_equal(idx.getListIndices(l), ids[l])


def test_ivfpq_add_reproduces_reference_lists(res, golden):
    """device-side assign -> residual -> PQ encode -> append gives the reference's lists"""
    import faiss_b200 as fb

    N, d, nlist, M, nq, k, nprobe = [int(v) for v in golden["ivfpq_shape"]]
    xb = o.float_rand(N * d, 21).reshape(N, d)
    codes, ids = _lists_from_golden(golden, "l2", M)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, 1)
    idx.setCoarseCentroids(golden["ivfpq_l2_centroids"])
    idx.setPQCentroids(golden["ivfpq_l2_pq"])
    idx.setIsTrained(True)
    idx.add(xb[:2500])
    idx.add(xb[2500:])  # two batches: append order must stay insertion order
    assert idx.ntotal == N
    bad = 0
    for l in range(nlist):
        gi = idx.getListIndices(l)
        gc = idx.getListVectorData(l).reshape(-1, M)
        if gi.size == ids[l].size and np.array_equal(gi, ids[l]):
            bad += int((gc != codes[l].reshape(-1, M)).any(axis=1).sum())
        else:  # an assignment flipped on an fp near-tie
            bad += len(set(gi.tolist()) ^ set(ids[l].tolist()))
    assert bad <= N * 0.002


@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize("d", [40, 128, 256])
def test_ivfflat_vs_oracle_and_preassigned(res, metric, d):
    import faiss_b200 as fb

    rs = np.random.RandomState(3)
    N, nlist, nq, k = 20000, 50, 60, 20
    xb = rs.rand(N, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    idx = fb.GpuIndexIVFFlat(res, d, nlist, metric)
    assert not idx.is_trained
    with pytest.raises(fb.FaissError):
        idx.add(xb[:10])  # "Index not trained"
    idx.train(xb)
    ids = (np.arange(N, dtype=np.int64) * 7 + 3)
    idx.add_with_ids(xb, ids)
    idx.nprobe = 9
    D, I = idx.search(xq, k)
    cent = idx.getCoarseCentroids()
    lv = [idx.getListVectorData(l).view(np.float32) for l in range(nlist)]
    li = [idx.getListIndices(l) for l in range(nlist)]
    assert sum(x.size for x in li) == N
    rD, rI = o.ivfflat_search(xq, k, 9, cent, lv, li, metric)
    o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.005)
    # search == search_preassigned, bit-exact (faiss/gpu/test/test_gpu_index.py:190-194)
    cD, cI = o.knn_flat(xq, cent, 9, metric)
    D2, I2 = idx.search_preassigned(xq, k, cI, cD)
    assert np.array_equal(I, I2) and np.array_equal(D, D2)
    # nprobe limit
    idx.nprobe = 4096
    with pytest.raises(fb.FaissError):
        idx.search(xq, k)


@pytest.mark.parametrize("M", [4, 16, 32])
def test_ivfpq_train_add_search_vs_oracle(res, M):
    import faiss_b200 as fb

    rs = np.random.RandomState(M)
    N, d, nlist, nq, k = 30000, 64, 40, 50, 100
    xb = rs.rand(N, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, 1)
    idx.setClustering(niter=5)
    idx.setPQClustering(niter=6)
    idx.train(xb)
    idx.add(xb)
    idx.nprobe = 6
    D, I = idx.search(xq, k)
    lc = [idx.getListVectorData(l) for l in range(nlist)]
    li = [idx.getListIndices(l) for l in range(nlist)]
    rD, rI = o.ivfpq_search(xq, k, 6, idx.getCoarseCentroids(), idx.getPQCentroids(), lc, li, 1)
    o.compare_lists(rD, rI, D, I, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)
    # recall sanity vs exact ground truth (tests/test_ivfpq_indexing.cpp:17-97 style)
    gt = o.knn_flat(xq, xb, 1, 1)[1]
    assert o.recall_at(I, gt, 100) > (0.15 if M == 4 else 0.3)
    # reserve / reclaim keep contents
    before = [idx.getListIndices(l).copy() for l in range(0, nlist, 7)]
    idx.reserveMemory(2 * N)
    idx.reclaimMemory()
    after = [idx.getListIndices(l) for l in range(0, nlist, 7)]
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    D3, I3 = idx.search(xq, k)
    assert np.array_equal(I, I3)
    # precomputed term-2 tables (GpuIndexIVFPQConfig::usePrecomputedTables, IndexIVFPQ::precompute_table)
    # and the direct per-list LUT are two evaluations of the same distance: both must meet the oracle bar
    for enable in (False, True):
        idx.setPrecomputedCodes(enable)
        Dp, Ip = idx.search(xq, k)
        o.compare_lists(rD, rI, Dp, Ip, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)


@pytest.mark.parametrize("kind", ["flat40", "flat128", "pq16", "pq32"])
def test_ivf_scan_batch_size_invariance(res, kind):
    """The scan kernels give a CTA one query x a chunk of its probes; the chunk size depends on the
    batch size (1 probe per CTA for small batches, all probes for large ones).  The results must not:
    a 3000-query batch (one CTA per query), 400-query batches (3 probes per CTA) and 50-query batches
    (1 probe per CTA) are compared bit for bit."""
    import faiss_b200 as fb

    rs = np.random.RandomState(11)
    N, nlist, nq, k, nprobe = 40000, 64, 3000, 50, 9
    d = {"flat40": 40, "flat128": 128, "pq16": 64, "pq32": 64}[kind]
    xb = rs.rand(N, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    if kind.startswith("flat"):
        idx = fb.GpuIndexIVFFlat(res, d, nlist, 1)
    else:
        idx = fb.GpuIndexIVFPQ(res, d, nlist, int(kind[2:]), 8, 1)
        idx.setClustering(niter=4)
        idx.setPQClustering(niter=4)
    idx.train(xb[:20000])
    idx.add(xb)
    idx.nprobe = nprobe
    D, I = idx.search(xq, k)
    for bs in (400, 50):
        for q0 in (0, 1200, nq - bs):
            Db, Ib = idx.search(xq[q0 : q0 + bs], k)
            assert np.array_equal(Db, D[q0 : q0 + bs])
            # ids may only differ inside runs of exactly tied distances
            diff = Ib != I[q0 : q0 + bs]
            if diff.any():
                Dq = D[q0 : q0 + bs]
                tied = np.zeros_like(diff)
                tied[:, 1:] |= Dq[:, 1:] == Dq[:, :-1]
                tied[:, :-1] |= Dq[:, :-1] == Dq[:, 1:]
                assert not (diff & ~tied).any()


def test_ivfpq_constraints(res):
    import faiss_b200 as fb

    with pytest.raises(fb.FaissError):
        fb.GpuIndexIVFPQ(res, 64, 16, 8, 4)  # nbits != 8 (faiss/gpu/GpuIndexIVFPQ.cu:124-131)
    with pytest.raises(fb.FaissError):
        fb.GpuIndexIVFPQ(res, 30, 16, 8, 8)  # d % M != 0


def test_kmeans_matches_reference(res, golden):
    """same seeds -> same sampling and init as faiss::Clustering; objective and centroids agree
    (test_gpu_basics.py:117-133 uses np.allclose on the objective)"""
    import faiss_b200 as fb

    x = o.float_rand(5000 * 8, 31).reshape(5000, 8)
    cent, obj = fb.kmeans(res, x, 20, niter=8, seed=123)
    assert np.allclose(obj, golden["kmeans_obj"], rtol=1e-4)
    assert np.allclose(cent, golden["kmeans_centroids"], rtol=1e-3, atol=1e-4)
    cent, obj = fb.kmeans(res, x, 4, niter=5, seed=99, max_points_per_centroid=256)  # subsampled run
    assert np.allclose(obj, golden["kmeans_sub_obj"], rtol=1e-4)
    assert np.allclose(cent, golden["kmeans_sub_centroids"], rtol=1e-3, atol=1e-4)


def test_kmeans_large_codebook_path(res):
    """k*d > shared memory -> global RED path; compare with the oracle"""
    import faiss_b200 as fb

    rs = np.random.RandomState(5)
    x = rs.rand(30000, 64).astype(np.float32)
    cent, obj = fb.kmeans(res, x, 512, niter=4, seed=7)
    co, oo = o.kmeans(x, 512, niter=4, seed=7)
    assert np.allclose(obj, oo, rtol=1e-4)
    assert np.allclose(cent, co, rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("threaded", [False, True])
def test_index_shards_flat_equals_unsharded(res, threaded):
    """faiss/gpu/test/test_multi_gpu.py:23-43: sharded flat == reference ids (np.all(I == I_ref))"""
    import faiss_b200 as fb

    rs = np.random.RandomState(1)
    d = 32
    xb = rs.rand(1000, d).astype(np.float32)
    xq = rs.rand(50, d).astype(np.float32)
    sh = fb.IndexShards(d, threaded=threaded, successive_ids=True)
    subs = [fb.GpuIndexFlatL2(res, d) for _ in range(3)]
    for s in subs:
        sh.add_shard(s)
    sh.add(xb)
    assert sh.ntotal == 1000 and [s.ntotal for s in subs] == [333, 333, 334]
    D, I = sh.search(xq, 10)
    rD, rI = o.knn_flat(xq, xb, 10, 1)
    assert np.array_equal(I, rI)
    one = fb.GpuIndexFlatL2(res, d)
    one.add(xb)
    D1, I1 = one.search(xq, 10)
    assert np.array_equal(I, I1) and np.array_equal(D, D1)
    with pytest.raises(fb.FaissError):
        sh.add_with_ids(xb[:3], np.arange(3))  # successive_ids + explicit ids (IndexShards.cpp:143-150)


def test_device_merge_kernel_vs_reference_merge(res, golden):
    import torch

    import faiss_b200 as fb

    allD = torch.from_numpy(golden["merge_allD"]).cuda().permute(1, 0, 2).contiguous()
    allI = torch.from_numpy(golden["merge_allI"]).cuda().permute(1, 0, 2).contiguous()
    D, I = fb.topk_merge(res, allD, allI, 5, 1)
    assert np.array_equal(I.cpu().numpy(), golden["merge_I"])
    assert np.array_equal(D.cpu().numpy(), golden["merge_D"])


@pytest.mark.parametrize("shard_type", [1])
def test_cloner_ivfpq_shards_equal_unsharded(res, shard_type):
    """index_cpu_to_gpu_multiple(shard=True) semantics on the payload: the same coarse quantiser and PQ
    in every sub-index, lists split by shard_type, IndexShards with explicit ids == the unsharded index
    (faiss/gpu/test/test_multi_gpu.py:60-119 compares sharded IVF against the CPU index the same way).
    Distances agree to the last ulp or two, not bit for bit: the rotated code layout sums a vector's M table
    entries in a cyclic order that starts at (slot in the list) mod 32, and re-sharding moves the slots
    (observed 2.3172128 vs 2.3172126).  The splitting rules for shard types 2 and 4 are covered on the CPU
    (tests/test_abi.py::test_cloner_shard_ivf_lists_rules)."""
    import faiss_b200 as fb
    from faiss_b200 import cloner

    rs = np.random.RandomState(21)
    N, d, nlist, M, nq, k = 20000, 32, 24, 16, 40, 30
    xb = rs.rand(N, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, 1)
    idx.setClustering(niter=4)
    idx.setPQClustering(niter=4)
    idx.train(xb)
    idx.add(xb)
    idx.nprobe = 5
    D, I = idx.search(xq, k)
    payload = {"d": d, "nlist": nlist, "metric": 1, "centroids": idx.getCoarseCentroids(), "pq": idx.getPQCentroids(),
               "codes": [idx.getListVectorData(l) for l in range(nlist)], "ids": [idx.getListIndices(l) for l in range(nlist)]}
    shards = cloner.gpu_ivf_shards_from_payload([res, res, res], payload, shard_type=shard_type, threaded=False)
    assert shards.ntotal == N
    for i in range(shards.count()):
        shards.at(i).nprobe = 5
    Ds, Is = shards.search(xq, k)
    assert np.allclose(Ds, D, rtol=1e-5, atol=0)
    o.compare_lists(D, I, Ds, Is, eps=1e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)


def test_pq_train_matches_reference_fixture(res, golden):
    """a16: GPU ProductQuantizer training (M independent k-means, same seeds and sampling) reproduces the
    centroids of faiss::ProductQuantizer::train (fixture minted from oracle/_ref, faiss/impl/ProductQuantizer.cpp:130-195)"""
    import faiss_b200 as fb

    n, d, M, niter, seed = [int(v) for v in golden["pqtrain_shape"]]
    x = o.float_rand(n * d, 41).reshape(n, d)
    c = fb.pq_train(res, x, M, niter=niter, seed=seed)
    g = golden["pqtrain_centroids"]
    assert c.shape == g.shape
    # same Lloyd trajectory: centroids agree to fp32 summation order
    assert np.allclose(c, g, rtol=1e-3, atol=1e-4)


def test_spherical_ip_kmeans_matches_reference_fixture(res, golden):
    """GpuIndexIVF trains METRIC_INNER_PRODUCT coarse quantisers with spherical k-means
    (faiss/gpu/GpuIndexIVF.cu:72-76): centroids renormalised after the init and after every iteration"""
    import faiss_b200 as fb

    x = o.float_rand(3000 * 8, 51).reshape(3000, 8) - np.float32(0.5)
    cent, obj = fb.kmeans_ex(res, x, 12, niter=6, seed=77, metric=fb.METRIC_INNER_PRODUCT, spherical=True)
    assert np.allclose(np.linalg.norm(cent, axis=1), 1.0, atol=1e-5)
    assert np.allclose(obj, golden["kmeans_sph_obj"], rtol=1e-4)
    assert np.allclose(cent, golden["kmeans_sph_centroids"], rtol=1e-3, atol=1e-4)
    # and the IVF index itself: IP coarse centroids come out unit-norm
    rs = np.random.RandomState(3)
    xb = (rs.rand(6000, 16).astype(np.float32) - 0.5) * rs.rand(6000, 1).astype(np.float32) * 10
    ivf = fb.GpuIndexIVFFlat(res, 16, 24, fb.METRIC_INNER_PRODUCT)
    ivf.train(xb)
    c = ivf.getCoarseCentroids()
    assert np.allclose(np.linalg.norm(c, axis=1), 1.0, atol=1e-4)


def test_ivfflat_golden_search(res, golden):
    """a7 pinned on the reference's own IndexIVFFlat fixture: same centroids, device-side add, search"""
    import faiss_b200 as fb

    N, d, nlist, M, nq, k, nprobe = [int(v) for v in golden["ivfpq_shape"]]
    xb = o.float_rand(N * d, 21).reshape(N, d)
    xq = o.float_rand(nq * d, 22).reshape(nq, d)
    idx = fb.GpuIndexIVFFlat(res, d, nlist, fb.METRIC_L2)
    idx.setCoarseCentroids(golden["ivfflat_centroids"])
    idx.setIsTrained(True)
    idx.add(xb)
    idx.nprobe = nprobe
    D, I = idx.search(xq, k)
    o.compare_lists(golden["ivfflat_D"], golden["ivfflat_I"], D, I, eps=1e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)
    # list membership equals the reference's up to assignment near-ties
    lens, ids_all = golden["ivfflat_lens"], golden["ivfflat_ids"]
    i0 = bad = 0
    for l, n in enumerate(lens):
        bad += len(set(idx.getListIndices(l).tolist()) ^ set(ids_all[i0 : i0 + n].tolist()))
        i0 += n
    assert bad <= N * 0.004


def test_bulk_clone_single_relayout(res, golden):
    """cloner: setListSizes reserves every list once; the clone equals the per-list path byte for byte"""
    import faiss_b200 as fb
    from faiss_b200 import cloner

    N, d, nlist, M, nq, k, nprobe = [int(v) for v in golden["ivfpq_shape"]]
    codes, ids = _lists_from_golden(golden, "l2", M)
    payload = {"d": d, "nlist": nlist, "metric": 1, "centroids": golden["ivfpq_l2_centroids"], "pq": golden["ivfpq_l2_pq"],
               "codes": codes, "ids": ids}
    idx = cloner.gpu_ivf_from_payload(res, payload)
    assert idx.ntotal == N
    for l in range(nlist):
        assert np.array_equal(idx.getListVectorData(l), codes[l])
        assert np.array_equal(idx.getListIndices(l), ids[l])
    xq = o.float_rand(nq * d, 22).reshape(nq, d)
    idx.nprobe = nprobe
    D, I = idx.search(xq, k)
    o.compare_lists(golden["ivfpq_l2_D"], golden["ivfpq_l2_I"], D, I, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)


def test_search_parameters_ivf_and_shared_quantizer(res):
    """per-call SearchParametersIVF (faiss/gpu/GpuIndexIVF.cu:383-406) and the constructors that share a coarse
    quantiser (GpuIndexIVFFlat.h:48-59, GpuIndexIVFPQ.h:69-82)"""
    import faiss_b200 as fb

    rs = np.random.RandomState(9)
    d, nlist = 32, 32
    xb = rs.rand(9000, d).astype(np.float32)
    xq = rs.rand(50, d).astype(np.float32)
    a = fb.GpuIndexIVFFlat(res, d, nlist)
    a.setClustering(niter=5)
    a.train(xb)
    a.add(xb)
    a.nprobe = 1
    D1, I1 = a.search(xq, 10)
    D8, I8 = a.search(xq, 10, params=fb.SearchParametersIVF(nprobe=8))
    a.nprobe = 8
    Dref, Iref = a.search(xq, 10)
    assert np.array_equal(I8, Iref) and np.array_equal(D8, Dref)
    a.nprobe = 1
    D1b, I1b = a.search(xq, 10)
    assert np.array_equal(I1, I1b)  # the per-call override did not stick
    with pytest.raises(fb.FaissError):
        a.search(xq, 10, params=fb.SearchParametersIVF(nprobe=4, max_codes=100))
    # shared quantiser: a second IVF index over the SAME GpuIndexFlat is trained at birth and assigns identically
    cq = fb.GpuIndexFlatL2(res, d)
    cq.add(a.getCoarseCentroids())
    b = fb.GpuIndexIVFFlat(res, d, nlist, quantizer=cq)
    assert b.is_trained
    b.add(xb)
    b.nprobe = 8
    Db, Ib = b.search(xq, 10)
    assert np.array_equal(Ib, Iref) and np.array_equal(Db, Dref)
    c = fb.GpuIndexIVFPQ(res, d, nlist, 8, 8, quantizer=cq)
    assert not c.is_trained  # the PQ still needs training
    c.setPQClustering(niter=4)
    c.train(xb)
    assert c.is_trained and np.array_equal(c.getCoarseCentroids(), a.getCoarseCentroids())
    c.add(xb)
    c.nprobe = 8
    Dc, Ic = c.search(xq, 10)
    assert (Ic >= 0).all()


def test_interrupt_callback(res):
    """faiss::InterruptCallback polled between pages / iterations: the call fails with 'computation interrupted'"""
    import faiss_b200 as fb

    rs = np.random.RandomState(2)
    xb = rs.rand(5000, 16).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, 16)
    idx.add(xb)
    calls = []
    fb.set_interrupt_callback(lambda: calls.append(1) or True)
    try:
        with pytest.raises(fb.FaissError, match="interrupted"):
            idx.search(xb[:10], 5)
        with pytest.raises(fb.FaissError, match="interrupted"):
            fb.kmeans(res, xb, 8, niter=3)
    finally:
        fb.set_interrupt_callback(None)
    assert calls
    D, I = idx.search(xb[:10], 5)
    assert (I[:, 0] == np.arange(10)).all()


def test_index_shards_ivf_common_quantizer(res, golden):
    """faiss::IndexShardsIVF / common_ivf_quantizer (faiss/IndexShardsIVF.cpp:163-251): the shards share ONE coarse
    quantiser, which is searched once; the merged result equals the unsharded index"""
    import faiss_b200 as fb
    from faiss_b200 import cloner

    N, d, nlist, M, nq, k, nprobe = [int(v) for v in golden["ivfpq_shape"]]
    codes, ids = _lists_from_golden(golden, "l2", M)
    xq = o.float_rand(nq * d, 22).reshape(nq, d)
    cq = fb.GpuIndexFlatL2(res, d)
    cq.add(golden["ivfpq_l2_centroids"])
    parts = cloner.shard_ivf_lists(codes, ids, M, 3, cloner.SHARD_BY_ID_MOD)
    shards = fb.IndexShardsIVF(cq, nlist, threaded=True, successive_ids=False)
    for ci, ii in parts:
        sub = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, fb.METRIC_L2, quantizer=cq)
        sub.setPQCentroids(golden["ivfpq_l2_pq"])
        sub.setListSizes(np.array([len(a) for a in ii], dtype=np.int64))
        for l in range(nlist):
            if len(ii[l]):
                sub.setList(l, ci[l], ii[l])
        sub.setIsTrained(True)
        sub.nprobe = nprobe
        shards.add_shard(sub)
    assert shards.ntotal == N
    D, I = shards.search(xq, k)
    o.compare_lists(golden["ivfpq_l2_D"], golden["ivfpq_l2_I"], D, I, eps=2e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)


@pytest.mark.parametrize("M", [32, 16])
def test_ivfpq_k2048(res, M):
    """k = 2048 (the documented GPU limit, faiss/gpu/utils/DeviceDefs.cuh:61-68) through the interleaved scan: the
    CTA-wide list holds it"""
    import faiss_b200 as fb

    rs = np.random.RandomState(M)
    N, d, nlist, k, nprobe = 60000, 64, 16, 2048, 8
    xb = rs.rand(N, d).astype(np.float32)
    xq = rs.rand(12, d).astype(np.float32)
    idx = fb.GpuIndexIVFPQ(res, d, nlist, M, 8)
    idx.setClustering(niter=4)
    idx.setPQClustering(niter=4)
    idx.train(xb[:20000])
    idx.add(xb)
    idx.nprobe = nprobe
    D, I = idx.search(xq, k)
    lc = [idx.getListVectorData(l) for l in range(nlist)]
    li = [idx.getListIndices(l) for l in range(nlist)]
    rD, rI = o.ivfpq_search(xq, k, nprobe, idx.getCoarseCentroids(), idx.getPQCentroids(), lc, li, o.METRIC_L2)
    o.compare_lists(rD, rI, D, I, eps=2e-4, pct_max_diff1=0.03, pct_max_diffN=0.015)
