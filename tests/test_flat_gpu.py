"""GPU parity tests for the Flat path (GpuIndexFlat{,L2,IP}), through the C ABI.

Model: the reference's CPU-vs-GPU differential tests (faiss/gpu/test/TestGpuIndexFlat.cpp:47-817,
compareLists in faiss/gpu/test/TestUtils.cpp:234-443), with tighter bars:
  * integer-valued inputs -> ids AND distances bit-exact vs the reference CPU result;
  * uniform floats -> distances within 1e-4 relative (north_star), ids up to fp32 near-ties;
  * the tensor-core path must return exactly what the exact SIMT path returns.
"""
import ctypes

import numpy as np
import pytest

from oracle import oracle_np as o

pytestmark = pytest.mark.gpu


def _ref_search(xb, xq, k, metric):
    """reference CPU IndexFlat when oracle/_ref travelled to this box, else the pinned oracle"""
    from oracle import ref

    if ref.available():
        idx = ref.IndexFlat(xb.shape[1], metric)
        idx.add(xb)
        return idx.search(xq, k)
    return o.knn_flat(xq, xb, k, metric)


@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize("N,d,nq,k", [(3000, 32, 24, 10), (5000, 128, 100, 100), (2000, 17, 9, 1), (2500, 20, 13, 257)])
def test_exact_kernel_vs_reference(res, N, d, nq, k, metric):
    import faiss_b200 as fb

    xb = o.float_rand(N * d, 1234).reshape(N, d)
    xq = o.float_rand(nq * d, 1235).reshape(nq, d)
    idx = fb.GpuIndexFlat(res, d, metric, use_tensor_cores=False)
    idx.add(xb)
    D, I = idx.search(xq, k)
    rD, rI = _ref_search(xb, xq, k, metric)
    # tolerance: 1e-4 relative on distances (north_star); ranks may swap only on fp32 near-ties
    o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)


def test_golden_flat_fixture(res, golden):
    import faiss_b200 as fb

    N, d, nq, k = [int(v) for v in golden["flat_shape"]]
    xb = o.float_rand(N * d, 1234).reshape(N, d)
    xq = o.float_rand(nq * d, 1235).reshape(nq, d)
    for metric, name in ((1, "l2"), (0, "ip")):
        idx = fb.GpuIndexFlat(res, d, metric)
        idx.add(xb)
        D, I = idx.search(xq, k)
        o.compare_lists(golden["flat_%s_D" % name], golden["flat_%s_I" % name], D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)


@pytest.mark.parametrize("k", [10, 100])
def test_golden_integer_regime_bit_exact(res, golden, k):
    """north_star: bit-exact indices for Flat integer top-k ordering (heap and reservoir handlers)"""
    import faiss_b200 as fb

    N, d, nq = [int(v) for v in golden["flatint_shape"]]
    xb = np.floor(o.float_rand(N * d, 11).reshape(N, d) * 16).astype(np.float32)
    xq = np.floor(o.float_rand(nq * d, 12).reshape(nq, d) * 16).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert np.array_equal(I, golden["flatint_l2_k%d_I" % k])
    assert np.array_equal(D, golden["flatint_l2_k%d_D" % k])


@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize("N,d,nq,k", [(70000, 128, 300, 100), (120000, 96, 130, 10), (50000, 64, 64, 1), (65000, 100, 40, 50), (40000, 128, 520, 512),
     # K-split kernel (128 < d <= 256: ring stages hold single K-blocks) and the large-k lists
     (70000, 192, 300, 100), (66000, 256, 530, 10), (50000, 130, 100, 33), (90000, 64, 300, 1024), (100000, 32, 70, 2048), (40000, 256, 64, 2048)])
def test_tensor_core_path_equals_exact_path(res, N, d, nq, k, metric):
    """wgmma scoring + certified re-rank must be indistinguishable from the exact kernel"""
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda")
    g.manual_seed(N + d + k)
    xb = torch.rand(N, d, device="cuda", generator=g)
    xq = torch.rand(nq, d, device="cuda", generator=g)
    idx = fb.GpuIndexFlat(res, d, metric)
    idx.add(xb)
    D, I = idx.search(xq, k)
    info = idx.lastSearchInfo()
    assert info["tensor_cores"] == 1
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 0
    assert torch.equal(I, Ie)
    assert torch.equal(D, De)
    # and both agree with float64 ground truth on a sample
    gt = o.knn_flat(xq[:8].cpu().numpy(), xb.cpu().numpy(), k, metric)
    o.compare_lists(gt[0], gt[1], D[:8].cpu().numpy(), I[:8].cpu().numpy(), eps=1e-4, pct_max_diff1=0.02, pct_max_diffN=0.005)


def test_tensor_core_integer_regime_vs_reference(res):
    """full chain on exact arithmetic with many ties: ids == reference CPU ids"""
    import faiss_b200 as fb

    rs = np.random.RandomState(4)
    N, d, nq, k = 60000, 64, 40, 100
    xb = np.floor(rs.rand(N, d) * 4).astype(np.float32)  # heavy ties
    xq = np.floor(rs.rand(nq, d) * 4).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    rD, rI = o.knn_flat(xq, xb, k, 1)
    assert np.array_equal(D, rD)
    assert np.array_equal(I, rI)


def test_tensor_core_adversarial_order_falls_back_correctly(res):
    """database sorted by distance to the queries and duplicate-heavy: whatever the certificate
    decides, the answer equals the exact kernel's"""
    import torch

    import faiss_b200 as fb

    N, d, nq, k = 50000, 64, 20, 30
    g = torch.Generator(device="cuda")
    g.manual_seed(9)
    base = torch.rand(1, d, device="cuda", generator=g)
    scale = torch.linspace(2.0, 0.0, N, device="cuda").unsqueeze(1)  # later rows are closer to `base`
    xb = base + scale * torch.rand(N, d, device="cuda", generator=g)
    xb[-2000:] = xb[-1]  # 2000 exact duplicates of the nearest row
    xq = base + 0.001 * torch.rand(nq, d, device="cuda", generator=g)
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    D, I = idx.search(xq, k)
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, k)
    assert torch.equal(I, Ie) and torch.equal(D, De)


def test_fallback_count_covers_every_query_batch(res):
    """lastSearchInfo()["fallback_queries"] counts the exact recomputes of the whole call, not of its last internal
    query batch (2048 queries at k = 1024): the certificate-failing queries come first, fillers fill later batches"""
    import faiss_b200 as fb

    rs = np.random.RandomState(5)
    d, k = 64, 1024
    # near-duplicate rows (16 points, 2500 copies each, one coordinate moved by 1): their queries fail the
    # certificate.  In the opposite orthant, rows and queries with spread-out distances: those queries pass it.
    base = np.floor(rs.rand(16, d) * 16).astype(np.float32)
    dup = np.repeat(base, 2500, axis=0)
    dup[np.arange(len(dup)), rs.randint(0, d, len(dup))] += 1.0
    far = -np.abs(rs.randn(40000, d) * 8).astype(np.float32)
    xb = np.vstack([dup, far])
    failing = base[rs.randint(0, 16, 64)]
    fillers = -np.abs(rs.randn(3000, d) * 8).astype(np.float32)
    xq = np.vstack([failing, fillers])
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)

    idx.search(fillers, k)
    assert idx.lastSearchInfo() == {"tensor_cores": 1, "fallback_queries": 0}
    idx.search(failing, k)
    alone = idx.lastSearchInfo()["fallback_queries"]
    assert alone > 0

    D, I = idx.search(xq, k)
    info = idx.lastSearchInfo()
    assert info["tensor_cores"] == 1 and info["fallback_queries"] >= alone
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, k)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)


def test_tcgen05_raw_scores(res):
    """unit test of the MMA path alone: fp16 operands, fp32 accumulation (wgmma, register accumulators)"""
    import torch

    import faiss_b200 as fb

    torch.manual_seed(0)
    for nq, N, dpad in [(128, 256, 64), (200, 1000, 128), (300, 5000, 128), (300, 5000, 192), (520, 9000, 256)]:
        Q = torch.randn(nq, dpad, device="cuda").half()
        Y = torch.randn(N, dpad, device="cuda").half()
        S = fb.flat_tc_scores_debug(res, Q, Y)
        ref = Q.double() @ Y.double().T
        err = (S[:, :N].double() - ref).abs().max().item()
        bound = dpad * 2.0 ** -22 * (Q.float().norm(dim=1).max() * Y.float().norm(dim=1).max()).item()
        assert err <= bound, (err, bound)


def test_edge_cases(res):
    import faiss_b200 as fb

    rs = np.random.RandomState(0)
    d = 24
    xb = rs.rand(100, d).astype(np.float32)
    idx = fb.GpuIndexFlatL2(res, d)
    # empty index: ids -1, distances FLT_MAX (faiss/gpu/impl/Distance.cu:152-164)
    D, I = idx.search(rs.rand(3, d).astype(np.float32), 5)
    assert (I == -1).all() and (D == np.finfo(np.float32).max).all()
    idx.add(xb)
    assert idx.ntotal == 100
    # empty query batch
    D, I = idx.search(np.zeros((0, d), dtype=np.float32), 5)
    assert D.shape == (0, 5)
    # k > ntotal: tail padded with -1 / FLT_MAX
    D, I = idx.search(xb[:4], 128)
    assert (I[:, 100:] == -1).all() and (I[:, :100] >= 0).all()
    assert (I[:, 0] == np.arange(4)).all() and (D[:, 0] == 0).all()
    # k limit (faiss/gpu/impl/IndexUtils.cu:21-34)
    with pytest.raises(fb.FaissError) as e:
        idx.search(xb[:2], 2049)
    assert e.value.code == -2 and "2048" in str(e.value)
    D, I = idx.search(xb[:2], 2048)
    assert I.shape == (2, 2048)
    # add_with_ids unsupported on Flat (faiss/gpu/GpuIndexFlat.cu:210)
    with pytest.raises(fb.FaissError):
        idx.add_with_ids(xb[:3], np.arange(3))
    # reconstruct / copyTo / residual
    assert np.array_equal(idx.reconstruct_n(10, 5), xb[10:15])
    assert np.array_equal(idx.reconstruct(7), xb[7])
    assert np.array_equal(idx.reconstruct_batch([5, 1, 99]), xb[[5, 1, 99]])
    assert np.array_equal(idx.copyTo(), xb)
    r = idx.compute_residual_n(xb[:3], np.array([3, 4, 5]))
    assert np.array_equal(r, xb[:3] - xb[3:6])
    idx.reset()
    assert idx.ntotal == 0
    idx.copyFrom(xb[:50])
    assert idx.ntotal == 50


def test_device_and_host_pointers_agree(res):
    import torch

    import faiss_b200 as fb

    rs = np.random.RandomState(2)
    xb = rs.rand(5000, 48).astype(np.float32)
    xq = rs.rand(33, 48).astype(np.float32)
    idx = fb.GpuIndexFlatIP(res, 48)
    idx.add(torch.from_numpy(xb).cuda())
    Dh, Ih = idx.search(xq, 7)
    Dd, Id = idx.search(torch.from_numpy(xq).cuda(), 7)
    assert np.array_equal(Ih, Id.cpu().numpy()) and np.array_equal(Dh, Dd.cpu().numpy())


def test_memory_info_and_oom(res):
    """getMemoryInfo shape {device: {allocType: (count, bytes)}} (StandardGpuResources.h:243) and the
    over-allocation test of faiss/gpu/test/TestGpuMemoryException.cpp:25-80"""
    import faiss_b200 as fb

    idx = fb.GpuIndexFlatL2(res, 16)
    idx.add(np.zeros((1000, 16), dtype=np.float32))
    info = res.getMemoryInfo()
    assert 0 in info and "FlatData" in info[0] and info[0]["FlatData"][1] >= 1000 * 16 * 4
    big = fb.GpuIndexIVFFlat(res, 64, 16)
    with pytest.raises(fb.FaissError) as e:
        big.reserveMemory(1 << 36)  # 64 Gi vectors x 256 B: one impossible cudaMalloc
    assert "failed to allocate" in str(e.value)
    # the failed allocation leaves both indexes usable
    big.setCoarseCentroids(np.random.RandomState(0).rand(16, 64).astype(np.float32))
    big.setIsTrained(True)
    big.add(np.random.RandomState(1).rand(100, 64).astype(np.float32))
    assert big.ntotal == 100
    D, I = idx.search(np.zeros((2, 16), dtype=np.float32), 3)
    assert I.shape == (2, 3)


@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize("N,d,nq", [(4096, 128, 3000), (70000, 96, 5000), (2048, 64, 17), (300000, 32, 700), (30000, 256, 2000), (5000, 160, 300)])
def test_streaming_argmin_equals_exact_path(res, N, d, nq, metric):
    """k = 1 takes the streaming tensor-core mode (self-tightening thresholds, fused select + re-rank): the k-means
    assignment path.  Must be indistinguishable from the exact kernel, ids and distances."""
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda")
    g.manual_seed(N + d)
    xb = torch.rand(N, d, device="cuda", generator=g)
    xq = torch.rand(nq, d, device="cuda", generator=g)
    idx = fb.GpuIndexFlat(res, d, metric)
    idx.add(xb)
    D, I = idx.search(xq, 1)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, 1)
    assert torch.equal(I, Ie) and torch.equal(D, De)


def test_streaming_argmin_with_masses_of_ties(res):
    """duplicated rows: every query has hundreds of exact ties for the minimum -- more than a candidate segment
    holds -- so the certificate fails over to the exact kernel; the answer is still the smallest id"""
    import torch

    import faiss_b200 as fb

    rs = np.random.RandomState(11)
    base = np.floor(rs.rand(64, 32) * 8).astype(np.float32)
    xb = np.tile(base, (1500, 1))  # 96000 rows, each distinct row 1500 times
    xq = base[rs.randint(0, 64, size=200)] + 0.0
    idx = fb.GpuIndexFlatL2(res, 32)
    idx.add(xb)
    D, I = idx.search(xq, 1)
    info = idx.lastSearchInfo()
    assert info["tensor_cores"] == 1
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, 1)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)
    assert (D == 0).all() and (I < 64).all()


@pytest.mark.parametrize("metric", [1, 0])
def test_bfknn_free_function(res, metric):
    """faiss.knn_gpu / bfKnn (faiss/gpu/GpuDistance.h:33-181; the reference's TestGpuDistance.cu compares it with a
    CPU IndexFlat the same way): host and device inputs, same tolerance as the index path."""
    import torch

    import faiss_b200 as fb

    N, d, nq, k = 4000, 40, 37, 20
    xb = o.float_rand(N * d, 77).reshape(N, d)
    xq = o.float_rand(nq * d, 78).reshape(nq, d)
    D, I = fb.bfKnn(res, xq, xb, k, metric)
    rD, rI = _ref_search(xb, xq, k, metric)
    o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)
    Dd, Id = fb.bfKnn(res, torch.from_numpy(xq).cuda(), torch.from_numpy(xb).cuda(), k, metric)
    assert np.array_equal(I, Id.cpu().numpy()) and np.array_equal(D, Dd.cpu().numpy())
    with pytest.raises(fb.FaissError):
        fb.bfKnn(res, xq, xb, 5000, metric)


@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize("N,d,nq,k,tc", [(3000, 32, 24, 10, False), (70000, 128, 300, 100, True), (50000, 64, 200, 1, True), (40000, 50, 33, 7, True)])
def test_float16_storage(res, N, d, nq, k, tc, metric):
    """GpuIndexFlatConfig::useFloat16 (faiss/gpu/GpuIndexFlat.h:26-35; the reference's TestGpuIndexFlat Float16 cases):
    vectors and queries are rounded to fp16, distances are exact between the rounded values -- i.e. a CPU IndexFlat over
    the rounded data.  Both paths (wgmma + certified re-rank, exact SIMT) must agree bit for bit."""
    import faiss_b200 as fb

    xb = o.float_rand(N * d, 91).reshape(N, d)
    xq = o.float_rand(nq * d, 92).reshape(nq, d)
    idx = fb.GpuIndexFlat(res, d, metric, use_float16=True)
    idx.add(xb[: N // 2])
    idx.add(xb[N // 2 :])
    D, I = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == int(tc)
    xb16 = xb.astype(np.float16).astype(np.float32)
    xq16 = xq.astype(np.float16).astype(np.float32)
    rD, rI = _ref_search(xb16, xq16, k, metric)
    o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, k)
    assert np.array_equal(I, Ie) and np.array_equal(D, De)
    # the stored payload is the rounded data
    assert np.array_equal(idx.reconstruct_n(5, 40), xb16[5:45])
    assert np.array_equal(idx.copyTo(), xb16)
    keys = np.array([3, N - 1, 17], dtype=np.int64)
    assert np.array_equal(idx.reconstruct_batch(keys), xb16[keys])
    r = idx.compute_residual_n(xq[:3], keys)
    assert np.array_equal(r, xq[:3] - xb16[keys])


def test_host_query_paging_pipeline():
    """searchFromCpuPaged_ (faiss/gpu/GpuIndex.cu:620-788): host queries above getMinPagingSize go through the pinned
    double buffer (stager thread + async-copy stream); the result must be the unpaged one, page boundaries included."""
    import faiss_b200 as fb

    res = fb.StandardGpuResources()
    res.setPinnedMemory(1 << 20)  # two 512 KiB halves -> 2048 queries of d = 64 per page
    rs = np.random.RandomState(5)
    xb = rs.rand(40000, 64).astype(np.float32)
    xq = rs.rand(2048 * 3 + 77, 64).astype(np.float32)  # 4 pages, ragged tail
    for make in (lambda: fb.GpuIndexFlatL2(res, 64), lambda: fb.GpuIndexIVFFlat(res, 64, 32, fb.METRIC_L2)):
        idx = make()
        if not idx.is_trained:
            idx.train(xb[:8000])
            idx.nprobe = 4
        idx.add(xb)
        assert idx.getMinPagingSize() == 256 << 20
        D0, I0 = idx.search(xq, 10)  # below the threshold: one block
        idx.setMinPagingSize(1 << 16)
        assert idx.getMinPagingSize() == 1 << 16
        D1, I1 = idx.search(xq, 10)
        assert np.array_equal(I0, I1) and np.array_equal(D0, D1)
        # k = 1 (streaming path) and a single-query tail page
        D2, I2 = idx.search(xq[: 2048 * 2 + 1], 1)
        idx.setMinPagingSize(256 << 20)
        D3, I3 = idx.search(xq[: 2048 * 2 + 1], 1)
        assert np.array_equal(I2, I3) and np.array_equal(D2, D3)
