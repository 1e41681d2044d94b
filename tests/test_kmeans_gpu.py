"""Sharded k-means runs the single-process Lloyd loop plus one all-reduce per iteration, so with one rank it must
return bit for bit what `kmeans` returns on the same rows.  This runs the communicator path, with its device
all-reduces, on a single GPU; `test_multigpu.py` covers several ranks where there are several GPUs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_sharded_kmeans_one_rank_equals_single_process():
    import torch  # noqa: F401  (maps PyTorch's NCCL, which the library then uses)

    import faiss_b200 as fb

    res = fb.StandardGpuResources()
    try:
        res.ncclInitAll([0])
    except fb.FaissError as e:
        if "NCCL unavailable" in str(e):
            pytest.skip("NCCL cannot be loaded: %s" % e)
        raise
    rs = np.random.RandomState(7)
    # 40 distinct integer points, each repeated 100 times, and k = 64 > 40: at most 40 clusters are non-empty,
    # so every iteration refills empty clusters with split_clusters
    pts = np.floor(rs.rand(40, 16) * 32).astype(np.float32)
    x = pts[rs.permutation(np.repeat(np.arange(40), 100))]
    k, niter, seed = 64, 8, 321
    cent, obj, st = fb.kmeans_sharded(res, x, k, niter=niter, seed=seed)
    c1, o1 = fb.kmeans(res, x, k, niter=niter, seed=seed, max_points_per_centroid=1 << 20)
    assert st["nsplit"] > 0
    assert np.array_equal(cent.view(np.uint32), c1.view(np.uint32))
    assert np.array_equal(obj.view(np.uint32), o1.view(np.uint32))
