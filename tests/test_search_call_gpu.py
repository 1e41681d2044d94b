"""A search call's state (parameters, selector mask, the row of each query page) travels with the call and is never
left on the index, so a call returns the same thing whatever the index searched before it."""
import numpy as np
import pytest

import faiss_b200 as fb
from oracle import oracle_cagra_np as oc

pytestmark = pytest.mark.gpu


def test_sharded_cagra_search_after_a_paged_search():
    import torch  # noqa: F401  (maps PyTorch's NCCL, which the library then uses)

    rs = np.random.RandomState(11)
    d, n, nq, k, m = 64, 3000, 100, 10, 20
    # integer data: every fp32 distance is exact, so the kernel must replay the model bit for bit
    xb = rs.randint(-8, 9, (n, d)).astype(np.float32)
    xq = rs.randint(-8, 9, (nq, d)).astype(np.float32)
    graph = rs.randint(0, n, (n, 24))
    res = fb.StandardGpuResources()
    res.setPinnedMemory(2 * 16 * d * 4)
    index = fb.GpuIndexCagra(res, d, fb.METRIC_L2)
    index.copyFrom(xb, graph)
    index.setMinPagingSize(0)
    index.search(xq, k)  # host queries paged through two pinned buffers of 16: the last page starts at row 96
    try:
        res.ncclInitAll([0])
    except fb.FaissError as e:
        if "NCCL unavailable" in str(e):
            pytest.skip("NCCL cannot be loaded: %s" % e)
        raise
    shards = fb.DistributedIndexShards(res, index)
    D, I = shards.search(xq[:m], k)
    Dm, Im, count = oc.search_single_cta(xb, graph, xq[:m], k, row0=0)
    np.testing.assert_array_equal(I, Im)
    np.testing.assert_array_equal(D, Dm)
    assert index.lastSearchDistanceCount() == count
