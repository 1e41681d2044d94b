"""The pipelined tensor-core Flat kernel (112 < d <= 128: half-tile ring stages, a warpgroup filters one 128-column half
of a tile while the MMAs of the other run).

The tensor-core path must return bit for bit what the exact SIMT path returns, at dimensions that take the pipelined
kernel and at database sizes whose last tile is full, has one row, ends at its column half or has one row in its
second half (N mod 256 in {0, 1, 128, 129}).
"""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize(
    "N,d,nq,k",
    [
        (40960, 113, 300, 100),  # N mod 256 = 0
        (40961, 120, 300, 300),  # 1: the last tile's second half lies wholly past N
        (41088, 127, 300, 100),  # 128: ... and ends at the half
        (41089, 113, 130, 300),  # 129
        (41088, 120, 200, 1),  # k = 1: the streaming mode
        (40961, 127, 1000, 1),
        (40960, 113, 700, 1),
        (41089, 127, 64, 300),
    ],
)
def test_pipelined_tensor_core_path_equals_exact_path(res, N, d, nq, k, metric):
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda")
    g.manual_seed(N + d + k)
    xb = torch.rand(N, d, device="cuda", generator=g)
    xq = torch.rand(nq, d, device="cuda", generator=g)
    idx = fb.GpuIndexFlat(res, d, metric)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 0
    assert torch.equal(I, Ie)
    assert torch.equal(D, De)


@pytest.mark.parametrize("metric", [1, 0])
@pytest.mark.parametrize("N,d,k", [(41088, 120, 100), (40961, 127, 1)])
def test_pipelined_float16_storage(res, N, d, k, metric):
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda")
    g.manual_seed(7 * N + d)
    xb = torch.rand(N, d, device="cuda", generator=g)
    xq = torch.rand(150, d, device="cuda", generator=g)
    idx = fb.GpuIndexFlat(res, d, metric, use_float16=True)
    idx.add(xb)
    D, I = idx.search(xq, k)
    assert idx.lastSearchInfo()["tensor_cores"] == 1
    idx.setUseTensorCores(False)
    De, Ie = idx.search(xq, k)
    assert torch.equal(I, Ie) and torch.equal(D, De)


@pytest.mark.parametrize("N", [2049, 2176, 4096])
def test_pipelined_raw_scores_exact(res, N):
    """Small-integer fp16 operands make every fp32 score exact: each of the tile's columns, both halves and the
    zero-filled rows past N included, must hold exactly its dot product."""
    import torch

    import faiss_b200 as fb

    g = torch.Generator(device="cuda")
    g.manual_seed(N)
    nq, dpad = 200, 128
    Q = torch.randint(-4, 5, (nq, dpad), device="cuda", generator=g).half()
    Y = torch.randint(-4, 5, (N, dpad), device="cuda", generator=g).half()
    S = fb.flat_tc_scores_debug(res, Q, Y)
    ref = torch.zeros_like(S)
    ref[:, :N] = (Q.double() @ Y.double().T).float()
    assert torch.equal(S, ref)
