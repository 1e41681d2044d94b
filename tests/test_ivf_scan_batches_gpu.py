"""Query batching of the IVF list scans.  A scan call splits its queries into batches that bound the partial-result
scratch: at most 65535 queries, and at most 2^30 / (CTAs per query * k * 12) of them.  Each batch is one scan launch
(one KernelTiming record) and one merge launch, and the result must equal that of the same queries searched in
blocks that fit one batch."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, NLIST = 20000, 64
L2, IP = 1, 0

# name: (index, d, metric, options, timing name)
CASES = {
    "flat_d128": ("flat", 128, L2, {}, b"ivfflat_scan"),
    "flat_d40_ip": ("flat", 40, IP, {}, b"ivfflat_scan"),
    "pq_m16_l2": ("pq", 64, L2, {"M": 16}, b"ivfpq_scan"),
    "pq_m16_ip": ("pq", 64, IP, {"M": 16}, b"ivfpq_scan"),
    "pq_m32_precomputed": ("pq", 64, L2, {"M": 32, "precomputed": True}, b"ivfpq_scan"),
    "pq_m8_vector_major": ("pq", 64, L2, {"M": 8}, b"ivfpq_scan"),
    "pq_m16_6bit_packed": ("pq", 64, L2, {"M": 16, "nbits": 6}, b"ivfpq_scan_packed"),
    "pq_m32_4bit_nibble": ("pq", 64, L2, {"M": 32, "nbits": 4}, b"ivfpq_scan"),
    "sq_8bit_d128": ("sq", 128, L2, {"qtype": 0}, b"ivfsq_scan"),
    "sq_6bit_d40_ip": ("sq", 40, IP, {"qtype": 6}, b"ivfsq_scan"),
}

# the vector-major and packed PQ scans run one CTA per (query, probe): their batch bound is 2^30 / (nprobe * k * 12)
ONE_CTA_PER_PROBE = {"pq_m8_vector_major", "pq_m16_6bit_packed"}


def _build(res, kind, d, metric, opt):
    import faiss_b200 as fb

    if kind == "flat":
        idx = fb.GpuIndexIVFFlat(res, d, NLIST, metric)
    elif kind == "pq":
        nbits = opt.get("nbits", 8)
        idx = fb.GpuIndexIVFPQ(res, d, NLIST, opt["M"], nbits, metric, interleaved_layout=nbits != 8)
        idx.setPQClustering(niter=4)
        if opt.get("precomputed"):
            idx.setPrecomputedCodes(True)
    else:
        idx = fb.GpuIndexIVFScalarQuantizer(res, d, NLIST, opt["qtype"], metric, encodeResidual=True)
    idx.setClustering(niter=4)
    xb = np.random.RandomState(5).rand(N, d).astype(np.float32)
    idx.train(xb)
    idx.add(xb)
    return idx


def _assert_same(D, I, Db, Ib):
    assert np.array_equal(Db, D)
    # ids may only differ inside runs of exactly tied distances
    diff = Ib != I
    if diff.any():
        tied = np.zeros_like(diff)
        tied[:, 1:] |= D[:, 1:] == D[:, :-1]
        tied[:, :-1] |= D[:, :-1] == D[:, 1:]
        assert not (diff & ~tied).any()


@pytest.mark.parametrize("name", sorted(CASES))
def test_ivf_scan_query_batches(res, name):
    import torch

    import faiss_b200 as fb

    kind, d, metric, opt, timing = CASES[name]
    idx = _build(res, kind, d, metric, opt)
    if name in ONE_CTA_PER_PROBE:
        nq, k, nprobe, block = 3000, 1024, 64, 1000
        batches = -(-nq // ((1 << 30) // (nprobe * k * 12)))  # 1365 queries per batch: 3 batches
    else:
        nq, k, nprobe, block = 70000, 5, 4, 35000
        batches = -(-nq // 65535)  # 2 batches
    assert batches in (2, 3)
    idx.nprobe = nprobe

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(17)
    xq = torch.rand((nq, d), dtype=torch.float32, device=dev, generator=g)
    cent = torch.from_numpy(idx.getCoarseCentroids()).to(dev)
    if metric == L2:
        cdis, assign = torch.cdist(xq, cent).square().topk(nprobe, dim=1, largest=False)
    else:
        cdis, assign = (xq @ cent.T).topk(nprobe, dim=1)
    cdis, assign = cdis.contiguous(), assign.contiguous()

    D, I = idx.search_preassigned(xq, k, assign, cdis)  # warm-up: term-2 tables, shared-memory probe
    fb.lib.faiss_b200_kernel_timing(1)
    kms, kn = ctypes.c_double(), ctypes.c_int()
    fb.lib.faiss_b200_kernel_timing_collect(timing, ctypes.byref(kms), ctypes.byref(kn))  # clears
    l0 = fb.lib.faiss_b200_launch_count()
    D2, I2 = idx.search_preassigned(xq, k, assign, cdis)
    torch.cuda.synchronize()
    launches = fb.lib.faiss_b200_launch_count() - l0
    fb.lib.faiss_b200_kernel_timing_collect(timing, ctypes.byref(kms), ctypes.byref(kn))
    fb.lib.faiss_b200_kernel_timing(0)
    assert launches == 2 * batches  # one scan and one merge per batch
    assert kn.value == batches

    D, I = D.cpu().numpy(), I.cpu().numpy()
    assert (I[:, 0] >= 0).all()
    _assert_same(D, I, D2.cpu().numpy(), I2.cpu().numpy())
    for q0 in range(0, nq, block):
        Db, Ib = idx.search_preassigned(xq[q0 : q0 + block], k, assign[q0 : q0 + block], cdis[q0 : q0 + block])
        _assert_same(D[q0 : q0 + block], I[q0 : q0 + block], Db.cpu().numpy(), Ib.cpu().numpy())
