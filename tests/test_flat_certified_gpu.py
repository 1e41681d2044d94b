"""Every Flat search route at d <= 256 against float64 truth on the device, under the certified top-k check
(oracle/oracle_bound_torch.certify_knn: check_topk's four conditions for every query against every row).

Each case names the route it is meant to take and asserts it took it (lastSearchInfo()["tensor_cores"] and
lastSearchOperandBits(): 0 for the exact kernel, 16 for fp16 tensor-core scoring, 8 for int8), so none quietly tests
only the exact kernel; the certificate must hold whatever the number of exact fallback recomputes.  knn_gpu cannot
report its route: it builds a default GpuIndexFlat over its rows (widened to fp32), so its cases assert the route on a
default index over the same widened rows and require knn_gpu's result to equal that index's bit for bit.  The equality
checks the conversions and the output paths; it does not pin the route, since every route returns the same bits on
integer data and the tensor-core paths equal the exact kernel on the rest.  test_case_list_covers_the_routes needs no
GPU.

Routes: the exact kernel (flat_exact.cu) over its tile configurations (k = 1, k <= 256, <= 1024, <= 2048), over
d = 1 ... 256 (float4 and scalar loads, the 16-wide chunk tail), nq = 1 and 5 (database split and merge) and
several query tiles, with fp32 and fp16 storage, a row mask and a compacted selector; the fp16 tensor-core search
(flat_tc.cu) in each dpad class (d <= 64, <= 112, the quad kernel at <= 128, the K-split at <= 256), in streaming
mode (k = 1), with bisection and with sorted base lists, at N = 32768 and one row past a whole tile, over one and
several query batches; the int8 search at 112 < d <= 128.  Data: uniform, clustered (queries next to rows: the
completeness clause has teeth), Gaussian inner products (cancellation) and small integers (every fp32 sum exact:
bound 0, the exact top-k including the rank-k tie group), with rows duplicated hundreds of times, so that tie groups
span tiles and rounds and some queries fail their certificate and are recomputed.
"""

import numpy as np
import pytest

from oracle import oracle_bound_np as ob

L2, IP = ob.METRIC_L2, ob.METRIC_INNER_PRODUCT
EXACT, TC16, TC8 = 0, 16, 8


# ------------------------------------------------------------------ data, generated on the device
def _data(kind, N, nq, d, seed):
    import torch

    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    dev = "cuda"
    if kind == "int":
        xb = torch.randint(0, 16, (N, d), generator=g, device=dev).float()
        xq = torch.randint(0, 16, (nq, d), generator=g, device=dev).float()
        if N >= 4096:  # three rows stored N / 48 times each, spread over the database
            dup = torch.randperm(N, generator=g, device=dev)[: 3 * (N // 48)].view(3, -1)
            for r in range(3):
                xb[dup[r]] = xb[dup[r, 0]].clone()
        # a third of the queries are stored rows (the duplicated ones among them): distance 0, ties at rank k
        src = torch.randint(0, N, (nq // 3,), generator=g, device=dev)
        if N >= 4096:
            src[::2] = dup.flatten()[torch.randint(0, dup.numel(), (src[::2].numel(),), generator=g, device=dev)]
        xq[: nq // 3] = xb[src].clone()
    elif kind == "uniform":
        xb = torch.rand((N, d), generator=g, device=dev)
        xq = torch.rand((nq, d), generator=g, device=dev)
    elif kind == "outlier":  # one huge coordinate: the int8 fitness test fails, fp16 serves the database
        xb = torch.rand((N, d), generator=g, device=dev)
        xb[N // 3, 0] = 1000.0
        xq = torch.rand((nq, d), generator=g, device=dev)
    elif kind == "gauss":
        xb = torch.randn((N, d), generator=g, device=dev)
        xq = torch.randn((nq, d), generator=g, device=dev)
    else:
        assert kind == "clustered"
        cent = torch.randn((64, d), generator=g, device=dev) * 2
        xb = cent[torch.randint(0, 64, (N,), generator=g, device=dev)] + 0.5 * torch.randn((N, d), generator=g, device=dev)
        xq = xb[torch.randint(0, N, (nq,), generator=g, device=dev)] + 0.01 * torch.randn((nq, d), generator=g, device=dev)
    return xb.contiguous(), xq.contiguous()


def _mask(N, frac, seed):
    rs = np.random.RandomState(seed)
    m = np.zeros(N, bool)
    m[rs.choice(N, max(1, int(N * frac)), replace=False)] = True
    return m


def _bitmap_params(fb, m):
    return fb.SearchParameters(sel=fb.IDSelectorBitmap(np.packbits(m, bitorder="little")))


# ------------------------------------------------------------------ the case list
# (route, api, d, k, N, nq, metric, kind, fp16 storage, selector): route EXACT / TC16 / TC8; api "index" (device
# queries), "host" (numpy queries), "bf_f32" / "bf_f16" / "bf_bf16" / "bf_colmajor" / "bf_i32" / "tiling" (knn_gpu),
# "shards" (IndexShards over two tensor-core shards); selector None, "mask" (half the rows: the masked search) or
# "compact" (1 row in 50: the gathered rows on the exact kernel)
K_EXACT = [1, 2, 100, 128, 129, 256, 257, 1024, 1025, 2048]  # Argmin, TQ 32 (LIST >= 128), TQ 16, TQ 8 / TN 128
D_EXACT = [1, 2, 3, 15, 16, 17, 63, 64, 65, 127, 128, 200, 255, 256]
NQ_EXACT = [1, 5, 70, 200, 33, 300]


def _cases():
    out = []
    kinds = ["uniform", "clustered", "int", "gauss"]
    # the exact kernel: every d with two k of the ladder, every k at least twice
    for i, d in enumerate(D_EXACT + D_EXACT[::-1]):
        k = K_EXACT[(i * 3) % len(K_EXACT)]
        metric = IP if i % 3 == 2 else L2
        kind = kinds[i % 4] if metric == L2 or kinds[i % 4] != "clustered" else "gauss"
        out.append((EXACT, "index" if i % 4 else "host", d, k, 20000, NQ_EXACT[i % len(NQ_EXACT)], metric, kind,
                    i % 3 == 1, None))
    out += [
        (EXACT, "index", 64, 100, 40000, 70, L2, "uniform", False, "mask"),
        (EXACT, "index", 200, 257, 40000, 5, IP, "gauss", True, "mask"),
        (EXACT, "index", 17, 1025, 20000, 33, L2, "int", False, "mask"),
        (EXACT, "index", 128, 100, 100000, 200, L2, "uniform", False, "compact"),
        (EXACT, "index", 65, 1025, 100000, 33, IP, "gauss", True, "compact"),
        (EXACT, "host", 17, 2048, 100000, 16, L2, "int", False, "compact"),  # 2000 rows selected, fewer than k
    ]
    # fp16 tensor cores: dpad classes x k regimes x N edges x batches
    out += [
        # d <= 64 (one K-block)
        (TC16, "index", 64, 10, 32768, 16, L2, "uniform", False, None),
        (TC16, "index", 32, 100, 40961, 129, IP, "gauss", False, None),
        (TC16, "host", 3, 64, 50000, 129, L2, "clustered", False, None),
        (TC16, "index", 1, 128, 32768, 40, L2, "int", False, None),
        (TC16, "index", 64, 1, 2048, 16, L2, "uniform", False, None),  # streaming from its N threshold
        (TC16, "index", 63, 129, 40961, 200, L2, "int", False, None),
        (TC16, "index", 64, 2048, 65536, 129, IP, "gauss", False, None),
        # 64 < d <= 112 (two K-blocks, whole-tile stages)
        (TC16, "index", 65, 128, 40961, 200, L2, "clustered", False, None),
        (TC16, "host", 100, 100, 100000, 129, IP, "gauss", False, None),
        (TC16, "index", 112, 256, 65536, 300, L2, "uniform", False, None),
        (TC16, "index", 96, 1, 100000, 500, L2, "clustered", False, None),
        (TC16, "index", 80, 1024, 32768, 64, L2, "int", False, None),
        # 112 < d <= 128: the quad kernel, kept on fp16 by IP, k = 1, k > 128 or an unfit database
        (TC16, "index", 128, 100, 100000, 129, IP, "gauss", False, None),
        (TC16, "index", 120, 1, 4096, 300, L2, "uniform", False, None),
        (TC16, "index", 128, 1, 50000, 129, L2, "int", False, None),
        (TC16, "index", 128, 129, 40961, 129, L2, "uniform", False, None),
        (TC16, "host", 113, 512, 65536, 200, L2, "clustered", False, None),
        (TC16, "index", 128, 100, 50000, 129, L2, "outlier", False, None),
        (TC16, "index", 127, 2048, 32768, 40, L2, "int", False, None),
        # 128 < d <= 256: K-split with 3 and 4 K-blocks
        (TC16, "index", 129, 100, 40961, 129, L2, "clustered", False, None),
        (TC16, "index", 192, 1024, 65536, 129, L2, "uniform", False, None),
        (TC16, "index", 200, 64, 100000, 200, IP, "gauss", False, None),
        (TC16, "index", 256, 2048, 40000, 33, L2, "int", False, None),
        (TC16, "index", 255, 1, 100000, 129, IP, "gauss", False, None),
        (TC16, "host", 256, 128, 32768, 16, IP, "int", False, None),
        (TC16, "index", 176, 410, 50000, 300, L2, "clustered", False, None),
        # more than one query batch: qBatch 2048 at k >= 1024, 3276 at k = 512, 67584 in streaming mode
        (TC16, "index", 64, 1024, 65536, 5000, L2, "int", False, None),
        (TC16, "index", 96, 2048, 40000, 4500, L2, "clustered", False, None),
        (TC16, "index", 32, 512, 50000, 7000, IP, "gauss", False, None),
        (TC16, "index", 32, 1, 40000, 140000, L2, "uniform", False, None),
        (TC16, "index", 16, 1, 40000, 140000, L2, "int", False, None),
        # fp16 storage and the selector's row mask
        (TC16, "index", 64, 100, 50000, 129, L2, "uniform", True, None),
        (TC16, "host", 200, 257, 40000, 129, IP, "gauss", True, None),
        (TC16, "index", 128, 1, 40000, 200, L2, "int", True, None),
        (TC16, "index", 64, 100, 50000, 129, L2, "uniform", False, "mask"),
        (TC16, "index", 200, 1024, 40000, 64, IP, "gauss", False, "mask"),
        (TC16, "index", 32, 1, 40000, 300, L2, "int", False, "mask"),
        (TC16, "index", 100, 2048, 100000, 5000, L2, "int", True, "mask"),
    ]
    # int8 tensor cores: every d of {113, 120, 127, 128} with two k of {2, 64, 100, 128}
    for i, (d, k) in enumerate(list(zip([113, 120, 127, 128], [2, 64, 100, 128]))
                               + list(zip([113, 120, 127, 128], [128, 100, 64, 2]))):
        out.append((TC8, "index" if i % 3 else "host", d, k, [32768, 40961, 100000, 200000][i % 4],
                    [16, 129, 1000, 300][(i + 1) % 4], L2, "int" if i % 2 else "uniform", False, None))
    out += [
        (TC8, "index", 120, 100, 40000, 140000, L2, "int", False, None),  # three query batches of 65536
        (TC8, "index", 128, 64, 100000, 129, L2, "uniform", False, "mask"),
        (TC8, "index", 128, 100, 50000, 129, L2, "int", True, None),
    ]
    # the bfKnn / knn_gpu entry points and IndexShards
    out += [
        (TC16, "bf_f32", 64, 100, 50000, 129, L2, "uniform", False, None),
        (TC16, "bf_f16", 64, 100, 50000, 129, L2, "clustered", False, None),
        (TC16, "bf_bf16", 200, 257, 40000, 64, IP, "gauss", False, None),
        (TC8, "bf_bf16", 128, 100, 50000, 129, L2, "int", False, None),
        (TC16, "bf_colmajor", 100, 128, 40961, 129, IP, "gauss", False, None),
        (EXACT, "bf_colmajor", 100, 1025, 20000, 33, L2, "uniform", False, None),
        (TC16, "bf_i32", 64, 1024, 50000, 129, L2, "int", False, None),
        (TC8, "bf_i32", 120, 2, 50000, 129, L2, "uniform", False, None),
        (TC16, "tiling", 64, 100, 100000, 129, L2, "clustered", False, None),
        (TC16, "tiling", 200, 1, 100000, 200, IP, "gauss", False, None),
        (TC16, "shards", 64, 100, 80000, 129, L2, "uniform", False, None),
        (TC16, "shards", 200, 257, 80000, 129, IP, "gauss", False, None),
    ]
    return out


CASES = _cases()


def _case_id(c):
    route, api, d, k, N, nq, metric, kind, fp16, sel = c
    return "%s-%s-d%d-k%d-N%d-nq%d-%s-%s%s%s" % (
        {EXACT: "exact", TC16: "tc16", TC8: "tc8"}[route], api, d, k, N, nq, "l2" if metric == L2 else "ip", kind,
        "-fp16" if fp16 else "", "-" + sel if sel else "")


IDS = [_case_id(c) for c in CASES]
assert len(set(IDS)) == len(IDS), "case ids must be unique"


# ------------------------------------------------------------------ running one case
def _index(fb, res, d, metric, fp16, route, rows):
    idx = fb.GpuIndexFlat(res, d, metric, use_float16=fp16)
    idx.add(rows)
    if route == EXACT:
        idx.setUseTensorCores(False)
    return idx


def _assert_route(info, bits, route, what):
    want_tc = int(route != EXACT)
    assert info["tensor_cores"] == want_tc and bits == route, "%s: took tensor_cores %d, operand bits %d" % (
        what, info["tensor_cores"], bits)


def _search_bf(fb, res, api, xq, xb, k, metric, route):
    """knn_gpu through one of its input forms, checked bit for bit against a default GpuIndexFlat over the same rows (what
    knn_gpu builds inside) whose route is asserted; returns (D, I, queries, rows as the kernel saw them, fallbacks)"""
    import torch

    if api == "tiling":
        shard = 40000  # three shards of 40000, 40000 and 20000 rows; k > 1: the last one on the exact kernel
        xqh, xbh = xq.cpu().numpy(), xb.cpu().numpy()
        D, I = fb.knn_gpu(res, xqh, xbh, k, metric=metric, vectorsMemoryLimit=shard * xb.shape[1] * 4)
        parts, fallbacks = [], 0
        for s0 in range(0, xb.shape[0], shard):
            idx = fb.GpuIndexFlat(res, xb.shape[1], metric)
            idx.add(xbh[s0:s0 + shard])
            pD, pI = idx.search(xqh, k)
            info = idx.lastSearchInfo()
            rows = min(shard, xb.shape[0] - s0)
            _assert_route(info, idx.lastSearchOperandBits(), route if rows >= (2048 if k == 1 else 32768) else EXACT,
                          "shard %d" % s0)
            fallbacks += info["fallback_queries"]
            parts.append((pD, np.where(pI >= 0, pI + s0, -1)))
        # shards in id order, each query's lists merged in the (key, id) order
        allD = np.concatenate([p[0] for p in parts], 1)
        allI = np.concatenate([p[1] for p in parts], 1)
        key = allD if metric == L2 else -allD
        wI = np.empty_like(I)
        wD = np.empty_like(D)
        for qi in range(xqh.shape[0]):
            o = np.lexsort((np.where(allI[qi] < 0, np.iinfo(np.int64).max, allI[qi]), key[qi]))[:k]
            wD[qi], wI[qi] = allD[qi, o], allI[qi, o]
        assert np.array_equal(D, wD) and np.array_equal(I, wI), "tiled knn_gpu differs from the merged shards"
        return D, I, xq, xb, fallbacks
    if api == "bf_f16":
        q, y = xq.half(), xb.half()
    elif api == "bf_bf16":
        q, y = xq.bfloat16(), xb.bfloat16()
    elif api == "bf_colmajor":
        q, y = xq.t().contiguous().t(), xb.t().contiguous().t()
        assert not y.is_contiguous() and y.t().is_contiguous()
    else:
        q, y = xq, xb
    if api == "bf_i32":
        I32 = torch.empty((xq.shape[0], k), dtype=torch.int32, device="cuda")
        D, I = fb.knn_gpu(res, q, y, k, I=I32, metric=metric)
        assert I is I32
    else:
        D, I = fb.bfKnn(res, q, y, k, metric)
    torch.cuda.synchronize()
    ref = fb.GpuIndexFlat(res, xb.shape[1], metric)
    ref.add(y.float().contiguous())
    rD, rI = ref.search(q.float().contiguous(), k)
    info = ref.lastSearchInfo()
    _assert_route(info, ref.lastSearchOperandBits(), route, "GpuIndexFlat over the knn_gpu rows")
    assert torch.equal(D, rD) and torch.equal(I.long(), rI), "knn_gpu differs from GpuIndexFlat over the same rows"
    return D, I, q, y, info["fallback_queries"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_flat_route_certified(res, case, record_property):
    import torch

    import faiss_b200 as fb
    from oracle import oracle_bound_torch as obt

    route, api, d, k, N, nq, metric, kind, fp16, sel = case
    what = _case_id(case)
    xb, xq = _data(kind, N, nq, d, seed=d * 7919 + k * 31 + N + nq)
    mask = None
    if api.startswith("bf_") or api == "tiling":
        D, I, Qk, Yk, fallbacks = _search_bf(fb, res, api, xq, xb, k, metric, route)
    elif api == "shards":
        shards = fb.IndexShards(d, threaded=False, successive_ids=True)
        parts = []
        for s in range(2):
            p = fb.GpuIndexFlat(res, d, metric)
            p.add(xb[s * (N // 2):(s + 1) * (N // 2)])
            parts.append(p)
            shards.add_shard(p)
        D, I = shards.search(xq.cpu().numpy(), k)
        fallbacks = 0
        for s, p in enumerate(parts):
            _assert_route(p.lastSearchInfo(), p.lastSearchOperandBits(), route, "shard %d" % s)
            fallbacks += p.lastSearchInfo()["fallback_queries"]
        Qk, Yk = xq, xb
    else:
        idx = _index(fb, res, d, metric, fp16, route, xb)
        params = None
        if sel is not None:
            mask = _mask(N, 0.5 if sel == "mask" else 0.02, seed=N + k)
            if sel == "compact":
                assert mask.sum() * 40 <= N  # the gathered rows on the exact kernel
            params = _bitmap_params(fb, mask)
        if api == "host":
            D, I = idx.search(xq.cpu().numpy(), k, params=params)
        else:
            D, I = idx.search(xq, k, params=params)
        info = idx.lastSearchInfo()
        _assert_route(info, idx.lastSearchOperandBits(), route, what)
        fallbacks = info["fallback_queries"]
        # what the kernels saw: fp16 storage rounds the rows and the queries
        Qk, Yk = (xq.half().float(), xb.half().float()) if fp16 else (xq, xb)
        if fp16:
            assert np.array_equal(idx.reconstruct_n(0, min(N, 1000)), Yk[:1000].cpu().numpy())
    record_property("fallback_queries", fallbacks)
    cand = None if mask is None else torch.from_numpy(mask).cuda()
    obt.certify_knn(D, I, Qk, Yk, k, metric, candidates=cand, exact=kind == "int",
                    what="%s (%d fallbacks)" % (what, fallbacks))


def test_case_list_covers_the_routes():
    """the axes of the list: every k and d of the exact kernel's ladders, every dpad class and k regime of the
    tensor-core search on both metrics, the int8 shapes, several query batches, every entry point"""
    ex = [c for c in CASES if c[0] == EXACT]
    assert {c[3] for c in ex} >= set(K_EXACT) and {c[2] for c in ex} >= set(D_EXACT)
    assert {c[5] for c in ex} >= {1, 5} and {c[8] for c in ex} == {False, True}
    assert {c[9] for c in ex} == {None, "mask", "compact"}
    tc = [c for c in CASES if c[0] == TC16]
    dpad = lambda d: 0 if d <= 64 else 1 if d <= 112 else 2 if d <= 128 else 3  # noqa: E731
    for cls in range(4):
        got = [c for c in tc if dpad(c[2]) == cls]
        assert {c[6] for c in got} == {L2, IP}, cls
        assert any(c[3] == 1 for c in got) and any(1 < c[3] <= 128 for c in got) and any(c[3] > 128 for c in got), cls
    assert {c[4] for c in tc} >= {2048, 32768, 40961}
    assert any(c[3] >= 1024 and c[5] > 2 * 2048 for c in tc) and any(c[3] == 1 and c[5] > 2 * 67584 for c in tc)
    t8 = [c for c in CASES if c[0] == TC8]
    assert {c[2] for c in t8} >= {113, 120, 127, 128} and {c[3] for c in t8} >= {2, 64, 100, 128}
    assert any(c[5] > 2 * 65536 for c in t8)
    assert {c[7] for c in CASES} == {"uniform", "clustered", "gauss", "int", "outlier"}
    assert {c[1] for c in CASES} == {"index", "host", "bf_f32", "bf_f16", "bf_bf16", "bf_colmajor", "bf_i32", "tiling",
                                     "shards"}
