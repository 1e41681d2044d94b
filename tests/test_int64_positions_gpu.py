"""Both sides of the 32-bit / 64-bit position switches.

Flat search past 2^31 rows leaves the tensor cores for the exact kernel, which keeps split-relative 32-bit ids and
rebases them in its merge; a selective filter compacts the selected rows of the whole index first.  The IVF list
scans keep 64-bit arena positions in their per-warp and per-CTA top-k lists once the arena (its capacity, not its
stored vectors) reaches 2^31 - 1 slots; below that the int sentinel 2^31 - 1 must never collide with a slot.

Flat data are small integers, so every fp32 distance is exact and the expected result is the (distance, id)
order computed in int64 on the device.  IVF cases hold a few thousand vectors: capacity alone sets the scan's
id width, so each wide index is compared bit for bit with a narrow twin holding the same lists, and with float64
truth over its probed lists.  All data come from seeds on the device.  The CPU tests at the end check the int64
reference and the arena arithmetic at small sizes.
"""
import numpy as np
import pytest

from oracle import oracle_bound_np as ob
from oracle import oracle_ivf_check_np as oc

L2, IP = ob.METRIC_L2, ob.METRIC_INNER_PRODUCT
METRIC_L1 = 2
f32 = np.float32
FLT_MAX = float(np.finfo(np.float32).max)
TWO31 = 1 << 31
GiB = 1 << 30


# ------------------------------------------------------------------ exact int64 reference (device or host)
def exact_knn_int64(torch, xb, xq, k, metric, sel=None, chunk=1 << 24):
    """(D, I) of the (distance, id) order over the integer-valued rows of xb, computed exactly in int64, chunk rows
    at a time.  key = dist * 2^32 + id (inner product: -sim * 2^32 + id) is unique, so the chunks' top-k merge to
    the exact answer.  sel(r0, r1) -> bool [r1 - r0] restricts the search to the rows it keeps."""
    n, d = xb.shape
    q = xq.to(torch.int64)
    none = torch.iinfo(torch.int64).max
    best = None
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        y = xb[r0:r1].to(torch.int64)
        dist = torch.zeros((q.shape[0], r1 - r0), dtype=torch.int64, device=xb.device)
        for j in range(d):
            if metric == IP:
                dist += q[:, j : j + 1] * y[None, :, j]
            else:
                diff = q[:, j : j + 1] - y[None, :, j]
                dist += diff * diff if metric == L2 else diff.abs()
        key = (-dist if metric == IP else dist) * (1 << 32) + torch.arange(r0, r1, device=xb.device)[None, :]
        if sel is not None:
            key = torch.where(sel(r0, r1)[None, :], key, torch.full_like(key, none))
        part = torch.topk(key, min(k, r1 - r0), dim=1, largest=False, sorted=False).values
        if best is not None:
            part = torch.cat([best, part], dim=1)
            part = torch.topk(part, min(k, part.shape[1]), dim=1, largest=False, sorted=False).values
        best = part
    best = torch.sort(best, dim=1).values
    if best.shape[1] < k:
        best = torch.cat([best, torch.full((best.shape[0], k - best.shape[1]), none, dtype=torch.int64, device=best.device)], 1)
    missing = best == none
    ids = best & ((1 << 32) - 1)
    dist = torch.div(best - ids, 1 << 32, rounding_mode="floor")
    D = (-dist if metric == IP else dist).to(torch.float32)
    D[missing] = -FLT_MAX if metric == IP else FLT_MAX
    ids[missing] = -1
    return D, ids


def round32(n):
    return (np.asarray(n, dtype=np.int64) + 31) // 32 * 32


def narrow_top_caps(lens, top):
    """capacities with sum(round_up(cap, 32)) == top: every list but the first at its length (so the last list's
    last slot is the arena's last), the first list taking the rest"""
    lens = np.asarray(lens, dtype=np.int64)
    caps = lens.copy()
    caps[0] = top - int(round32(lens[1:]).sum())
    assert caps[0] >= lens[0] and caps[0] % 32 == 0
    return caps


def wide_list0_caps(lens, top):
    """list 0 reserved to round_up(top - 1, 32) == top slots: every other list starts at or past position top"""
    caps = np.asarray(lens, dtype=np.int64).copy()
    caps[0] = top - 1
    return caps


def reserve_caps(nlist, total):
    """IVFBase::reserveMemory's even spread of total vectors over nlist lists"""
    return np.full(nlist, -(-total // nlist), dtype=np.int64)


# ------------------------------------------------------------------ Flat past 2^31 rows
FLAT_N = TWO31 + (1 << 20)
FLAT_WINDOW = 1 << 19  # rows [2^31 - FLAT_WINDOW, N) hold the values nearest the queries


def _free_bytes(torch):
    return torch.cuda.mem_get_info()[0]


def _flat_rows(torch, N, d, B, window, seed, chunk=1 << 26):
    """integer rows: -1000..0 everywhere, 1..600 in [B - window, N) (ties across B for every value there)"""
    xb = torch.empty((N, d), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda")
    for c0 in range(0, N, chunk):
        c1 = min(N, c0 + chunk)
        g.manual_seed(seed + c0 // chunk)
        xb[c0:c1] = torch.randint(-1000, 1, (c1 - c0, d), generator=g, device="cuda", dtype=torch.int32).float()
    g.manual_seed(seed - 1)
    w0 = B - window
    xb[w0:] = torch.randint(1, 601, (N - w0, d), generator=g, device="cuda", dtype=torch.int32).float()
    return xb


def _flat_queries(torch, xb, N, d, B, nq, seed):
    """queries 700..1000 with exact matches planted at B - 1, B, B + 1 and N - 1, and one stored row duplicated on
    both sides of B"""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    xq = torch.randint(700, 1001, (nq, d), generator=g, device="cuda", dtype=torch.int32).float()
    for qi, row in enumerate((B - 1, B, B + 1, N - 1)):
        xb[row] = xq[qi]
    xb[B - 3] = xq[4]
    xb[B + 3] = xq[4]
    xb[B - 2] = xq[5]
    xb[N - 2] = xq[5]
    return xq


# class scope: the rows and the index are freed before the IVF cases need the memory
@pytest.fixture(scope="class", params=[(1, False), (2, True)], ids=["fp32_d1", "fp16_d2"])
def flat_big(request, res):
    import torch

    import faiss_b200 as fb

    d, fp16 = request.param
    N, nq = FLAT_N, 16
    # the rows, two indexes (the L2 one and one other metric at a time) and the reference's chunk temporaries
    need = N * d * 4 + 2 * N * d * (2 if fp16 else 4) + 12 * GiB
    if _free_bytes(torch) < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    xb = _flat_rows(torch, N, d, TWO31, FLAT_WINDOW, seed=4100 + d)
    xq = _flat_queries(torch, xb, N, d, TWO31, nq, seed=4200 + d)
    idx = fb.GpuIndexFlat(res, d, L2, use_float16=fp16)
    idx.add(xb)
    assert idx.ntotal == N
    yield d, fp16, xb, xq, idx
    del idx, xb, xq
    torch.cuda.empty_cache()


def _assert_equal_knn(D, I, eD, eI, what):
    import torch

    bad = ~((D == eD) & (I == eI)).all(dim=1)
    if bool(bad.any()):
        q = int(torch.nonzero(bad)[0])
        col = int(torch.nonzero((D[q] != eD[q]) | (I[q] != eI[q]))[0])
        raise AssertionError("%s: query %d rank %d: got (%r, %d), expected (%r, %d)" % (
            what, q, col, float(D[q, col]), int(I[q, col]), float(eD[q, col]), int(eI[q, col])))


@pytest.mark.gpu
class TestFlatPast2e31Rows:
    def test_flat_search_past_2e31_rows(self, res, flat_big):
        """search at k 1 ... 1024, L2 and IP (and L1 at one k), on the exact kernel: bit-exact with the int64 order"""
        import torch

        import faiss_b200 as fb

        d, fp16, xb, xq, idx = flat_big
        N = xb.shape[0]
        for metric in (L2, IP, METRIC_L1):
            index = idx if metric == L2 else fb.GpuIndexFlat(res, d, metric, use_float16=fp16)
            if metric != L2:
                index.add(xb)
            ks = (1, 10, 100, 1024) if metric != METRIC_L1 else (100,)
            eD, eI = exact_knn_int64(torch, xb, xq, max(ks), metric)
            for k in ks:
                D, I = index.search(xq, k)
                assert index.lastSearchInfo()["tensor_cores"] == 0
                _assert_equal_knn(D, I, eD[:, :k], eI[:, :k], "metric %d k %d" % (metric, k))
            if metric == L2:  # the planted exact matches on both sides of 2^31, and the duplicate pair's id order
                assert I[:4, 0].tolist() == [TWO31 - 1, TWO31, TWO31 + 1, N - 1] and bool((D[:4, 0] == 0).all())
                assert I[4, :2].tolist() == [TWO31 - 3, TWO31 + 3] and I[5, :2].tolist() == [TWO31 - 2, N - 2]
            assert bool((eI[:, :] >= TWO31).any(dim=1).all()), "every query's top 1024 reaches past 2^31"
            if metric != L2:
                del index
        torch.cuda.empty_cache()


    def test_flat_selectors_past_2e31_rows(self, res, flat_big):
        """a range around 2^31 keeping fewer than 1 row in 40 (the compacted search), its negation (the masked full
        search) and a bitmap: each equals the int64 reference restricted to the selected rows"""
        import torch

        import faiss_b200 as fb

        d, fp16, xb, xq, idx = flat_big
        N, k = xb.shape[0], 100
        lo, hi = TWO31 - (1 << 24), TWO31 + (1 << 19)  # its negation keeps rows on both sides of 2^31
        assert (hi - lo) * 40 <= N
        rng = fb.IDSelectorRange(lo, hi)

        def in_range(r0, r1):
            r = torch.arange(r0, r1, device="cuda")
            return (r >= lo) & (r < hi)

        # bitmap: rows whose byte index is odd, or rows 2^31 - 1 ... 2^31 + 6 (covering the planted matches)
        nbytes = (N + 7) // 8
        bm = np.zeros(nbytes, dtype=np.uint8)
        bm[1::2] = 0xFF
        bm[(TWO31 - 8) // 8] |= 0x80
        bm[TWO31 // 8] |= 0x7F
        bm_dev = torch.from_numpy(bm).cuda()

        def in_bitmap(r0, r1):
            r = torch.arange(r0, r1, device="cuda")
            return ((bm_dev[r >> 3] >> (r & 7).to(torch.uint8)) & 1).bool()

        cases = [
            ("range", rng, in_range),
            ("not range", fb.IDSelectorNot(rng), lambda r0, r1: ~in_range(r0, r1)),
            ("bitmap", fb.IDSelectorBitmap(bm), in_bitmap),
        ]
        for name, sel, member in cases:
            D, I = idx.search(xq, k, params=fb.SearchParameters(sel=sel))
            eD, eI = exact_knn_int64(torch, xb, xq, k, L2, sel=member)
            _assert_equal_knn(D, I, eD, eI, name)
            assert bool((I >= TWO31).any()), name
        torch.cuda.empty_cache()


    def test_flat_retrieval_past_2e31_rows(self, res, flat_big):
        """search_and_reconstruct and reconstruct_batch return the stored rows at ids past 2^31"""
        import torch

        d, fp16, xb, xq, idx = flat_big
        N = xb.shape[0]
        D, I, R = idx.search_and_reconstruct(xq, 10)
        assert bool((I >= TWO31).any())
        assert torch.equal(R, xb[I.reshape(-1)].reshape(I.shape[0], 10, d))
        keys = np.array([0, TWO31 - 2, TWO31 - 1, TWO31, TWO31 + 1, TWO31 + 12345, N - 2, N - 1], dtype=np.int64)
        assert np.array_equal(idx.reconstruct_batch(keys), xb[torch.from_numpy(keys).cuda()].cpu().numpy())
        assert np.array_equal(idx.reconstruct(N - 1), xb[N - 1].cpu().numpy())


# ------------------------------------------------------------------ IVF arenas on both sides of the switch
IVF_N, IVF_NQ, IVF_NLIST, IVF_NPROBE, IVF_K = 8192, 32, 64, 8, 50
NARROW_TOP = TWO31 - 32  # the largest arena whose slots all fit below the int sentinel 2^31 - 1
RESERVE = TWO31 + (1 << 26)  # reserveMemory over 64 lists: the last list starts past 2^31

# (kind, d, metric, option): IVF-Flat on integers (bit-exact); the four SQ codecs and 8bit_direct on integers
# (bit-exact); PQ M = 2 vector-major (8-bit) and packed (6-bit); PQ M = 16 8-bit, the interleaved CtaTopK scan
IVF_CASES = [
    ("flat", 1, L2, None),
    ("flat", 2, L2, None),
    ("flat", 2, IP, None),
    ("sq", 4, L2, 0),  # QT_8bit
    ("sq", 8, L2, 1),  # QT_4bit
    ("sq", 4, L2, 6),  # QT_6bit
    ("sq", 2, L2, 4),  # QT_fp16
    ("sq", 4, L2, 5),  # QT_8bit_direct
    ("pq", 4, L2, (2, 8)),
    ("pq", 4, L2, (2, 6)),
    ("pq", 16, L2, (16, 8)),
]
LAYOUTS = ["narrow_top", "wide_list0", "wide_reserve"]


def _make_ivf(res, kind, d, metric, opt):
    import faiss_b200 as fb

    if kind == "flat":
        return fb.GpuIndexIVFFlat(res, d, IVF_NLIST, metric)
    if kind == "sq":
        return fb.GpuIndexIVFScalarQuantizer(res, d, IVF_NLIST, opt, metric, encodeResidual=opt != fb.QT_8bit_direct)
    M, nbits = opt
    idx = fb.GpuIndexIVFPQ(res, d, IVF_NLIST, M, nbits, metric, interleaved_layout=nbits != 8)
    idx.setPrecomputedCodes(False)
    return idx


def _ivf_data(torch, kind, d, opt, n, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    if kind == "flat":
        return torch.randint(-1000, 1001, (n, d), generator=g, device="cuda", dtype=torch.int32).float()
    if kind == "sq" and opt == 5:  # 8bit_direct stores integers 0..255 as they are
        return torch.randint(0, 256, (n, d), generator=g, device="cuda", dtype=torch.int32).float()
    cent = torch.randn((64, d), generator=g, device="cuda") * 2
    pick = torch.randint(0, 64, (n,), generator=g, device="cuda")
    return cent[pick] + 0.5 * torch.randn((n, d), generator=g, device="cuda")


def _arena_bytes(layout, code_size, lens):
    slot = code_size + 8
    if layout == "narrow_top":
        return NARROW_TOP * slot
    if layout == "wide_list0":
        return (TWO31 + int(round32(lens[1:]).sum())) * slot
    return int(round32(reserve_caps(IVF_NLIST, RESERVE)).sum()) * slot


def _ivf_truth_check(idx, kind, d, metric, opt, xq, D, I, probes):
    """each query against float64 truth over its probed lists (bound 0 where the data are integers)"""
    cent = idx.getCoarseCentroids()
    exact = kind == "flat" or (kind == "sq" and opt == 5)
    for qi in range(xq.shape[0]):
        ids_all, t_all, b_all = [], [], []
        for l, li, raw in oc.probed_lists(idx, probes[qi]):
            if kind == "flat":
                Y = raw.view(f32).reshape(-1, d)
                t, b = ob.l2_truth(xq[qi], Y) if metric == L2 else ob.ip_truth(xq[qi], Y)
            elif kind == "sq":
                X, vmin, vdiff = oc.sq_exact_decode(raw, opt, idx.getTrained(), d)
                r = xq[qi].astype(np.float64) - (0.0 if opt == 5 else cent[l].astype(np.float64))
                t, b = ob.sq_l2_truth(r, X, vmin, vdiff)
            else:
                M, nbits = opt
                pq = idx.getPQCentroids()
                codes = oc.unpack(raw.reshape(li.size, -1), M, nbits)
                Yd = pq[np.arange(M)[None, :], codes].reshape(li.size, d)
                t, b = ob.pq_l2_truth(xq[qi].astype(np.float64) - cent[l], Yd, d // M, M)
            ids_all.append(li)
            t_all.append(t)
            b_all.append(np.zeros_like(t) if exact else b)
        ob.check_topk(D[qi], I[qi], np.concatenate(ids_all), np.concatenate(t_all), np.concatenate(b_all), IVF_K,
                      metric, what="%s d=%d query %d" % (kind, d, qi))


def _ivf_selectors(fb, n):
    """non-callback selectors over the ids 0..n-1"""
    rs = np.random.RandomState(n)
    bm = rs.randint(0, 256, (n + 7) // 8).astype(np.uint8)
    rng = fb.IDSelectorRange(n // 5, 3 * n // 4)
    arr = fb.IDSelectorArray(rs.choice(n, n // 3, replace=False))
    return [
        ("range", rng),
        ("array", arr),
        ("bitmap", fb.IDSelectorBitmap(bm)),
        ("not", fb.IDSelectorNot(rng)),
        ("and", fb.IDSelectorAnd(arr, fb.IDSelectorNot(rng))),
    ]


def _ivf_same(wide, twin, kind, d, metric, opt, xq, what):
    """everything a user reads from the wide index equals the narrow twin, bit for bit"""
    import torch

    import faiss_b200 as fb

    k, n = IVF_K, twin.ntotal
    assert wide.ntotal == n
    for l in range(IVF_NLIST):
        assert np.array_equal(wide.getListIndices(l), twin.getListIndices(l)), "%s list %d ids" % (what, l)
        assert np.array_equal(wide.getListVectorData(l), twin.getListVectorData(l)), "%s list %d codes" % (what, l)
    for idx in (wide, twin):
        idx.nprobe = IVF_NPROBE
    xq_d = torch.from_numpy(xq).cuda()

    def same(a, b, name):
        for x, y in zip(a, b):
            assert torch.equal(x, y) if torch.is_tensor(x) else np.array_equal(x, y), "%s: %s" % (what, name)

    same(wide.search(xq_d, k), twin.search(xq_d, k), "search")
    probes, cdis = oc.probes(xq, wide.getCoarseCentroids(), IVF_NPROBE, metric)
    D, I = wide.search_preassigned(xq, k, probes, cdis)
    same((D, I), twin.search_preassigned(xq, k, probes, cdis), "search_preassigned")
    _ivf_truth_check(wide, kind, d, metric, opt, xq, D, I, probes)
    for name, sel in _ivf_selectors(fb, n):
        p = fb.SearchParametersIVF(nprobe=IVF_NPROBE, sel=sel)
        same(wide.search(xq_d, k, params=p), twin.search(xq_d, k, params=p), "filtered search (%s)" % name)
    same(wide.search_and_reconstruct(xq_d, k), twin.search_and_reconstruct(xq_d, k), "search_and_reconstruct")
    same(wide.search_and_return_codes(xq_d, k, include_listnos=True),
         twin.search_and_return_codes(xq_d, k, include_listnos=True), "search_and_return_codes")
    assert np.array_equal(wide.reconstruct_n(0, n), twin.reconstruct_n(0, n)), what
    for key in (0, n // 2, n - 1):
        assert np.array_equal(wide.reconstruct(key), twin.reconstruct(key)), what


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("kind,d,metric,opt", IVF_CASES)
def test_ivf_arena_id_width(res, kind, d, metric, opt, layout):
    """a wide (or largest narrow) arena holding a few thousand vectors scans, filters, reconstructs, reclaims and
    grows exactly like a twin holding the same lists in an ordinary arena"""
    import torch

    seed = 1000 + 10 * IVF_CASES.index((kind, d, metric, opt))
    twin = _make_ivf(res, kind, d, metric, opt)
    x = _ivf_data(torch, kind, d, opt, IVF_N, seed)
    twin.setClustering(niter=4, seed=5)
    if kind == "pq":
        twin.setPQClustering(niter=4, seed=6)
    twin.train(x)
    # trim the last list to a multiple of 32, so an exact-fit last list ends on the arena's last slot
    twin.add(x)
    last = twin.getListIndices(IVF_NLIST - 1)
    keep = torch.ones(IVF_N, dtype=torch.bool, device="cuda")
    keep[torch.from_numpy(last[: last.size % 32]).cuda()] = False
    x = x[keep].contiguous()
    twin.reset()
    twin.add(x)
    lens = np.array([twin.getListLength(l) for l in range(IVF_NLIST)], dtype=np.int64)
    assert lens[-1] >= 32 and lens[-1] % 32 == 0
    cs = twin._code_size()
    arena = _arena_bytes(layout, cs, lens)
    # search_and_reconstruct also holds one 8-byte slot number per arena slot
    need = arena + arena // (cs + 8) * 8 + 4 * GiB
    if _free_bytes(torch) < need:
        pytest.skip("needs %.1f GB of free device memory for a %s arena" % (need / 1e9, layout))

    wide = _make_ivf(res, kind, d, metric, opt)
    wide.setCoarseCentroids(twin.getCoarseCentroids())
    if kind == "pq":
        wide.setPQCentroids(twin.getPQCentroids())
    if kind == "sq" and twin.getTrained().size:
        wide.setTrained(twin.getTrained())
    wide.setIsTrained(True)
    if layout == "narrow_top":
        wide.setListSizes(narrow_top_caps(lens, NARROW_TOP))
    elif layout == "wide_list0":
        wide.setListSizes(wide_list0_caps(lens, TWO31))
    else:
        wide.reserveMemory(RESERVE)
    wide.add(x)  # every list fits its capacity: no relayout
    xq = _ivf_data(torch, kind, d, opt, IVF_NQ, seed + 1)
    xq[: IVF_NQ // 2] = x[torch.arange(0, x.shape[0], x.shape[0] // (IVF_NQ // 2), device="cuda")[: IVF_NQ // 2]]
    xq = xq.cpu().numpy()
    what = "%s d=%d metric=%d %s %s" % (kind, d, metric, opt, layout)
    free, total = torch.cuda.mem_get_info()
    print("\n[%s] arena %.2f GB, device memory in use %.2f GB" % (what, arena / 1e9, (total - free) / 1e9))
    _ivf_same(wide, twin, kind, d, metric, opt, xq, what)
    # reclaim: the arena shrinks to exact fit (the freed bytes confirm the arena the layout meant)
    freed = wide.reclaimMemory()
    assert freed == arena - int(round32(lens).sum()) * (cs + 8), what
    _ivf_same(wide, twin, kind, d, metric, opt, xq, what + " after reclaim")
    # grow from the exact-fit arena
    x2 = _ivf_data(torch, kind, d, opt, 1000, seed + 2)
    twin.add(x2)
    wide.add(x2)
    _ivf_same(wide, twin, kind, d, metric, opt, xq, what + " after reclaim and add")
    del wide


# ------------------------------------------------------------------ CPU checks of the reference and the arithmetic
@pytest.mark.parametrize("metric", [L2, IP, METRIC_L1])
def test_exact_knn_int64_matches_numpy(metric):
    """the chunked int64 reference equals a numpy (distance, id) sort, with ties and a selection"""
    import torch

    rs = np.random.RandomState(metric)
    n, d, nq, k = 5003, 2, 7, 64
    xb = rs.randint(-20, 21, (n, d)).astype(f32)
    xq = rs.randint(-20, 21, (nq, d)).astype(f32)
    keep = rs.rand(n) < 0.3
    for sel in (None, keep):
        D, I = exact_knn_int64(
            torch, torch.from_numpy(xb), torch.from_numpy(xq), k, metric, chunk=611,
            sel=None if sel is None else (lambda r0, r1: torch.from_numpy(keep[r0:r1])))
        for qi in range(nq):
            q, y = xq[qi].astype(np.int64), xb.astype(np.int64)
            t = (q * y).sum(1) if metric == IP else ((q - y) ** 2).sum(1) if metric == L2 else np.abs(q - y).sum(1)
            ids = np.arange(n) if sel is None else np.nonzero(keep)[0]
            eD, eI = ob.exact_topk(t[ids].astype(np.float64), ids, k, IP if metric == IP else L2)  # L1: smallest first
            assert np.array_equal(D[qi].numpy(), eD) and np.array_equal(I[qi].numpy(), eI)


def test_exact_knn_int64_pads_missing():
    import torch

    D, I = exact_knn_int64(torch, torch.zeros((5, 1)), torch.zeros((2, 1)), 8, L2, sel=lambda r0, r1: torch.arange(r0, r1) < 3)
    assert I[0].tolist() == [0, 1, 2, -1, -1, -1, -1, -1] and float(D[0, 3]) == FLT_MAX


@pytest.mark.parametrize("top", [1 << 13, TWO31])
def test_arena_layouts(top):
    """the layouts' slot arithmetic at a small and at the real switch"""
    rs = np.random.RandomState(top % 1000)
    lens = rs.randint(1, 60, IVF_NLIST).astype(np.int64)
    lens[-1] = 96
    caps = narrow_top_caps(lens, top - 32)
    assert int(round32(caps).sum()) == top - 32 and caps[-1] == lens[-1]
    start_last = int(round32(caps[:-1]).sum())
    assert start_last + lens[-1] - 1 == top - 33  # the last list's last vector sits in the arena's top slot
    caps = wide_list0_caps(lens, top)
    assert int(round32(caps[:1]).sum()) == top and (caps[1:] == lens[1:]).all()
    if top == TWO31:
        caps = reserve_caps(IVF_NLIST, RESERVE)
        starts = np.concatenate([[0], np.cumsum(round32(caps))[:-1]])
        assert starts[-1] >= TWO31 and round32(caps).sum() >= TWO31 - 1
        assert _arena_bytes("narrow_top", 4, lens) == (TWO31 - 32) * 12
