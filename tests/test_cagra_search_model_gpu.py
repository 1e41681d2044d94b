"""GpuIndexCagra against its numpy restatement (oracle/oracle_cagra_np.py).

The search is deterministic (DESIGN §3.10): entry ids are splitmix64(seed, row, i) mod N, the top-k is ordered by
(key, id), and the visited set is refilled on a schedule of gather slots.  On integer-valued data every fp32 distance is
exact, so the kernel must return the model's D and I bit for bit, and its distance count exactly, at every team size,
block size, itopk, search width, iteration limit and refill schedule.  Graphs are loaded with copyFrom, so the search
is tested apart from the build; the build is then compared with the exact-kNN-then-optimise oracle on data where its
candidates cover every row, and cagra_optimize with the oracle over more shapes."""
import ctypes

import numpy as np
import pytest

import faiss_b200 as fb
from faiss_b200 import cloner
from oracle import oracle_cagra_np as oc

pytestmark = pytest.mark.gpu

NQ = 16
U32 = 2.0**-24  # fp32 unit roundoff


@pytest.fixture(scope="module")
def res():
    return fb.StandardGpuResources()


def _int_data(rs, n, d):
    # integers in [-8, 8]: every partial sum of an L2 (<= 256 d) or inner product (<= 64 d) stays below 2^24 up to
    # d = 1000, so fp32 is exact for both metrics
    return rs.randint(-8, 9, (n, d)).astype(np.float32)


def _random_graph(rs, n, K):
    """a directed graph with duplicate entries, self entries and -1 scattered through the rows"""
    g = rs.randint(0, n, (n, K))
    m = rs.rand(n, K)
    g[m < 0.1] = -1
    rows = np.arange(n)[:, None]
    g = np.where((m >= 0.1) & (m < 0.15), rows, g)  # self entries
    if K > 1:
        dup = (m >= 0.15) & (m < 0.2)
        g[:, 1:] = np.where(dup[:, 1:], g[:, :-1], g[:, 1:])  # repeat the entry before
    return g


_GRAPHS = {}


def _graph(kind, x, K, ip, seed):
    n = x.shape[0]
    key = (kind, x.tobytes(), K, ip, seed)
    if key not in _GRAPHS:
        rs = np.random.RandomState(seed)
        if kind == "knn":
            K0 = min(2 * K, n - 1)
            _GRAPHS[key] = oc.optimize(oc.exact_knn_graph(x, K0, ip), min(K, K0))
        elif kind == "rand":
            _GRAPHS[key] = _random_graph(rs, n, K)
        elif kind == "disc":
            # islands of 3 nodes (n % 3 == 0), each row's two island mates at random slots among -1: a walk
            # reaches the islands of its samples only
            assert n % 3 == 0 and K >= 2
            g = np.full((n, K), -1)
            for u in range(n):
                base = u - u % 3
                g[u, rs.choice(K, 2, replace=False)] = [v for v in (base, base + 1, base + 2) if v != u]
            _GRAPHS[key] = g
        else:
            raise ValueError(kind)
    return _GRAPHS[key]


def _index(res, xb, graph, ip):
    index = fb.GpuIndexCagra(res, xb.shape[1], fb.METRIC_INNER_PRODUCT if ip else fb.METRIC_L2)
    index.copyFrom(xb, graph)
    return index


# (id, n, d, graph kind, K, k, params): every sweep point of DESIGN §3.10's search occurs at least once
CASES = [
    ("d1-knn", 2000, 1, "knn", 16, 10, {}),
    ("d3-team4-itopk33", 2000, 3, "rand", 3, 10, dict(itopk_size=33, team_size=4)),
    ("d3-team16-blk64", 2000, 3, "rand", 24, 10, dict(team_size=16, thread_block_size=64)),
    ("d5-k1-itopk10-blk1024-seedmax", 2000, 5, "rand", 24, 1, dict(itopk_size=10, thread_block_size=1024, seed=2**64 - 1)),
    ("d5-k=itopk64", 2000, 5, "knn", 24, 64, dict(itopk_size=64)),
    ("d17-k=itopk96-sw3-team8", 2000, 17, "knn", 32, 96, dict(itopk_size=96, search_width=3, team_size=8)),
    ("d64-itopk500-blk512-team16", 2000, 64, "rand", 128, 10, dict(itopk_size=500, thread_block_size=512, team_size=16)),
    ("d64-itopk256-blk1024-team4-sw3", 2000, 64, "rand", 24, 10, dict(itopk_size=256, thread_block_size=1024, team_size=4, search_width=3)),
    ("d64-sw8-fill0.1", 2000, 64, "rand", 24, 10, dict(search_width=8, hashmap_max_fill_rate=0.1)),
    ("d100-k=itopk512-sw8-blk256", 2000, 100, "knn", 32, 512, dict(itopk_size=512, search_width=8, thread_block_size=256)),
    ("d129-k=itopk32-team32-nrs2", 2000, 129, "rand", 24, 32, dict(itopk_size=32, team_size=32, num_random_samplings=2)),
    ("d257-seed0-fill0.1", 2000, 257, "knn", 24, 10, dict(seed=0, hashmap_max_fill_rate=0.1)),
    ("d1000-blk128-bitlen15", 1000, 1000, "rand", 24, 10, dict(thread_block_size=128, hashmap_min_bitlen=15, hashmap_max_fill_rate=0.9)),
    ("deg1-maxit1-minit7", 2000, 16, "rand", 1, 10, dict(max_iterations=1, min_iterations=7)),
    ("deg3-maxit5-minit300", 2000, 16, "rand", 3, 10, dict(max_iterations=5, min_iterations=300)),
    ("deg128-itopk512-nrs2", 2000, 16, "rand", 128, 100, dict(itopk_size=512, num_random_samplings=2)),
    ("gather4096-nrs2-fill0.9", 20000, 16, "rand", 128, 10, dict(search_width=32, num_random_samplings=2, hashmap_max_fill_rate=0.9)),
    ("disconnected-k32", 600, 8, "disc", 4, 32, dict(itopk_size=32, search_width=1)),
    ("disconnected-k=itopk96-nrs2", 600, 8, "disc", 8, 96, dict(itopk_size=96, num_random_samplings=2)),
    ("n1", 1, 8, "rand", 3, 10, dict(itopk_size=32)),
    ("n20<numInit", 20, 8, "rand", 24, 20, dict(itopk_size=33, num_random_samplings=2)),
]


@pytest.mark.parametrize("ip", [False, True], ids=["L2", "IP"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_search_replays_model_bit_exact(res, case, ip):
    _, n, d, kind, K, k, params = case
    rs = np.random.RandomState(n + 7 * d + K)
    xb = _int_data(rs, n, d)
    xq = _int_data(rs, NQ, d)
    graph = _graph(kind, xb, K, ip, n + K)
    index = _index(res, xb, graph, ip)
    D, I = index.search(xq, k, params=fb.SearchParametersCagra(**params))
    Dm, Im, count = oc.search_single_cta(xb, graph, xq, k, params, metric_ip=ip)
    np.testing.assert_array_equal(I, Im)
    np.testing.assert_array_equal(D, Dm)  # by value: -0.0 == 0.0
    assert index.lastSearchDistanceCount() == count
    if kind == "disc" or n < k:
        assert (I == -1).any()  # fewer reachable nodes than k: -1 / +-FLT_MAX tails
        assert np.all(D[I == -1] == (-oc.FLT_MAX if ip else oc.FLT_MAX))


def test_search_splits_replay_model(res):
    import torch

    rs = np.random.RandomState(11)
    d, n, nq, k = 64, 3000, 100, 10
    xb = _int_data(rs, n, d)
    xq = _int_data(rs, nq, d)
    graph = _graph("rand", xb, 24, False, 3)
    params = dict(itopk_size=64, seed=12345)
    Dm, Im, count = oc.search_single_cta(xb, graph, xq, k, params)  # each query at its row of the whole call
    index = _index(res, xb, graph, False)

    def check(D, I):
        np.testing.assert_array_equal(I, Im)
        np.testing.assert_array_equal(D, Dm)
        assert index.lastSearchDistanceCount() == count  # the total over the call

    check(*index.search(xq, k, params=fb.SearchParametersCagra(max_queries=37, **params)))
    Dd, Id = index.search(torch.from_numpy(xq).cuda(), k, params=fb.SearchParametersCagra(**params))
    torch.cuda.synchronize()
    check(Dd.cpu().numpy(), Id.cpu().numpy())
    # host queries paged through two pinned buffers of 16 queries each
    r2 = fb.StandardGpuResources()
    r2.setPinnedMemory(2 * 16 * d * 4)
    index = cloner.gpu_cagra_from_payload(r2, cloner.cagra_payload(index))
    index.setMinPagingSize(0)
    check(*index.search(xq, k, params=fb.SearchParametersCagra(**params)))
    check(*index.search(xq, k, params=fb.SearchParametersCagra(max_queries=7, **params)))


# both sides of every plan limit: shared memory, 2^16 visited-set slots, search_width * K <= 4096, samples <= 8192
LIMIT_CASES = [
    (16, 128, 10, dict(search_width=32, hashmap_max_fill_rate=0.9)),
    (16, 128, 10, dict(search_width=32)),  # b = 16: 295616 bytes of shared memory
    (16, 128, 10, dict(search_width=32, hashmap_max_fill_rate=0.2)),  # b = 17
    (16, 128, 10, dict(search_width=33, hashmap_max_fill_rate=0.9)),
    (16, 128, 10, dict(search_width=16, num_random_samplings=4)),  # 8192 samples
    (16, 128, 10, dict(search_width=16, num_random_samplings=5)),
    (16, 128, 10, dict(hashmap_min_bitlen=15)),
    (16, 128, 10, dict(hashmap_min_bitlen=16)),  # 2^16 slots never fit shared memory
    (16, 128, 10, dict(itopk_size=512, search_width=24, hashmap_max_fill_rate=0.9)),
    (16, 128, 10, dict(itopk_size=512, search_width=32, hashmap_max_fill_rate=0.9)),
    (16, 128, 512, dict(itopk_size=512)),
    (16, 128, 513, dict(itopk_size=513)),
    (16, 128, 33, dict(itopk_size=32)),
]


def test_plan_limits_throw_exactly_where_the_model_says(res):
    rs = np.random.RandomState(2)
    n, d, K = 3000, 16, 128
    xb = _int_data(rs, n, d)
    xq = _int_data(rs, 4, d)
    index = _index(res, xb, _random_graph(rs, n, K), False)
    D0, I0 = index.search(xq, 10)
    thrown = 0
    for d_, K_, k, params in LIMIT_CASES:
        plan = oc.search_plan(n, d_, K_, k, params)
        if plan["error"]:
            thrown += 1
            with pytest.raises(fb.FaissError, match=plan["error"].replace("*", r"\*").replace("^", r"\^")):
                index.search(xq, k, params=fb.SearchParametersCagra(**params))
            D, I = index.search(xq, 10)
            assert D.tobytes() == D0.tobytes() and I.tobytes() == I0.tobytes()
        else:
            index.search(xq, k, params=fb.SearchParametersCagra(**params))
    assert 0 < thrown < len(LIMIT_CASES)


def _team(d, params):
    return params.get("team_size") or min(32, max(4, 1 << max(0, (d + 15) // 16 - 1).bit_length()))


FLOAT_CASES = [c for c in CASES if c[0] not in ("n1",)] + [
    ("d2048-knn", 1000, 2048, "rand", 24, 10, {}),
    ("d2048-team4", 1000, 2048, "rand", 24, 10, dict(team_size=4, itopk_size=128)),
]


@pytest.mark.parametrize("ip", [False, True], ids=["L2", "IP"])
@pytest.mark.parametrize("case", FLOAT_CASES, ids=[c[0] for c in FLOAT_CASES])
def test_search_fp32_results_are_valid_and_accurate(res, case, ip):
    _, n, d, kind, K, k, params = case
    rs = np.random.RandomState(n + 3 * d + K)
    xb = rs.randn(n, d).astype(np.float32)
    xq = rs.randn(NQ, d).astype(np.float32)
    graph = _graph(kind, xb, K, ip, n + K)
    index = _index(res, xb, graph, ip)
    D, I = index.search(xq, k, params=fb.SearchParametersCagra(**params))
    team = _team(d, params)
    # a lane's fma chain is at most ceil(d / team) + 3 terms long (float4 loads round its share up to 4), then
    # log2(team) shuffle additions; L2's x - y adds one rounding to each squared term
    m = -(-d // team) + 3 + int(np.log2(team)) + (0 if ip else 2)
    gamma = m * U32 / (1 - m * U32)
    x64, q64 = xb.astype(np.float64), xq.astype(np.float64)
    for r in range(NQ):
        ids = I[r]
        valid = ids >= 0
        nv = int(valid.sum())
        assert valid[:nv].all(), "row %d: -1 before a valid id: %s" % (r, ids)
        got = ids[:nv]
        assert len(set(got.tolist())) == nv and (got < n).all()
        dr = D[r, :nv].astype(np.float64)
        assert np.all(np.diff(dr) <= 0) if ip else np.all(np.diff(dr) >= 0), "row %d: D not sorted" % r
        assert np.all(D[r, nv:] == (-oc.FLT_MAX if ip else oc.FLT_MAX))
        terms = x64[got] * q64[r] if ip else (x64[got] - q64[r]) ** 2
        exact = terms.sum(1)
        bound = gamma * np.abs(terms).sum(1)
        err = np.abs(dr - exact)
        assert np.all(err <= bound), "row %d: error %g > bound %g" % (r, (err - bound).max(), bound[np.argmax(err - bound)])


# ---------------------------------------------------------------------------------------------------------------------
# The build against the oracle, end to end


def _build(res, x, ip, K0, K, pq_bits=8, refine_rate=2.4, batch=7, n_probes=1024):
    cfg = fb.GpuIndexCagraConfig()
    cfg.intermediate_graph_degree = K0
    cfg.graph_degree = K
    cfg.refine_rate = refine_rate
    bp = fb.IVFPQBuildCagraConfig()
    bp.pq_bits = pq_bits
    bp.kmeans_trainset_fraction = 0.5
    cfg.ivf_pq_params = bp
    sp = fb.IVFPQSearchCagraConfig()
    sp.n_probes = n_probes
    sp.max_internal_batch_size = batch
    cfg.ivf_pq_search_params = sp
    index = fb.GpuIndexCagra(res, x.shape[1], fb.METRIC_INNER_PRODUCT if ip else fb.METRIC_L2, cfg)
    index.train(x)
    return index


BUILD_CASES = [
    # (a) IVF-PQ candidates that cover every row: C = ceil(2.4 * K0) + 1 >= N, every list probed.  N = 300 at f = 0.5:
    # 150 training rows (>= 2^6), 3 lists, C = 309; pq_bits 8 needs 256 training rows: N = 600, K0 = 256, C = 616,
    # 7 lists.  7 rows per refine page: pages start at rows 7, 14, ...
    ("ivfpq4", 300, 128, 64, 4),
    ("ivfpq5", 300, 128, 33, 5),
    ("ivfpq6", 300, 128, 17, 6),
    ("ivfpq8", 600, 256, 64, 8),
    # (b) fewer than 2^pq_bits training rows: every row takes the exact Flat fallback
    ("fallback6", 100, 40, 20, 6),
    ("fallback8", 300, 64, 31, 8),
    # (c) the clamps: K0 = N - 1, K = min(graph_degree, K0)
    ("clamp-n2", 2, 128, 64, 8),
    ("clamp-n3", 3, 128, 64, 8),
    ("clamp-n50", 50, 128, 64, 8),
]


@pytest.mark.parametrize("ip", [False, True], ids=["L2", "IP"])
@pytest.mark.parametrize("case", BUILD_CASES, ids=[c[0] for c in BUILD_CASES])
def test_build_matches_exact_knn_then_optimize(res, case, ip):
    _, n, K0, K, pq_bits = case
    rs = np.random.RandomState(n + K0 + pq_bits)
    x = _int_data(rs, n, 16)
    index = _build(res, x, ip, K0, K, pq_bits=pq_bits)
    K0c = min(K0, n - 1)
    Kc = min(K, K0c)
    assert index.graph_degree == Kc
    np.testing.assert_array_equal(index.get_knngraph(), oc.optimize(oc.exact_knn_graph(x, K0c, ip), Kc))


# ---------------------------------------------------------------------------------------------------------------------
# cagra_optimize against the oracle


def _random_g0(rs, N, K0):
    """distinct ids other than the row's own: u + 1 + distinct offsets in [0, N - 1), mod N"""
    off = np.empty((N, K0), np.int64)
    for u in range(N):
        while True:
            o = rs.randint(0, N - 1, K0) if K0 * 8 < N else rs.permutation(N - 1)[:K0]
            if len(np.unique(o)) == K0:
                break
        off[u] = o
    return (np.arange(N)[:, None] + 1 + off) % N


def _star_g0(rs, N, K0):
    """every row but 0 starts with 0, so R[0] holds N - 1 rows, far more than K"""
    g = _random_g0(rs, N, K0)
    for u in range(1, N):
        row = [0] + [v for v in g[u].tolist() if v != 0]
        g[u] = row[:K0]
    return g


OPT_CASES = [
    (40, 1, 1, "rand"),
    (40, 2, 1, "rand"),
    (500, 31, 7, "rand"),
    (500, 31, 7, "knn"),
    (500, 33, 33, "knn"),
    (800, 100, 51, "rand"),
    (800, 100, 51, "star"),
    (1000, 256, 128, "knn"),
    (1100, 1024, 64, "rand"),
    (1100, 1024, 1024, "knn"),
    (4096, 32, 16, "rand"),
    (4096, 64, 63, "star"),
    (70000, 16, 8, "rand"),
]


@pytest.mark.parametrize("N,K0,K,kind", OPT_CASES, ids=["%d-%d-%d-%s" % c for c in OPT_CASES])
def test_optimize_matches_oracle_shapes(res, N, K0, K, kind):
    rs = np.random.RandomState(N + K0 + K)
    if kind == "knn":
        G0 = oc.exact_knn_graph(_int_data(rs, N, 8), K0)
    elif kind == "star":
        G0 = _star_g0(rs, N, K0)
    else:
        G0 = _random_g0(rs, N, K0)
    np.testing.assert_array_equal(fb.cagra_optimize(res, G0, K), oc.optimize(G0, K))


@pytest.mark.parametrize("bad,msg", [("minus_one", ">= n"), ("out_of_range", ">= n"), ("self", "own id")])
def test_optimize_rejects_bad_g0_before_writing(res, bad, msg):
    import torch

    rs = np.random.RandomState(9)
    N, K0, K = 300, 16, 8
    G0 = _random_g0(rs, N, K0)
    G0[17, 5] = {"minus_one": -1, "out_of_range": N, "self": 17}[bad]
    g0 = torch.from_numpy(G0).to(device="cuda", dtype=torch.int32).contiguous()
    G = torch.full((N, K), 12345, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    rc = fb.lib.b200_cagra_optimize(res._h, 0, ctypes.c_void_p(g0.data_ptr()), ctypes.c_int64(N), K0, K,
                                    ctypes.c_void_p(G.data_ptr()))
    with pytest.raises(fb.FaissError, match=msg):
        fb.check(rc)
    res.syncDefaultStream(0)
    assert bool((G == 12345).all())
    with pytest.raises(fb.FaissError, match=msg):
        fb.cagra_optimize(res, G0, K)
