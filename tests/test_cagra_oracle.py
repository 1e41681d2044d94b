"""The numpy restatement of GpuIndexCagra (oracle/oracle_cagra_np.py).  The graph optimisation: hand-worked graphs,
invariants on random inputs, and a round trip through the reference's IndexHNSWCagra (where oracle/_ref was built).
The search model: hand-worked walks, the refill schedule, and the host plan's values and limits."""
import numpy as np
import pytest

from oracle import oracle_cagra_np as oc

# N = 4, K0 = 3.  Row 0 = [1, 2, 3]: 2 is reached from 1 through G0[1][0] = 2 (i = 0, p = 0 < j = 1) and 3 from 2
# through G0[2][0] = 3 (i = 1, p = 0 < j = 2), while G0[1][2] = 3 does not count (p = 2 is not < j = 2)
G0_SMALL = np.array([[1, 2, 3], [2, 0, 3], [3, 0, 1], [0, 1, 2]])


def test_detour_counts_hand_worked():
    np.testing.assert_array_equal(oc.detour_counts(G0_SMALL), [[0, 1, 1], [0, 0, 1], [0, 1, 2], [0, 1, 2]])


def test_prune_breaks_count_ties_by_position():
    # row 0 counts [0, 1, 1]: the tie between positions 1 and 2 keeps position 1
    np.testing.assert_array_equal(oc.prune(G0_SMALL, 2), [[1, 2], [2, 0], [3, 0], [0, 1]])


def test_reverse_edges_order_by_position_then_row():
    P = oc.prune(G0_SMALL, 2)
    assert oc.reverse_edges(P) == [[3, 1, 2], [0, 3], [1, 0], [2]]


def test_optimize_reverse_edge_overflow():
    # K = 2: one forward edge, then one slot for R[u]; R[0] = [3, 1, 2] overflows after 3
    np.testing.assert_array_equal(oc.optimize(G0_SMALL, 2), [[1, 3], [2, 0], [3, 1], [0, 2]])


def test_optimize_skips_reverse_edges_already_kept():
    # K = 3: P = G0 order by (count, position); R[0] = [3, 1, 2] gives 3, skips 1 (kept), then 2
    np.testing.assert_array_equal(oc.optimize(G0_SMALL, 3), [[1, 3, 2], [2, 0, 3], [3, 1, 0], [0, 2, 1]])


def test_optimize_fills_from_pruned_list_when_reverse_edges_run_out():
    # a star: every row's first neighbour is 0, so only row 0 has reverse edges
    N, K0 = 6, 4
    G0 = np.array([[1, 2, 3, 4]] + [[0] + [v for v in range(1, N) if v != u][:K0 - 1] for u in range(1, N)])
    G = oc.optimize(G0, 4)
    P = oc.prune(G0, 4)
    R = oc.reverse_edges(P)
    for u in range(1, N):
        new_r = [v for v in R[u] if v not in P[u, :2]][:2]
        expect = list(P[u, :2]) + new_r
        expect += [v for v in P[u, 2:] if v not in expect][: 4 - len(expect)]
        np.testing.assert_array_equal(G[u], expect)


def _random_g0(rs, N, K0):
    G0 = np.empty((N, K0), np.int64)
    for u in range(N):
        c = rs.choice(N - 1, K0, replace=False)
        G0[u] = c + (c >= u)  # no self edge, no duplicate
    return G0


@pytest.mark.parametrize("N,K0,K", [(50, 8, 4), (200, 16, 8), (300, 32, 32), (120, 12, 5)])
def test_optimize_invariants_random(N, K0, K):
    rs = np.random.RandomState(N + K0)
    G0 = _random_g0(rs, N, K0)
    G = oc.optimize(G0, K)
    P = oc.prune(G0, K)
    R = oc.reverse_edges(P)
    assert G.shape == (N, K)
    for u in range(N):
        row = G[u].tolist()
        assert u not in row
        assert len(set(row)) == K
        assert set(row) <= set(G0[u].tolist()) | set(R[u])
        np.testing.assert_array_equal(G[u, : K // 2], P[u, : K // 2])


def test_exact_graph_round_trip_through_reference_hnsw_cagra(tmp_path):
    from oracle import ref_cagra

    if not ref_cagra.available():
        pytest.skip("oracle/_ref not built (needs /root/reference at build time)")
    from bench import synthetic_dataset

    _, xb, xq = synthetic_dataset(64, 0, 10000, 100)
    k = 12
    G = oc.optimize(oc.exact_knn_graph(xb, 64), 32)
    # efSearch = 256: at 64 the CPU base-level search itself misses about 11% of the top-12 on this data, with this
    # graph or with the exact kNN graph, so only a wide search tests the graph and the shim
    D, I = ref_cagra.search_graph(xb, G, 1, xq, k, ef_search=256, base_level_only=True)
    x = xb.astype(np.float64)
    q = xq.astype(np.float64)
    dist = (q * q).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2 * q @ x.T
    gI = np.argsort(dist, axis=1, kind="stable")[:, :k]
    gD = np.take_along_axis(dist, gI, 1).astype(np.float32)
    oc.check_knn_with_ties(gD, gI, D, I, rtol=1e-4)


# ---------------------------------------------------------------------------------------------------------------------
# The search model: search_plan and search_single_cta


def test_mix64_is_splitmix64():
    # splitmix64's first output from state 0
    assert oc.mix64(0) == 0xE220A8397B1DCDAF
    assert oc.mix64((1 << 64) - 1) < (1 << 64)


# a 6-node path 0 - 1 - ... - 5 on the line (d = 1, x[u] = u), -1 past the ends; the query sits on node 5
PATH_X = np.arange(6, dtype=np.float32)[:, None]
PATH_G = np.array([[u - 1 if u > 0 else -1, u + 1 if u < 5 else -1] for u in range(6)])
PATH_Q = np.array([[5.0]], np.float32)


def test_walk_hand_worked_path():
    # seed 7, row 0: both samples (numInit = search_width * K = 2) are node 0, so one distinct start and count 1.
    #   iteration 1: parent 0, gathers -1 (skipped) and 1 -> top (16, 1) (25, 0*)          count 2
    #   iteration 2: parent 1, gathers 0 (visited) and 2   -> (9, 2) ...                    count 3
    #   iterations 3, 4, 5: parents 2, 3, 4 reach 3, 4, 5                                  count 6
    #   iteration 6: parent 5 gathers 4 (visited) and -1; iteration 7 finds no parent and stops
    # (* expanded).  The visited set never refills: 2 + 6 * 2 insertions stay below hashLimit = 256.
    params = dict(itopk_size=32, seed=7)
    row_key = oc.mix64(7 ^ oc.mix64(0))
    assert [oc.mix64(row_key + i) % 6 for i in range(2)] == [0, 0]
    plan = oc.search_plan(6, 1, 2, 6, params)
    assert (plan["numInit"], plan["gather"], plan["hashLimit"]) == (2, 2, 256)
    D, I, count = oc.search_single_cta(PATH_X, PATH_G, PATH_Q, 6, params)
    np.testing.assert_array_equal(I, [[5, 4, 3, 2, 1, 0]])
    np.testing.assert_array_equal(D, [[0, 1, 4, 9, 16, 25]])
    assert count == 6
    # max_iterations = 3 stops after parents 0, 1, 2: nodes 0 - 3 found, the last two results missing
    D, I, count = oc.search_single_cta(PATH_X, PATH_G, PATH_Q, 6, dict(params, max_iterations=3))
    np.testing.assert_array_equal(I, [[3, 2, 1, 0, -1, -1]])
    np.testing.assert_array_equal(D, [[4, 9, 16, 25, oc.FLT_MAX, oc.FLT_MAX]])
    assert count == 4
    # inner product: keys -5u, so node 5 is best; D = +5u
    D, I, _ = oc.search_single_cta(PATH_X, PATH_G, PATH_Q, 6, params, metric_ip=True)
    np.testing.assert_array_equal(I, [[5, 4, 3, 2, 1, 0]])
    np.testing.assert_array_equal(D, [[25, 20, 15, 10, 5, 0]])
    D, I, _ = oc.search_single_cta(PATH_X, PATH_G, PATH_Q, 6, dict(params, max_iterations=1), metric_ip=True)
    np.testing.assert_array_equal(I[0, :2], [1, 0])
    np.testing.assert_array_equal(D[0, 2:], [-oc.FLT_MAX] * 4)


def test_walk_hand_worked_path_with_refill():
    # K = 8 (the path's two edges scattered among -1 slots) and 28 samplings: numInit = 224 covers all 6 nodes (count
    # 6).  need = max(224 + 32, 4 * (32 + 8)) = 256 gives b = 9 at fill 0.5, hashLimit 256.  Insertions count gather
    # slots: 232, 240, 248, 256 after iterations 1 - 4; iteration 5 would reach 264 > 256, so the visited set is refilled
    # from the top-k, which holds all 6 nodes: nothing is scored again, and the result is the path's.
    G = np.full((6, 8), -1)
    G[:, 2] = PATH_G[:, 0]
    G[:, 5] = PATH_G[:, 1]
    params = dict(itopk_size=32, seed=7, num_random_samplings=28)
    plan = oc.search_plan(6, 1, 8, 6, params)
    assert (plan["numInit"], plan["hashBits"], plan["hashLimit"]) == (224, 9, 256)
    D, I, count = oc.search_single_cta(PATH_X, G, PATH_Q, 6, params)
    np.testing.assert_array_equal(I, [[5, 4, 3, 2, 1, 0]])
    np.testing.assert_array_equal(D, [[0, 1, 4, 9, 16, 25]])
    assert count == 6


def test_refill_rescoring_counts_but_changes_nothing():
    # 3000 integer rows: the refill-heavy plan (fill 0.1) scores dropped ids again, the refill-free one (2^15 slots at
    # 0.9) never does; the results are the same bytes
    rs = np.random.RandomState(5)
    x = rs.randint(-8, 9, (3000, 8)).astype(np.float32)
    q = rs.randint(-8, 9, (8, 8)).astype(np.float32)
    G = rs.randint(0, 3000, (3000, 16))
    often = dict(itopk_size=64, hashmap_max_fill_rate=0.1)
    never = dict(itopk_size=64, hashmap_max_fill_rate=0.9, hashmap_min_bitlen=15)
    assert oc.search_plan(3000, 8, 16, 10, often)["hashLimit"] < oc.search_plan(3000, 8, 16, 10, never)["hashLimit"]
    D1, I1, c1 = oc.search_single_cta(x, G, q, 10, often)
    D2, I2, c2 = oc.search_single_cta(x, G, q, 10, never)
    np.testing.assert_array_equal(I1, I2)
    np.testing.assert_array_equal(D1, D2)
    assert c1 > c2


def test_walk_model_reaches_exact_top_k():
    rs = np.random.RandomState(0)
    x = rs.randint(-8, 9, (2000, 16)).astype(np.float32)
    q = rs.randint(-8, 9, (20, 16)).astype(np.float32)
    G = oc.optimize(oc.exact_knn_graph(x, 64), 32)
    D, I, _ = oc.search_single_cta(x, G, q, 10, dict(itopk_size=128))
    key = ((q[:, None, :].astype(np.int64) - x[None].astype(np.int64)) ** 2).sum(-1)
    gI = np.lexsort((np.broadcast_to(np.arange(2000), key.shape), key))[:, :10]
    np.testing.assert_array_equal(I, gI)
    np.testing.assert_array_equal(D, np.take_along_axis(key, gI, 1))


@pytest.mark.parametrize(
    "n,d,K,k,params,expect",
    [
        # defaults at d = 128, K = 64: need = max(64 + 64, 4 * 128) = 512, 2^10 * 0.5 = 512 -> b = 10;
        # 4 * 128 + 8 * 64 + 8 * 64 + 4 * (1024 + 1) = 5636
        (10000, 128, 64, 10, {}, dict(itopk=64, bufSize=64, candSize=64, hashBits=10, hashLimit=512, smem=5636,
                                      teamSize=8, blockSize=64, maxIterations=144)),
        # itopk 512: need 4 * 576 = 2304 -> b = 13; 512 + 4096 + 512 + 4 * (8192 + 1) = 37892
        (10000, 128, 64, 10, dict(itopk_size=512), dict(itopk=512, bufSize=512, hashBits=13, smem=37892,
                                                        blockSize=256, maxIterations=1040)),
        # 4096 gathers at fill 0.9 (0.899999976 as a float): need 4 * 4160 = 16640, 2^15 * 0.9f = 29491.2 -> b = 15;
        # 64 + 512 + 8 * 4096 + 4 * (32768 + 32) = 164544
        (10000, 16, 128, 10, dict(search_width=32, hashmap_max_fill_rate=0.9),
         dict(candSize=4096, hashBits=15, hashLimit=29491, smem=164544, teamSize=4, maxIterations=20)),
        # itopk_size 33 rounds to 64; 96 stays 96 in a buffer of 128; d = 1000 -> team 32 (next_pow2(63) = 64, clamped)
        (5000, 1000, 24, 33, dict(itopk_size=33), dict(itopk=64, bufSize=64, teamSize=32)),
        (5000, 257, 24, 10, dict(itopk_size=96), dict(itopk=96, bufSize=128, teamSize=32, blockSize=128)),
        (5000, 129, 24, 10, {}, dict(teamSize=16)),
        # max_iterations 5 with min_iterations 40: the larger wins; 0 with min 1000: the auto cap 2 * 64 / 3 + 16 = 58
        # is raised to 1000
        (5000, 16, 24, 10, dict(max_iterations=5, min_iterations=40), dict(maxIterations=40)),
        (5000, 16, 24, 10, dict(search_width=3, min_iterations=1000), dict(maxIterations=1000)),
        (5000, 16, 24, 10, dict(search_width=3), dict(maxIterations=58)),
        # 2 samplings x 4096 gathers = 8192 samples: need 8192 + 64 -> b = 14 at 0.9 (2^14 * 0.9f = 14745.6 < 16640 ->
        # b = 15)
        (10000, 16, 128, 10, dict(search_width=32, num_random_samplings=2, hashmap_max_fill_rate=0.9),
         dict(numInit=8192, candSize=8192, hashBits=15, smem=64 + 512 + 65536 + 4 * (32768 + 32))),
        (10000, 16, 24, 10, dict(hashmap_min_bitlen=15, hashmap_max_fill_rate=0.9), dict(hashBits=15, hashLimit=29491)),
    ],
)
def test_search_plan_values(n, d, K, k, params, expect):
    plan = oc.search_plan(n, d, K, k, params)
    assert plan["error"] is None
    for key, v in expect.items():
        assert plan[key] == v, (key, plan[key], v)


@pytest.mark.parametrize(
    "d,K,k,params,msg",
    [
        (16, 128, 10, dict(search_width=32), "shared memory"),  # fill 0.5: b = 16, 295616 bytes
        (16, 128, 10, dict(search_width=32, hashmap_max_fill_rate=0.1), "2^18"),
        (16, 128, 10, dict(search_width=33), "4224 > 4096"),
        (16, 128, 10, dict(search_width=16, num_random_samplings=5), "10240 > 8192"),
        (16, 24, 10, dict(itopk_size=513), "513 > 512"),
        (16, 24, 40, dict(itopk_size=32), "k 40 > itopk_size 32"),
        (16, 24, 10, dict(team_size=2), "team_size"),
        (16, 24, 10, dict(thread_block_size=32), "thread_block_size"),
        (16, 24, 10, dict(hashmap_max_fill_rate=0.95), "fill_rate"),
        (16, 24, 10, dict(hashmap_min_bitlen=17), "min_bitlen"),
        (16, 24, 10, dict(search_width=0), "search_width"),
        (16, 24, 10, dict(num_random_samplings=0), "num_random_samplings"),
    ],
)
def test_search_plan_limits(d, K, k, params, msg):
    err = oc.search_plan(10000, d, K, k, params)["error"]
    assert err is not None and msg in err, err
