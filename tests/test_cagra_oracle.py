"""The numpy restatement of the GpuIndexCagra graph optimisation (oracle/oracle_cagra_np.py): hand-worked graphs,
invariants on random inputs, and a round trip through the reference's IndexHNSWCagra (where oracle/_ref was built)."""
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
