"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the GpuIndexCagra graph optimisation (DESIGN "GpuIndexCagra",
faiss_b200/csrc/cagra_build.cu), and the tie-aware k-NN comparison the CAGRA tests use.

    detours  c[u][j] = #{ i < j : some p < j has G0[G0[u][i]][p] = G0[u][j] }
    prune    P[u] = the K entries of G0[u] with the smallest (c, j), in that order
    reverse  R[w] = every u with w in P[u], ordered by (position of w in P[u], u)
    merge    G[u] = P[u][0:K/2], then the entries of R[u] not present yet, then the rest of P[u], cut to K
"""
import numpy as np


def detour_counts(G0):
    """c [N, K0] int64"""
    G0 = np.asarray(G0, dtype=np.int64)
    N, K0 = G0.shape
    c = np.zeros((N, K0), np.int64)
    rank = np.full(N, -1, np.int64)
    i_idx = np.arange(K0)[:, None]
    p_idx = np.arange(K0)[None, :]
    for u in range(N):
        row = G0[u]
        rank[row] = np.arange(K0)
        J = rank[G0[row]]  # J[i, p] = rank in G0[u] of G0[G0[u][i]][p], or -1
        ok = (J > i_idx) & (J > p_idx)
        hit = np.zeros((K0, K0), bool)  # hit[j, i]
        hit[J[ok], np.broadcast_to(i_idx, J.shape)[ok]] = True
        c[u] = hit.sum(axis=1)
        rank[row] = -1
    return c


def prune(G0, K):
    G0 = np.asarray(G0, dtype=np.int64)
    c = detour_counts(G0)
    N, K0 = G0.shape
    P = np.empty((N, K), np.int64)
    j = np.arange(K0)
    for u in range(N):
        order = np.lexsort((j, c[u]))  # by c, then by position
        P[u] = G0[u][order[:K]]
    return P


def reverse_edges(P):
    """R[w] = [u, ...] in (position of w in P[u], u) order"""
    N, K = P.shape
    R = [[] for _ in range(N)]
    for pos in range(K):
        for u in range(N):
            R[int(P[u, pos])].append(u)
    return R


def merge(P, R):
    N, K = P.shape
    half = K // 2
    G = np.empty((N, K), np.int64)
    for u in range(N):
        out = [int(x) for x in P[u, :half]]
        seen = set(out)
        for v in list(R[u]) + [int(x) for x in P[u, half:]]:
            if len(out) == K:
                break
            if v not in seen:
                out.append(v)
                seen.add(v)
        G[u] = out
    return G


def optimize(G0, K):
    """G0 [N, K0] (distinct ids per row, no self edges) -> G [N, K] int64"""
    P = prune(G0, K)
    return merge(P, reverse_edges(P))


def exact_knn_graph(x, K0, metric_ip=False):
    """G0 of the exact kNN of every row (self excluded), ordered by (distance, id); IP ranks larger first"""
    x = np.asarray(x, dtype=np.float64)
    if metric_ip:
        key = -(x @ x.T)
    else:
        sq = (x * x).sum(1)
        key = sq[:, None] + sq[None, :] - 2 * (x @ x.T)
    np.fill_diagonal(key, np.inf)
    N = x.shape[0]
    G0 = np.empty((N, K0), np.int64)
    ids = np.arange(N)
    for u in range(N):
        order = np.lexsort((ids, key[u]))
        G0[u] = order[:K0]
    return G0


def check_knn_with_ties(Dref, Iref, Dnew, Inew, rtol=1e-5):
    """Dnew equals Dref to rtol; per row the ids agree, except that ids whose distances tie (within rtol of the row's
    largest distance) may come in any order, and the last group of tied distances may be cut anywhere.  Raises
    AssertionError with the first offending row."""
    np.testing.assert_allclose(Dnew, Dref, rtol=rtol)
    for i in range(Iref.shape[0]):
        if np.array_equal(Iref[i], Inew[i]):
            continue
        tol = rtol * np.abs(Dref[i]).max()
        # group positions into runs of distances within tol of the run's first distance
        groups = np.zeros(Dref.shape[1], np.int64)
        g, start = 0, Dref[i, 0]
        for j in range(1, Dref.shape[1]):
            if abs(Dref[i, j] - start) > tol:
                g += 1
                start = Dref[i, j]
            groups[j] = g
        for gi in range(groups[-1]):  # every group but the last
            m = groups == gi
            assert set(Iref[i, m].tolist()) == set(Inew[i, m].tolist()), (
                "row %d: ids %s vs %s at distances %s" % (i, Iref[i, m], Inew[i, m], Dref[i, m])
            )
