"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the GpuIndexCagra graph optimisation (DESIGN "GpuIndexCagra",
faiss_b200/csrc/cagra_build.cu), of its single-CTA search (faiss_b200/csrc/cagra_search.cu: search_plan,
search_single_cta), and the tie-aware k-NN comparison the CAGRA tests use.

    detours  c[u][j] = #{ i < j : some p < j has G0[G0[u][i]][p] = G0[u][j] }
    prune    P[u] = the K entries of G0[u] with the smallest (c, j), in that order
    reverse  R[w] = every u with w in P[u], ordered by (position of w in P[u], u)
    merge    G[u] = P[u][0:K/2], then the entries of R[u] not present yet, then the rest of P[u], cut to K
"""
import bisect

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


# ---------------------------------------------------------------------------------------------------------------------
# The single-CTA search (GpuIndexCagra::searchImpl_ in index.cu, cagra_search_kernel in cagra_search.cu; DESIGN §3.10)

# SearchParametersCagra's defaults (faiss_b200/csrc/index.h)
SEARCH_DEFAULTS = dict(
    max_queries=0, itopk_size=64, max_iterations=0, team_size=0, search_width=1, min_iterations=0,
    thread_block_size=0, hashmap_min_bitlen=0, hashmap_max_fill_rate=0.5, num_random_samplings=1, seed=0x128394,
)
SMEM_LIMIT = 227 * 1024
FLT_MAX = float(np.finfo(np.float32).max)
_M64 = (1 << 64) - 1


def _next_pow2(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def _round_up(x, m):
    return (x + m - 1) // m * m


def mix64(x):
    """the splitmix64 finaliser of cagra_search.cu, on Python ints masked to 64 bits"""
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def search_plan(n, d, K, k, params=None):
    """The host plan of one search: a dict with itopk, bufSize, candSize, numInit, maxIterations, teamSize, blockSize,
    hashBits, hashLimit, smem (dynamic shared-memory bytes) and error (None, or the text of the exception the search
    throws; once a limit throws, the fields after it are left out)."""
    p = dict(SEARCH_DEFAULTS, **(params or {}))
    plan = dict(error=None)

    def fail(msg):
        plan["error"] = msg
        return plan

    if p["itopk_size"] > 512:
        return fail("itopk_size %d > 512" % p["itopk_size"])
    if k > p["itopk_size"]:
        return fail("k %d > itopk_size %d" % (k, p["itopk_size"]))
    if p["search_width"] < 1:
        return fail("search_width must be >= 1")
    if p["num_random_samplings"] < 1:
        return fail("num_random_samplings must be >= 1")
    if p["team_size"] not in (0, 4, 8, 16, 32):
        return fail("team_size must be 0, 4, 8, 16 or 32")
    if p["thread_block_size"] not in (0, 64, 128, 256, 512, 1024):
        return fail("thread_block_size must be 0, 64, 128, 256, 512 or 1024")
    fill = float(np.float32(p["hashmap_max_fill_rate"]))  # a C++ float, widened to double where it is used
    if not (np.float32(0.1) <= fill <= np.float32(0.9)):
        return fail("hashmap_max_fill_rate must be in [0.1, 0.9]")
    if p["hashmap_min_bitlen"] > 16:
        return fail("hashmap_min_bitlen must be <= 16")
    itopk = _round_up(max(p["itopk_size"], 1), 32)
    sw = p["search_width"]
    gather = sw * K
    num_init = p["num_random_samplings"] * gather
    plan.update(itopk=itopk, bufSize=_next_pow2(itopk), searchWidth=sw, gather=gather)
    if gather > 4096:
        return fail("search_width * graph_degree = %d > 4096" % gather)
    if num_init > 8192:
        return fail("num_random_samplings * search_width * graph_degree = %d > 8192" % num_init)
    plan.update(numInit=num_init, candSize=_next_pow2(max(num_init, gather)))
    auto_iter = 2 * itopk // sw + 16
    plan["maxIterations"] = min(max(p["max_iterations"] or auto_iter, p["min_iterations"]), 1 << 20)
    plan["teamSize"] = p["team_size"] or min(32, max(4, _next_pow2((d + 15) // 16)))
    plan["blockSize"] = p["thread_block_size"] or (64 if itopk <= 64 else 128 if itopk <= 256 else 256)
    need = max(float(num_init + itopk), 4.0 * (itopk + gather))
    bits = max(8, p["hashmap_min_bitlen"])
    while float(1 << bits) * fill < need:
        bits += 1
    if bits > 16:
        return fail("the visited set would need 2^%d entries" % bits)
    plan.update(hashBits=bits, hashLimit=int(float(1 << bits) * fill))
    plan["smem"] = 4 * _round_up(d, 4) + 8 * plan["bufSize"] + 8 * plan["candSize"] + 4 * ((1 << bits) + sw)
    if plan["smem"] > SMEM_LIMIT:
        return fail("the search does not fit shared memory")
    return plan


def search_single_cta(xb, graph, xq, k, params=None, metric_ip=False, row0=0):
    """The search of every query row, restated step by step: -> (D [nq, k] float32, I [nq, k] int64, distance count).
    graph [n, K] int64 with -1 for no edge.  Query r is row row0 + r of its call (the entry points depend on it).
    Distances are exact int64 when xb and xq hold integers, float64 otherwise."""
    xb = np.asarray(xb)
    xq = np.asarray(xq)
    n, d = xb.shape
    graph = np.asarray(graph, dtype=np.int64)
    K = graph.shape[1]
    plan = search_plan(n, d, K, k, params)
    if plan["error"]:
        raise ValueError(plan["error"])
    p = dict(SEARCH_DEFAULTS, **(params or {}))
    itopk, sw, num_init = plan["itopk"], plan["searchWidth"], plan["numInit"]
    n_gather, hash_limit = plan["gather"], plan["hashLimit"]
    integer = np.array_equal(xb, np.round(xb)) and np.array_equal(xq, np.round(xq))
    X = xb.astype(np.int64 if integer else np.float64)
    Q = xq.astype(np.int64 if integer else np.float64)
    conv = int if integer else float
    # entries >= n stand for -1 (the kernel reads the graph as uint32)
    rows = [[int(v) for v in g if 0 <= v < n] for g in graph]
    seed = int(p["seed"]) & _M64
    D = np.empty((len(xq), k), np.float32)
    I = np.empty((len(xq), k), np.int64)
    count = 0

    for r in range(len(xq)):
        q = Q[r]

        def score(ids):
            y = X[ids]
            key = -(y @ q) if metric_ip else ((y - q) ** 2).sum(1)
            return [(conv(a), b) for a, b in zip(key.tolist(), ids)]

        # start: the distinct samples, best itopk by (key, id)
        row_key = mix64(seed ^ mix64((row0 + r) & _M64))
        visited = set()
        fresh = []
        for i in range(num_init):
            v = mix64((row_key + i) & _M64) % n
            if v not in visited:
                visited.add(v)
                fresh.append(v)
        count += len(fresh)
        top = sorted(score(fresh))[:itopk]
        expanded = set()
        first_open = 0  # every entry before it is expanded
        inserted = num_init
        for _ in range(plan["maxIterations"]):
            parents = []
            pos = first_open
            while pos < len(top) and len(parents) < sw:
                v = top[pos][1]
                if v not in expanded:
                    parents.append(v)
                    expanded.add(v)
                pos += 1
            first_open = pos
            if not parents:
                break
            if inserted + n_gather > hash_limit:  # the refill: the visited set becomes the ids in the top-k
                visited = {v for _, v in top}
                inserted = itopk
            inserted += n_gather
            fresh = []
            for u in parents:
                for v in rows[u]:
                    if v not in visited:
                        visited.add(v)
                        fresh.append(v)
            count += len(fresh)
            for e in sorted(score(fresh)):
                if len(top) == itopk and e >= top[-1]:
                    break  # the rest are worse still
                at = bisect.bisect_left(top, e)
                top.insert(at, e)
                first_open = min(first_open, at)
                if len(top) > itopk:
                    expanded.discard(top.pop()[1])
                    first_open = min(first_open, len(top))
        for j in range(k):
            if j < len(top):
                key, v = top[j]
                D[r, j] = -key if metric_ip else key
                I[r, j] = v
            else:
                D[r, j] = -FLT_MAX if metric_ip else FLT_MAX
                I[r, j] = -1
    return D, I, count
