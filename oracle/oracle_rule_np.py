"""TEST INFRASTRUCTURE ONLY -- numpy model of the reference's result rule, and data whose expected answer does not
depend on summation order.

The rule (faiss/impl/ResultHandler.h:275-282 against the neutral elements of faiss/utils/ordered_key_value.h): a
candidate is a result only if its distance is strictly better than the heap's neutral element -- dis < FLT_MAX for
L2, dis > -FLT_MAX for inner product; NaN never qualifies.  Results are ordered by (key, id) and the list is padded
with (FLT_MAX, -1) (-FLT_MAX for inner product).  The IVF coarse quantiser applies the same rule when it assigns a
vector at add time, so a vector without a result is not stored (faiss/IndexIVFFlat.cpp:122).  A stored id of -1 is
the one id the reference does not return: heap_reorder takes it for an empty slot after the selection.

Every distance the generators below produce is exact in fp32 whatever the summation order: small integers, or a sum
with exactly one coordinate that is non-finite or whose square overflows, or exactly FLT_MAX (a row (A, B) against a
query that is zero there: A*A rounds to one ulp below FLT_MAX, B*B is that ulp, and the remaining terms are far below
half an ulp).  So the model computes the distances in fp32 numpy and must equal every kernel bit for bit.

Only tests/ import this module.
"""
import numpy as np

METRIC_INNER_PRODUCT = 0
METRIC_L2 = 1

FLT_MAX = np.float32(np.finfo(np.float32).max)
HUGE = np.float32(1e20)  # squared, it overflows fp32 whatever the order of the sum
FMAX_A = np.float32(1.8446743e19)  # A*A rounds to FLT_MAX - ulp
FMAX_B = np.float32(2.0**52)  # B*B == ulp(FLT_MAX) == 2^104


def distances(xq, xb, metric):
    """[nq, n] fp32 distances; exact for the data of this module"""
    xq = np.asarray(xq, np.float32)
    xb = np.asarray(xb, np.float32)
    out = np.empty((xq.shape[0], xb.shape[0]), np.float32)
    with np.errstate(all="ignore"):
        for q in range(xq.shape[0]):
            t = xq[q] - xb if metric == METRIC_L2 else xq[q] * xb
            out[q] = (t * t if metric == METRIC_L2 else t).sum(axis=1, dtype=np.float32)
    return out


def keys_of(dis, metric):
    """key space: smaller is better"""
    with np.errstate(all="ignore"):
        return dis if metric == METRIC_L2 else -dis


def is_result(dis, metric):
    """the reference rule: strictly better than the neutral element; NaN fails both comparisons"""
    with np.errstate(all="ignore"):
        return keys_of(np.asarray(dis, np.float32), metric) < FLT_MAX


def select(dis, ids, k, metric):
    """one query's candidates (dis [m], ids [m]) -> (D [k], I [k]): results only, ordered by (key, id), padded"""
    dis = np.asarray(dis, np.float32)
    ids = np.asarray(ids, np.int64)
    ok = is_result(dis, metric)
    d, i = dis[ok], ids[ok]
    order = np.lexsort((i, keys_of(d, metric)))[:k]
    # a stored id of -1 takes its rank in the selection, then heap_reorder drops it as an empty slot and the results
    # behind it move up (faiss/utils/Heap.h:427-456)
    order = order[i[order] != -1]
    D = np.full(k, FLT_MAX if metric == METRIC_L2 else -FLT_MAX, np.float32)
    I = np.full(k, -1, np.int64)
    D[: order.size] = d[order]
    I[: order.size] = i[order]
    return D, I


def knn(xq, xb, k, metric, ids=None):
    """brute-force search under the rule"""
    dis = distances(xq, xb, metric)
    ids = np.arange(xb.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, np.int64)
    out = [select(dis[q], ids, k, metric) for q in range(dis.shape[0])]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def assign(x, centroids, metric):
    """the coarse assignment at add time: the best centroid under the rule, or -1 where no centroid is a result"""
    D, I = knn(x, centroids, 1, metric)
    return I[:, 0]


def ivf_lists(x, ids, centroids, metric):
    """the ids each list holds after add_with_ids(x, ids), in insertion order; rows without a result are dropped"""
    a = assign(x, centroids, metric)
    ids = np.asarray(ids, np.int64)
    return [ids[a == l] for l in range(centroids.shape[0])]


def ivfflat_search(xq, k, nprobe, centroids, lists_x, lists_ids, metric):
    """IndexIVFFlat::search under the rule: probes are the query's coarse results (at most nprobe), the stored
    vectors of the probed lists are the candidates"""
    Dc, Ic = knn(xq, centroids, nprobe, metric)
    Ds, Is = [], []
    for q in range(xq.shape[0]):
        probes = [int(l) for l in Ic[q] if l >= 0]
        if probes:
            xs = np.concatenate([lists_x[l] for l in probes]).reshape(-1, xq.shape[1])
            ii = np.concatenate([lists_ids[l] for l in probes])
        else:
            xs, ii = np.zeros((0, xq.shape[1]), np.float32), np.zeros(0, np.int64)
        D, I = select(distances(xq[q : q + 1], xs, metric)[0], ii, k, metric)
        Ds.append(D)
        Is.append(I)
    return np.stack(Ds), np.stack(Is)


# ------------------------------------------------------------------------------------------------------------------
# data
# ------------------------------------------------------------------------------------------------------------------
def special_rows(d, metric):
    """(rows [m, d], kinds [m]): every kind of non-ordinary row, zero outside its one or two set coordinates.  Their
    distance to a query of `queries` is non-finite, overflowing or exactly FLT_MAX (or +-FLT_MAX for inner product),
    so under L2 none of them is a result and under inner product only +inf and +FLT_MAX are."""
    rows, kinds = [], []

    def row(kind, **cols):
        r = np.zeros(d, np.float32)
        for c, v in cols.items():
            r[int(c[1:])] = v
        rows.append(r)
        kinds.append(kind)

    if metric == METRIC_L2:
        # queries are zero in columns 0 and 1
        row("inf", c2=np.inf)
        row("-inf", c3=-np.inf)
        row("nan", c2=np.nan)
        row("huge", c3=HUGE)
        row("-huge", c2=-HUGE)
        row("flt_max", c0=FMAX_A, c1=FMAX_B)
    else:
        # queries are zero in column 0, nonzero in column 1 (sign varies), one in column 2
        row("inf*0", c0=np.inf)  # NaN
        row("inf", c1=np.inf)  # +-inf by the query's sign
        row("-inf", c1=-np.inf)
        row("flt_max", c2=FLT_MAX)  # +FLT_MAX: a result
        row("-flt_max", c2=-FLT_MAX)  # -FLT_MAX: not a result
        row("nan", c3=np.nan)
    return np.stack(rows), kinds


def queries(rs, nq, d, metric):
    q = rs.randint(-3, 4, (nq, d)).astype(np.float32)
    if metric == METRIC_L2:
        q[:, :2] = 0
    else:
        q[:, 0] = 0
        q[:, 1] = rs.choice([-2, -1, 1, 2], nq)
        q[:, 2] = 1
    return q


def database(rs, n, d, metric, n_ordinary, positions=None):
    """n rows: n_ordinary small-integer rows and n - n_ordinary special rows (cycling through the kinds).  The
    special rows sit at `positions` when given (first row, last row, inside the first tile, around the database
    split), the rest spread at random."""
    spec, _ = special_rows(d, metric)
    n_spec = n - n_ordinary
    chosen = [] if positions is None else [p for p in dict.fromkeys(positions) if 0 <= p < n][:n_spec]
    rest = np.setdiff1d(np.arange(n), chosen)
    extra = rs.choice(rest, n_spec - len(chosen), replace=False) if n_spec > len(chosen) else np.zeros(0, np.int64)
    where = np.concatenate([np.asarray(chosen, np.int64), extra.astype(np.int64)])
    xb = rs.randint(-3, 4, (n, d)).astype(np.float32)
    xb[where] = spec[np.arange(where.size) % spec.shape[0]]
    return xb, np.sort(where)


def special_queries(d, metric):
    """queries that have no result at all under the rule (against finite data): NaN and +-inf / huge coordinates
    under L2, a NaN coordinate under inner product"""
    qs = []
    for v in ([np.nan, np.inf, -np.inf, HUGE] if metric == METRIC_L2 else [np.nan]):
        for c in (0, d - 1):
            q = np.ones(d, np.float32)
            q[c] = v
            qs.append(q)
    return np.stack(qs)
