"""numpy restatement of IDSelector::is_member (faiss/impl/IDSelector.{h,cpp}) and of filtered Flat search.

A selector is a tuple:
    ("range", imin, imax)   imin <= id < imax
    ("array", ids) / ("batch", ids)   id in ids
    ("bitmap", uint8 bytes)   (uint64)id >> 3 < len(bytes) and bit (id & 7) of byte id >> 3
    ("not", s), ("and", a, b), ("or", a, b), ("xor", a, b)
"""
import numpy as np

from oracle import oracle_np as o


def is_member(sel, ids):
    """bool array: which of the int64 ids `sel` accepts"""
    ids = np.asarray(ids, dtype=np.int64)
    kind = sel[0]
    if kind == "range":
        return (ids >= sel[1]) & (ids < sel[2])
    if kind in ("array", "batch"):
        return np.isin(ids, np.asarray(sel[1], dtype=np.int64))
    if kind == "bitmap":
        bm = np.asarray(sel[1], dtype=np.uint8)
        u = ids.astype(np.uint64)
        byte = u >> np.uint64(3)
        inside = byte < np.uint64(bm.size)
        out = np.zeros(ids.shape, dtype=bool)
        b = byte[inside].astype(np.int64)
        out[inside] = ((bm[b] >> (u[inside] & np.uint64(7)).astype(np.uint8)) & 1).astype(bool)
        return out
    if kind == "not":
        return ~is_member(sel[1], ids)
    a, b = is_member(sel[1], ids), is_member(sel[2], ids)
    if kind == "and":
        return a & b
    if kind == "or":
        return a | b
    if kind == "xor":
        return a ^ b
    raise ValueError(kind)


def knn_flat_sel(xq, xb, k, sel, metric=o.METRIC_L2):
    """IndexFlat::search with SearchParameters::sel, by membership: the k best selected rows by (distance, id),
    padded with -1 / +-FLT_MAX"""
    rows = np.nonzero(is_member(sel, np.arange(xb.shape[0], dtype=np.int64)))[0]
    nq = np.asarray(xq).shape[0]
    if rows.size == 0:
        D = np.full((nq, k), np.finfo(np.float32).max if metric == o.METRIC_L2 else -np.finfo(np.float32).max, np.float32)
        return D, np.full((nq, k), -1, np.int64)
    D, I = o.knn_flat(xq, np.asarray(xb)[rows], k, metric)
    return D, np.where(I >= 0, rows[np.maximum(I, 0)], -1)


def reference_selectors(num):
    """The eight selectors of the reference GPU tests (faiss/gpu/test/TestUtils.cpp:433-475) over ids [0, num)"""
    rng = ("range", num // 5, num * 4 // 5)
    arr = ("array", np.arange(0, num, 3, dtype=np.int64))
    bat = ("batch", np.arange(1, num, 5, dtype=np.int64))
    bm = np.zeros(num, dtype=np.uint8)  # num bytes, as the reference's IDSelectorBitmap(numAdd, ...)
    for i in range(0, num, 4):
        bm[i // 8] |= 1 << (i % 8)
    nt = ("not", rng)
    return {
        "Range": rng,
        "Array": arr,
        "Batch": bat,
        "Bitmap": ("bitmap", bm),
        "Not": nt,
        "And": ("and", rng, arr),
        "Or": ("or", rng, bat),
        "XOr": ("xor", nt, arr),
    }


def ivf_ids(n, seed=11):
    """add_with_ids ids for the IVF cases: a permutation mixing small ids, ids >= 2^40 and negative ids (-1 is never
    used: it marks a missing result)"""
    rs = np.random.RandomState(seed)
    ids = rs.permutation(n).astype(np.int64) * 3
    ids[::7] += 1 << 40
    ids[3::11] = -ids[3::11] - 2
    return ids


def ivf_selectors(ids):
    """the eight selector kinds over arbitrary stored ids: Range and Array from the sorted ids, a random 10 % Batch,
    a Bitmap over the small ids only"""
    ids = np.asarray(ids, dtype=np.int64)
    s = np.sort(ids)
    rng = ("range", int(s[len(s) // 5]), int(s[len(s) * 4 // 5]))
    arr = ("array", s[::3])
    bat = ("batch", np.random.RandomState(4).choice(ids, len(ids) // 10, replace=False))
    small = int(max(0, ids[(ids >= 0) & (ids < (1 << 40))].max(initial=0)))
    bm = np.zeros(small // 8 + 1, dtype=np.uint8)
    for i in range(0, small + 1, 2):
        bm[i // 8] |= 1 << (i % 8)
    nt = ("not", rng)
    return {
        "Range": rng,
        "Array": arr,
        "Batch": bat,
        "Bitmap": ("bitmap", bm),
        "Not": nt,
        "And": ("and", rng, arr),
        "Or": ("or", rng, bat),
        "XOr": ("xor", nt, arr),
    }


def ivfflat_search_sel(xq, k, nprobe, centroids, xb, ids, assign, sel, metric=o.METRIC_L2):
    """IndexIVFFlat::search with SearchParametersIVF{nprobe, sel}: the coarse search is not filtered; the selected
    entries of the probed lists are ranked by (exact distance, id).  Stored ids may be any int64 (negative ones
    included), so missing results are tracked by count, not by id."""
    xq = np.asarray(xq, dtype=np.float32)
    _, probes = o.knn_flat(xq, centroids, nprobe, metric)
    keep = is_member(sel, ids)
    big = np.finfo(np.float32).max if metric == o.METRIC_L2 else -np.finfo(np.float32).max
    D = np.full((xq.shape[0], k), big, np.float32)
    I = np.full((xq.shape[0], k), -1, np.int64)
    for q in range(xq.shape[0]):
        m = keep & np.isin(assign, probes[q][probes[q] >= 0])
        if not m.any():
            continue
        dis = o.pairwise(xq[q : q + 1], xb[m], metric, exact=True)[0]
        key = dis if metric == o.METRIC_L2 else -dis
        order = np.lexsort((ids[m], key))[:k]
        D[q, : order.size], I[q, : order.size] = dis[order], ids[m][order]
    return D, I


def equal_up_to_ties(D, I, rD, rI):
    """same distances, and the same ids for every distance value but the last of a row (the reference CPU's
    similarity heap orders a tie group by decreasing id, and a tie group cut by k may keep other members)"""
    if not np.array_equal(D, rD):
        return False
    for d, i, ri in zip(D, I, rI):
        for v in np.unique(d[d != d[-1]]):
            if set(i[d == v]) != set(ri[d == v]):
                return False
    return True
