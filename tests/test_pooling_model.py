"""CPU model of the sharded Flat search protocol (DESIGN.md 4, `FlatTcDatabase::search` with a FlatTcShard):
geometric rounds over each shard's rows, per-shard threshold selection on APPROXIMATE scores (|S' - S| <= eps),
cross-shard pooling of two certified lower bounds per query after every round
    c0 = (shard's k-th best S') - eps        c1 = (shard's ceil(k/S)-th best S') - eps
    T  = max(max_r c0, min_r c1)             thr_r = max(thr_r, T - eps)
and an exact re-rank of each shard's surviving base list, followed by the merge.  The model restates the protocol in
numpy (it does not call the product) and checks the property the design rests on: the merged result equals the exact
top-k of the whole database, for every shard count -- including 8 shards, where a shard keeps only ~k/8 of the ~k
entries in its (unsorted) base list.  It also restates the list walk of `tc_rerank_kernel`: groups of 32 entries, ended
only by a group of sentinels; the walk that ended at the first group without an entry above the pooled threshold (the
first bisection-select build) loses results at 8 shards, and the test shows that it would."""
import numpy as np
import pytest

LIST = 256


def _kth_largest(v, k):
    return np.partition(v, len(v) - k)[len(v) - k] if len(v) >= k else None


def _search(true_scores, approx, eps, k, nshard, r0, growth, rs, walk):
    n = true_scores.size
    bounds = [n * i // nshard for i in range(nshard + 1)]
    shards = [np.arange(bounds[i], bounds[i + 1]) for i in range(nshard)]
    order = [rs.permutation(s) for s in shards]  # each shard's permuted scan order
    kfrac = -(-k // nshard)
    thr = [-np.inf] * nshard
    base = [np.empty(0, dtype=np.int64) for _ in range(nshard)]  # row ids, unsorted
    nmax = max(len(s) for s in shards)
    seen = 0
    while seen < nmax:
        end = min(nmax, r0 if seen == 0 else seen * growth)
        c0, c1 = [], []
        for r in range(nshard):
            new = order[r][seen:end]
            cand = new[approx[new] > thr[r]]  # the kernel's filter
            pool = np.concatenate([base[r], cand])
            sc = approx[pool]
            kth = _kth_largest(sc, k)
            if kth is not None:
                thr[r] = max(thr[r], np.nextafter(kth - 2 * eps, -np.inf))
            keep = pool[approx[pool] > thr[r]]
            assert len(keep) <= LIST, "model sized so that the base list never overflows"
            base[r] = keep[rs.permutation(len(keep))]  # compacted, order carries no meaning
            c0.append(kth - eps if kth is not None else -np.inf)
            f = _kth_largest(sc, kfrac)
            c1.append(f - eps if f is not None else -np.inf)
        T = max(max(c0), min(c1))
        if T > -np.inf:
            for r in range(nshard):
                thr[r] = max(thr[r], np.nextafter(T - eps, -np.inf))
        seen = end
    # exact re-rank of each shard's base list + merge
    out = []
    for r in range(nshard):
        ids = np.full(LIST, -1, dtype=np.int64)
        ids[: len(base[r])] = base[r]
        got = []
        for g0 in range(0, LIST, 32):
            grp = ids[g0 : g0 + 32]
            present = grp >= 0
            valid = present & (approx[np.where(present, grp, 0)] > thr[r])
            if walk == "until_no_survivor" and not valid.any():
                break
            if walk == "until_sentinels" and not present.any():
                break
            got.extend(grp[valid].tolist())
        got = np.array(got, dtype=np.int64)
        got = got[np.argsort(-true_scores[got], kind="stable")][:k]
        out.append(got)
    allc = np.concatenate(out)
    return np.sort(allc[np.argsort(-true_scores[allc], kind="stable")][:k])


@pytest.mark.parametrize("nshard", [1, 2, 4, 8])
def test_pooled_thresholds_keep_the_exact_topk(nshard):
    # shard sizes 512 * 8^j: the last round is a full growth step, so the pooled threshold of the round before it is
    # ~8x looser than the final one and a shard's final base list holds ~k entries of which ~k/S survive the pooling
    k, n, eps = 100, 32768 * nshard, 2e-4
    lost_by_old_walk = 0
    for trial in range(40 if nshard == 8 else 6):  # a walk that stops early loses a shard's tail in ~1 % of the cases
        rs = np.random.RandomState(100 * nshard + trial)
        true_scores = rs.randn(n)
        approx = true_scores + rs.uniform(-eps, eps, n)
        exact = np.sort(np.argsort(-true_scores, kind="stable")[:k])
        got = _search(true_scores, approx, eps, k, nshard, r0=512, growth=8 if nshard >= 4 else 4, rs=rs, walk="until_sentinels")
        assert np.array_equal(got, exact), (nshard, trial)
        old = _search(true_scores, approx, eps, k, nshard, r0=512, growth=8 if nshard >= 4 else 4, rs=rs, walk="until_no_survivor")
        lost_by_old_walk += k - np.intersect1d(old, exact).size
    if nshard == 8:
        assert lost_by_old_walk > 0, "the model no longer reproduces the 8-shard failure it documents"
    if nshard == 1:
        assert lost_by_old_walk == 0
