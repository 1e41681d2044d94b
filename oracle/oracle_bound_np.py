"""TEST INFRASTRUCTURE ONLY -- certified top-k check of a k-NN result against float64 truth.

numpy only; it does not import the product.  A search result (D, I) of one query is checked against its
candidate set S (the whole database, the union of the probed lists, or the vectors the index's own codes
decode to), the float64 true distance t(i) of every candidate and a worst-case bound beta(i) on the error
of the fp32 arithmetic the kernel does for that candidate.  check_topk asserts:

  1. the first min(k, |S|) ids are unique members of S, the rest are -1 with the sentinel distance
     (FLT_MAX for L2, -FLT_MAX for inner product);
  2. |D[j] - t(I[j])| <= beta(I[j]) for every returned entry;
  3. D is monotone in the metric's direction, and equal fp32 distances come with ascending ids (the
     (key, id) total order of every list and merge, select.cuh);
  4. completeness: no candidate left out is certainly better than a returned one.  For L2, every
     i in S \\ I has t(i) + beta(i) >= max_j (t(I_j) - beta(I_j)); for IP the mirror image.

Error bounds.  u = 2^-24 is the unit roundoff of fp32 (round to nearest) and gamma(n) = n u / (1 - n u).
A sum of n terms s = sum_i p_i, each p_i a product formed with at most one rounding and the sum
accumulated in fp32 with n - 1 roundings, in ANY association (sequential, an FMA chain, pairwise, a
32-lane butterfly, two interleaved chains), satisfies |fl(s) - s| <= gamma(n) sum_i |p_i| (Higham,
Accuracy and Stability of Numerical Algorithms, 2nd ed., 3.1 and 3.5: each term passes through at most
n roundings, and an FMA only removes roundings).  That is why one checker serves every kernel: the
bounds below depend on how many roundings a term meets, never on the order of the additions.

  exact L2   (q_i - y_i) is rounded once, squared (once, or not at all inside an FMA), then d terms are
             summed: each term meets at most d + 2 roundings, |err| <= gamma(d + 3) * sum (q - y)^2.
  IP         d products summed: |err| <= gamma(d + 1) * sum |q_i y_i|.
  IVF-PQ     residual r~ = fl(q - c) (|r~_i - r_i| <= u |r_i|), each LUT entry an fma chain of dsub
             terms (r~_i - y_i)^2, then the M entries of a code summed: with t_i = r_i - y_i and
             e_i = 2 u |r_i| a bound on the residual's effect on the component,
               |err| <= gamma(dsub + M + 3) sum (|t_i| + e_i)^2 + sum (2 |t_i| e_i + e_i^2)
             (the second sum is how far ((|t| + e)^2 can move a square).  Precomputed tables evaluate
             ||q - c||^2 + sum_m (||y||^2 + 2 <c|y> - 2 <q|y>) instead, equal to the same value in exact
             arithmetic; every elementary term meets at most d + 2 dsub + M + 6 roundings, so
               |err| <= gamma(d + 2 dsub + M + 6) (||r||^2 + sum_i (y_i^2 + 2 |c_i y_i| + 2 |q_i y_i|)).
             IP: t = <q|c> + sum <q|y>, the coarse term handed in rounded to fp32, one add per lookup chain:
               |err| <= gamma(dsub + M + 5) (sum |q_i y_i| + sum |q_i c_i|).
  IVF-SQ     as IVF-PQ L2 with d terms, plus a per-component decode term: the kernel decodes
             x_i = m_i + b_i c_i with b_i = fl(vdiff_i / s) and m_i = fl(vmin_i + b_i / 2), forms
             a_i = fl(r~_i - m_i) and fma(-b_i, c_i, a_i).  Against the exact decode
             vmin_i + vdiff_i (c_i + 1/2) / s that moves the component by at most
             u|r_i| + u(|vmin_i| + |vdiff_i|) + (c_i + 1/2) u |vdiff_i| / s + u |a_i| (first order), which
             e_i = 4 u (|r_i| + |vmin_i| + |vdiff_i|) covers with room for the second-order terms.

The float64 truth itself carries a rounding error; callers add slack() of the magnitudes involved, far
below every fp32 bound (d 2^-53 against d 2^-24).
"""
import numpy as np

U = 2.0 ** -24
FLT_MAX = float(np.finfo(np.float32).max)
METRIC_INNER_PRODUCT = 0
METRIC_L2 = 1


def gamma(n):
    """gamma_n = n u / (1 - n u), u = 2^-24"""
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1.0 - n * U)


def slack(mag, d):
    """float64 rounding of a truth computed from d-term sums of magnitude `mag` (generous: 4 d 2^-53)"""
    return 4.0 * d * 2.0 ** -53 * np.asarray(mag, dtype=np.float64)


# ------------------------------------------------------------------ truth and bounds, one query x candidates
def l2_truth(q, Y):
    """t_i = sum_j (q_j - Y_ij)^2 in float64 and its fp32 bound gamma(d + 3) t_i (+ float64 slack)"""
    q = np.asarray(q, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    d = q.shape[0]
    t = ((Y - q[None, :]) ** 2).sum(1)
    return t, gamma(d + 3) * t + slack(t, d)


def ip_truth(q, Y):
    """t_i = <q | Y_i> in float64 and its fp32 bound gamma(d + 1) sum_j |q_j Y_ij|"""
    q = np.asarray(q, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    d = q.shape[0]
    t = Y @ q
    a = np.abs(Y) @ np.abs(q)
    return t, gamma(d + 1) * a + slack(a, d)


def l2_truth_many(Q, Y):
    """[nq, n] float64 L2 distances and bounds for many queries (matmul form; the slack covers its
    cancellation)"""
    Q = np.asarray(Q, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    d = Q.shape[1]
    qn = (Q * Q).sum(1)[:, None]
    yn = (Y * Y).sum(1)[None, :]
    t = np.maximum(qn + yn - 2.0 * (Q @ Y.T), 0.0)
    return t, gamma(d + 3) * t + slack(qn + yn, 4 * d)


def ip_truth_many(Q, Y):
    Q = np.asarray(Q, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    d = Q.shape[1]
    a = np.abs(Q) @ np.abs(Y).T
    return Q @ Y.T, gamma(d + 1) * a + slack(a, d)


def perturbed_l2_bound(t_comp, e_comp, n):
    """sum over the last axis of a perturbed squared-difference sum: components t_i (exact differences),
    e_i bounds on how far the kernel's component can sit from t_i before its final rounding, n the
    roundings a term meets in the sum: gamma(n) sum (|t| + e)^2 + sum (2 |t| e + e^2)"""
    at = np.abs(t_comp)
    e = np.asarray(e_comp, dtype=np.float64)
    return gamma(n) * ((at + e) ** 2).sum(-1) + (2.0 * at * e + e * e).sum(-1)


def pq_l2_truth(r, Yd, dsub, M):
    """IVF-PQ L2 without precomputed tables.  r: [d] float64 residual q - c of the probed list, Yd: [n, d]
    decoded codes.  Returns (t, beta)."""
    r = np.asarray(r, dtype=np.float64)
    tc = r[None, :] - np.asarray(Yd, dtype=np.float64)
    t = (tc * tc).sum(1)
    e = np.broadcast_to(2.0 * U * np.abs(r)[None, :], tc.shape)
    return t, perturbed_l2_bound(tc, e, dsub + M + 3) + slack(t, r.shape[0])


def pq_l2_precomp_truth(q, c, Yd, dsub, M):
    """IVF-PQ L2 through the precomputed tables (||q - c||^2 + ||y||^2 + 2<c|y> - 2<q|y>)."""
    q = np.asarray(q, dtype=np.float64)
    c = np.asarray(c, dtype=np.float64)
    Y = np.asarray(Yd, dtype=np.float64)
    d = q.shape[0]
    r = q - c
    t = ((r[None, :] - Y) ** 2).sum(1)
    a = (r * r).sum() + (Y * Y).sum(1) + 2.0 * (np.abs(Y) @ np.abs(c)) + 2.0 * (np.abs(Y) @ np.abs(q))
    return t, gamma(d + 2 * dsub + M + 6) * a + slack(a, d)


def pq_ip_truth(q, c, Yd, dsub, M):
    """IVF-PQ inner product: <q|c> + <q|y> (the coarse term handed to the scan rounded to fp32)."""
    q = np.asarray(q, dtype=np.float64)
    c = np.asarray(c, dtype=np.float64)
    Y = np.asarray(Yd, dtype=np.float64)
    t = float(q @ c) + Y @ q
    a = np.abs(Y) @ np.abs(q) + float(np.abs(q) @ np.abs(c))
    return t, gamma(dsub + M + 5) * a + slack(a, q.shape[0])


def sq_l2_truth(r, X, vmin, vdiff):
    """IVF-SQ L2.  r: [d] float64 residual (or the query without one), X: [n, d] the float64 EXACT decode
    vmin + vdiff (c + 1/2) / s (fp16 / 8bit_direct: the stored value, vmin = vdiff = 0)."""
    r = np.asarray(r, dtype=np.float64)
    tc = r[None, :] - np.asarray(X, dtype=np.float64)
    t = (tc * tc).sum(1)
    e = 4.0 * U * (np.abs(r) + np.abs(np.asarray(vmin, np.float64)) + np.abs(np.asarray(vdiff, np.float64)))
    e = np.broadcast_to(e[None, :], tc.shape)
    return t, perturbed_l2_bound(tc, e, r.shape[0] + 3) + slack(t, r.shape[0])


# ------------------------------------------------------------------ the checker
class CertificateError(AssertionError):
    pass


def _fail(what, msg):
    raise CertificateError(("%s: " % what if what else "") + msg)


def check_topk(D, I, cand_ids, t, beta, k, metric, what=""):
    """Certify one query's result.  D [k] float32, I [k] int64 as returned; cand_ids [|S|] the candidate
    ids (unique), t / beta [|S|] their float64 truth and fp32 error bound.  beta = 0 demands exact
    arithmetic: every distance bit-exact and the top-k exactly the best min(k, |S|) (ties in any order of
    membership, but listed by ascending id)."""
    D = np.asarray(D, dtype=np.float32).reshape(-1)
    I = np.asarray(I, dtype=np.int64).reshape(-1)
    cand_ids = np.asarray(cand_ids, dtype=np.int64).reshape(-1)
    t = np.asarray(t, dtype=np.float64).reshape(-1)
    beta = np.broadcast_to(np.asarray(beta, dtype=np.float64), t.shape)
    l2 = metric == METRIC_L2
    if D.shape[0] != k or I.shape[0] != k:
        _fail(what, "result has %d/%d entries, expected k = %d" % (D.shape[0], I.shape[0], k))
    n = cand_ids.shape[0]
    nv = min(k, n)
    # 1. valid prefix, -1 padding with the sentinel
    if np.any(I[:nv] == -1):
        j = int(np.argmax(I[:nv] == -1))
        _fail(what, "entry %d is -1 but %d candidates exist (expected %d valid entries)" % (j, n, nv))
    if np.any(I[nv:] != -1):
        _fail(what, "entries past %d must be -1, got %s" % (nv, I[nv:][I[nv:] != -1][:5]))
    sentinel = np.float32(FLT_MAX if l2 else -FLT_MAX)
    if np.any(D[nv:] != sentinel):
        _fail(what, "padding distances must be %r" % sentinel)
    Iv, Dv = I[:nv], D[:nv].astype(np.float64)
    if np.unique(Iv).shape[0] != nv:
        u, c = np.unique(Iv, return_counts=True)
        _fail(what, "duplicate ids %s" % u[c > 1][:5])
    order = np.argsort(cand_ids, kind="stable")
    sc = cand_ids[order]
    pos = np.searchsorted(sc, Iv)
    pos = np.minimum(pos, n - 1) if n else pos
    if n == 0 or np.any(sc[pos] != Iv):
        bad = Iv if n == 0 else Iv[sc[pos] != Iv]
        _fail(what, "ids not in the candidate set: %s" % bad[:5])
    pos = order[pos]
    # 2. every distance within its bound
    err = np.abs(Dv - t[pos])
    over = err > beta[pos]
    if np.any(over):
        j = int(np.argmax(over))
        _fail(what, "entry %d (id %d): distance %r, truth %r, |error| %.3e > bound %.3e"
              % (j, Iv[j], float(D[j]), t[pos][j], err[j], beta[pos][j]))
    # 3. order, ties by ascending id
    if nv > 1:
        a, b = D[: nv - 1], D[1:nv]
        wrong = (a > b) if l2 else (a < b)
        if np.any(wrong):
            j = int(np.argmax(wrong))
            _fail(what, "distances out of order at %d: %r then %r" % (j, float(a[j]), float(b[j])))
        tie = (a == b) & (Iv[: nv - 1] >= Iv[1:nv])
        if np.any(tie):
            j = int(np.argmax(tie))
            _fail(what, "equal distances %r at %d with ids %d, %d (must ascend)" % (float(a[j]), j, Iv[j], Iv[j + 1]))
    # 4. completeness
    if nv < n:
        left = np.ones(n, dtype=bool)
        left[pos] = False
        if l2:
            worst = np.max(t[pos] - beta[pos])
            better = t[left] + beta[left] < worst
        else:
            worst = np.min(t[pos] + beta[pos])
            better = t[left] - beta[left] > worst
        if np.any(better):
            i = int(np.argmax(better))
            _fail(what, "candidate id %d (truth %r, bound %.3e) is certainly better than a returned entry (%r)"
                  % (cand_ids[left][i], t[left][i], beta[left][i], worst))


def check_knn(D, I, cand_ids, T, B, k, metric, what=""):
    """check_topk for every row of D / I; T, B [nq, |S|] over one common candidate set"""
    for qi in range(D.shape[0]):
        check_topk(D[qi], I[qi], cand_ids, T[qi], B[qi], k, metric, what="%s query %d" % (what, qi))


def exact_topk(t, ids, k, metric):
    """The (key, id) total order's top-k of exactly computed distances: key = t (L2) or -t (IP), ties by
    ascending id; padded with -1 / the sentinel."""
    t = np.asarray(t, dtype=np.float64)
    ids = np.asarray(ids, dtype=np.int64)
    key = t if metric == METRIC_L2 else -t
    o = np.lexsort((ids, key))[:k]
    D = np.full(k, FLT_MAX if metric == METRIC_L2 else -FLT_MAX, dtype=np.float32)
    I = np.full(k, -1, dtype=np.int64)
    D[: o.shape[0]] = t[o].astype(np.float32)
    I[: o.shape[0]] = ids[o]
    return D, I
