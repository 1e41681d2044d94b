"""TEST INFRASTRUCTURE ONLY -- the certified top-k check of oracle_bound_np.check_topk, with the float64 truth
computed by torch on the device that holds the database.

torch only (the bound constants come from oracle_bound_np); it does not import the product.  certify_knn asserts,
for every row of a k-NN result (D, I) over a database Y of any size, the four conditions check_topk asserts:

  1. the first min(k, |S|) ids are unique members of the candidate set S, the rest are -1 with the sentinel
     distance (FLT_MAX for L2, -FLT_MAX for inner product);
  2. |D[j] - t(I[j])| <= beta(I[j]) for every returned entry, t computed in direct form in float64;
  3. D is monotone in the metric's direction, and equal distances come with ascending ids;
  4. completeness: no candidate left out is certainly better than the worst returned one.

The bounds are those of l2_truth_many / ip_truth_many: gamma(d + 3) t + slack(qn + yn, 4d) for L2 and
gamma(d + 1) |q|.|y| + slack(|q|.|y|, d) for inner product.  Completeness runs over row chunks of Y in float64
GEMM form, one query block at a time: the transient device memory is a few [q_block, row_chunk] float64
matrices, never the whole [nq, n] truth.

exact=True: integer-valued Q and Y whose every fp32 sum is exact (checked, else ValueError).  The bound is 0 and
the result must be the (key, id) total order's top-k (oracle_bound_np.exact_topk) bit for bit, including which
members of the tie group at rank k are kept: the smallest ids.

Q and Y are taken as the kernel saw them (fp16 storage: both rounded to fp16; fp16 / bf16 inputs: as they are,
widened here); the certifier does not round anything itself.
"""
import torch

from oracle.oracle_bound_np import FLT_MAX, METRIC_L2, CertificateError, gamma, slack

EXACT_LIMIT = 2.0 ** 24  # every partial sum of an fp32 accumulation of integers below this is exact


def _fail(what, msg):
    raise CertificateError(("%s: " % what if what else "") + msg)


def _first(mask):
    """(row, col) of the first set entry of a 2-D bool tensor"""
    r, c = (int(v) for v in mask.nonzero()[0])
    return r, c


def _exact_regime(Q, Y, metric, row_chunk):
    """refuse data whose fp32 sums are not all exact integers"""
    d = Q.shape[1]
    qmax, ymax = 0.0, 0.0
    if Q.numel():
        q = Q.double()
        if not bool((q == q.round()).all()):
            raise ValueError("exact mode needs integer-valued queries")
        qmax = float(q.abs().max())
    for r0 in range(0, Y.shape[0], row_chunk):
        y = Y[r0:r0 + row_chunk].double()
        if not bool((y == y.round()).all()):
            raise ValueError("exact mode needs integer-valued rows (rows %d..%d are not)" % (r0, r0 + y.shape[0]))
        ymax = max(ymax, float(y.abs().max()))
    worst = d * (qmax + ymax) ** 2 if metric == METRIC_L2 else d * qmax * ymax
    if worst >= EXACT_LIMIT:
        raise ValueError("exact mode: sums up to %g are not exact in fp32 (limit 2^24)" % worst)


def _returned_truth(Q64, Y, Iv, l2, d, exact, elems):
    """[nq, nv] float64 truth (direct form) and bound of every returned entry, in query sub-blocks of at most
    `elems` gathered float64 components"""
    nq, nv = Iv.shape
    T = torch.zeros((nq, nv), dtype=torch.float64, device=Y.device)
    B = torch.zeros_like(T)
    if nv == 0:
        return T, B
    sb = max(1, elems // max(1, nv * d))
    g = float(gamma(d + 3 if l2 else d + 1))
    s = float(slack(1.0, 4 * d if l2 else d))
    for q0 in range(0, nq, sb):
        q = Q64[q0:q0 + sb]
        y = Y[Iv[q0:q0 + sb]].double()  # [b, nv, d]
        if l2:
            T[q0:q0 + sb] = ((y - q[:, None, :]) ** 2).sum(-1)
            B[q0:q0 + sb] = g * T[q0:q0 + sb] + s * ((q * q).sum(1)[:, None] + (y * y).sum(-1))
        else:
            T[q0:q0 + sb] = (y * q[:, None, :]).sum(-1)
            a = (y.abs() * q.abs()[:, None, :]).sum(-1)
            B[q0:q0 + sb] = g * a + s * a
        del y
    if exact:
        B.zero_()
    return T, B


def certify_knn(D, I, Q, Y, k, metric, candidates=None, exact=False, q_block=2048, row_chunk=1 << 16, what=""):
    """Certify a k-NN result.  D [nq, k] float32 and I [nq, k] integer ids (numpy or torch, any device), Q [nq, d]
    and Y [n, d] torch tensors of any float dtype (Y's device runs the check), candidates: None (every row) or a
    bool mask [n] of the rows a selector admits.  Raises CertificateError on the first violation; q_block * row_chunk
    bounds the float64 elements of each transient matrix (1 GiB at the defaults)."""
    dev = Y.device
    n, d = Y.shape
    Q = torch.as_tensor(Q).to(dev)
    nq = Q.shape[0]
    D = torch.as_tensor(D).to(dev, torch.float32)
    I = torch.as_tensor(I).to(dev, torch.int64)
    l2 = metric == METRIC_L2
    if tuple(D.shape) != (nq, k) or tuple(I.shape) != (nq, k):
        _fail(what, "result has shape %s / %s, expected (%d, %d)" % (tuple(D.shape), tuple(I.shape), nq, k))
    if Q.shape[1] != d:
        _fail(what, "queries of dimension %d against rows of %d" % (Q.shape[1], d))
    if exact:
        _exact_regime(Q, Y, metric, row_chunk)
    if candidates is not None:
        candidates = torch.as_tensor(candidates).to(dev, torch.bool)
        assert candidates.shape == (n,), "candidates must be a bool mask over the %d rows" % n
        nS = int(candidates.sum())
    else:
        nS = n
    nv = min(k, nS)
    Iv, Dv = I[:, :nv], D[:, :nv]

    # 1. valid prefix, -1 padding with the sentinel
    bad = Iv == -1
    if bool(bad.any()):
        qi, j = _first(bad)
        _fail(what, "query %d: entry %d is -1 but %d candidates exist (expected %d valid entries)" % (qi, j, nS, nv))
    bad = I[:, nv:] != -1
    if bool(bad.any()):
        qi, j = _first(bad)
        _fail(what, "query %d: entries past %d must be -1, got %d at %d" % (qi, nv, int(I[qi, nv + j]), nv + j))
    sentinel = torch.tensor(FLT_MAX if l2 else -FLT_MAX, dtype=torch.float32, device=dev)
    bad = D[:, nv:] != sentinel
    if bool(bad.any()):
        qi, j = _first(bad)
        _fail(what, "query %d: padding distance %r at %d, must be %r" % (qi, float(D[qi, nv + j]), nv + j, float(sentinel)))
    if nv > 1:
        srt = Iv.sort(1).values
        bad = srt[:, 1:] == srt[:, :-1]
        if bool(bad.any()):
            qi, j = _first(bad)
            _fail(what, "query %d: duplicate id %d" % (qi, int(srt[qi, j])))
    bad = (Iv < 0) | (Iv >= n)
    if candidates is not None and not bool(bad.any()):
        bad = ~candidates[Iv]
    if bool(bad.any()):
        qi, j = _first(bad)
        _fail(what, "query %d: id %d at %d is not in the candidate set" % (qi, int(Iv[qi, j]), j))

    # 2. every distance within its bound
    Q64 = Q.double()
    Tr, Br = _returned_truth(Q64, Y, Iv, l2, d, exact, q_block * row_chunk // 2)
    err = (Dv.double() - Tr).abs()
    bad = ~(err <= Br)  # NaN fails too
    if bool(bad.any()):
        qi, j = _first(bad)
        _fail(what, "query %d: entry %d (id %d): distance %r, truth %r, |error| %.3e > bound %.3e"
              % (qi, j, int(Iv[qi, j]), float(Dv[qi, j]), float(Tr[qi, j]), float(err[qi, j]), float(Br[qi, j])))

    # 3. order, ties by ascending id
    if nv > 1:
        a, b = Dv[:, :-1], Dv[:, 1:]
        bad = (a > b) if l2 else (a < b)
        if bool(bad.any()):
            qi, j = _first(bad)
            _fail(what, "query %d: distances out of order at %d: %r then %r" % (qi, j, float(a[qi, j]), float(b[qi, j])))
        bad = (a == b) & (Iv[:, :-1] >= Iv[:, 1:])
        if bool(bad.any()):
            qi, j = _first(bad)
            _fail(what, "query %d: equal distances %r at %d with ids %d, %d (must ascend)"
                  % (qi, float(a[qi, j]), j, int(Iv[qi, j]), int(Iv[qi, j + 1])))

    # 4. completeness
    if nv == 0 or nv >= nS:
        return
    worst = (Tr - Br).max(1).values if l2 else (Tr + Br).min(1).values  # [nq]
    last_id = Iv[:, nv - 1]  # exact: the largest id of the rank-k tie group (ascending within ties, checked above)
    g = float(gamma(d + 3 if l2 else d + 1))
    s = float(slack(1.0, 4 * d if l2 else d))
    for q0 in range(0, nq, q_block):
        q = Q64[q0:q0 + q_block]
        b = q.shape[0]
        qn = (q * q).sum(1, keepdim=True)
        w = worst[q0:q0 + q_block, None]
        ret = Iv[q0:q0 + q_block]
        rows = torch.arange(b, device=dev)[:, None].expand_as(ret)
        last = last_id[q0:q0 + q_block, None]
        for r0 in range(0, n, row_chunk):
            y = Y[r0:r0 + row_chunk].double()
            rc = y.shape[0]
            cols = torch.arange(r0, r0 + rc, device=dev)[None, :]
            if l2:
                t = q @ y.T  # [b, rc]
                yn = (y * y).sum(1)[None, :]
                t.mul_(-2.0).add_(qn).add_(yn).clamp_(min=0.0)
                if exact:
                    mark = (t < w) | ((t == w) & (cols < last))
                else:
                    t.mul_(1.0 + g).add_(qn, alpha=s).add_(yn, alpha=s)  # t + beta
                    mark = t < w
                del t
            else:
                t = q @ y.T
                if exact:
                    mark = (t > w) | ((t == w) & (cols < last))
                else:
                    a = q.abs() @ y.abs().T
                    t.sub_(a.mul_(g + s))  # t - beta
                    del a
                    mark = t > w
                del t
            if candidates is not None:
                mark &= candidates[None, r0:r0 + rc]
            rel = ret - r0
            inside = (rel >= 0) & (rel < rc)
            mark[rows[inside], rel[inside]] = False
            if bool(mark.any()):
                qi, c = _first(mark)
                qq, yy = q[qi], y[c]
                if l2:
                    tt = float(((qq - yy) ** 2).sum())
                    bb = g * tt + s * float((qq * qq).sum() + (yy * yy).sum())
                else:
                    tt = float((qq * yy).sum())
                    bb = (g + s) * float((qq.abs() * yy.abs()).sum())
                _fail(what, "query %d: candidate id %d (truth %r, bound %.3e) is certainly better than a returned "
                      "entry (%r%s)" % (q0 + qi, r0 + c, tt, 0.0 if exact else bb, float(w[qi, 0]),
                                        ", rank-k tie kept id %d" % int(last[qi, 0]) if exact else ""))
