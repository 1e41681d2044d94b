"""Benchmark of IVF retrieval: search against search_and_reconstruct, reconstruct_n over the whole index, and
reconstruct_batch of random ids, on the README's IVF configs.

    python bench_reconstruct.py [--n 10000000] [--nq 10000] [--k 100] [--reps 3] [--batch 1000000]

Configs (N = --n rows, d = 128, nlist = 4096, nq = 10k, k = 100, everything resident on the device): IVF-Flat and
IVF-SQ8 at nprobe = 64, IVF-PQ M = 32 at nprobe = 32.  Per config and call, one JSON line with the median of --reps
timed calls after a warm-up call (CUDA events; the calls end in a device synchronise):

  * search / search_and_reconstruct: both times, and the ratio.  search_and_reconstruct's extra work is the per-call
    table of arena slots the scans read as their id table (8 B per stored slot, reported), the slot-carrying merge
    and the decode of nq * k rows.
  * reconstruct_n(0, N): bytes moved over the call's time against the data-sheet 3.35 TB/s of the H100 SXM.  Bytes:
    the ids-to-slots pass reads 8 B of id per arena slot and writes 8 B per row; the decode reads the 8 B slot, the
    code (codeSize B) and writes d * 4 B per row.
  * reconstruct_batch of --batch random stored ids, including the ids-to-slots pass (key sort, arena pass).

Every line checks its own result: D and I of search_and_reconstruct equal search's; the decoded rows of the ids of 8
sampled lists equal the numpy restatement of the CPU IndexIVF decode (oracle/oracle_recons_np.py, pinned bit for bit
against the reference library by tests/test_reconstruct_oracle.py); search_and_reconstruct's rows equal
reconstruct_batch of the returned ids (ids are unique here).  The card's name, power limit and SM clock are read in
the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_metrics import gpu_identity, timed  # noqa: E402

HBM_TBPS = 3.35


def median_ms(torch, fn, reps):
    fn()
    return float(np.median([timed(torch, fn) for _ in range(reps)]))


def sampled_truth(fb, idx, kind, kw, lists):
    """{id: decoded row} for every entry of the sampled lists, by the numpy restatement of the CPU decode"""
    from oracle import oracle_recons_np as rn

    cent = idx.getCoarseCentroids()
    out = {}
    for l in lists:
        ids = idx.getListIndices(l)
        if ids.size == 0:
            continue
        x = rn.reconstruct_list(kind, idx.getListVectorData(l), l, idx.d, cent, **kw)
        out.update({int(i): x[r] for r, i in enumerate(ids)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1_000_000)
    a = ap.parse_args()

    import torch

    import faiss_b200 as fb
    from oracle import oracle_recons_np as rn
    from oracle import oracle_sq_np as so

    assert torch.cuda.is_available(), "bench_reconstruct.py measures on a GPU"
    card = gpu_identity(0)
    res = fb.StandardGpuResources()
    d, nlist = 128, 4096
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1234)
    xb = torch.rand((a.n, d), generator=gen, device="cuda")
    xq = torch.rand((a.nq, d), generator=gen, device="cuda")
    configs = [
        ("ivfflat", rn.FLAT, lambda: fb.GpuIndexIVFFlat(res, d, nlist), 64),
        ("ivfsq8", rn.SQ, lambda: fb.GpuIndexIVFScalarQuantizer(res, d, nlist, so.QT_8bit), 64),
        ("ivfpq_m32", rn.PQ, lambda: fb.GpuIndexIVFPQ(res, d, nlist, 32, 8), 32),
    ]
    rs = np.random.RandomState(7)
    for name, kind, make, nprobe in configs:
        idx = make()
        idx.train(xb[: nlist * 64])
        idx.add(xb)
        idx.nprobe = nprobe
        torch.cuda.synchronize()
        if kind == rn.PQ:
            kw = {"M": 32, "nbits": 8, "pq": idx.getPQCentroids()}
        elif kind == rn.SQ:
            kw = {"qtype": so.QT_8bit, "by_residual": True, "trained": idx.getTrained()}
        else:
            kw = {}
        ccs, cs = idx.code_sizes()
        truth = sampled_truth(fb, idx, kind, kw, rs.choice(nlist, 8, replace=False))
        base = {"config": name, "N": a.n, "d": d, "nlist": nlist, "nprobe": nprobe, "nq": a.nq, "k": a.k,
                "code_size": cs, "gpu": card}

        # search against search_and_reconstruct
        out = {}

        def s():
            out["s"] = idx.search(xq, a.k)

        def sr():
            out["sr"] = idx.search_and_reconstruct(xq, a.k)

        t_s = median_ms(torch, s, a.reps)
        t_sr = median_ms(torch, sr, a.reps)
        D0, I0 = out["s"]
        D, I, R = out["sr"]
        ok = bool(torch.equal(D, D0) and torch.equal(I, I0))
        qs = rs.choice(a.nq, 32, replace=False)
        Iq = I[qs].reshape(-1).cpu().numpy()
        Rq = R[qs].reshape(-1, d).cpu().numpy()
        valid = Iq >= 0
        ok = ok and np.array_equal(Rq[valid].view(np.uint32), idx.reconstruct_batch(Iq[valid]).view(np.uint32))
        hits = [(r, truth[int(i)]) for r, i in enumerate(Iq) if int(i) in truth]
        ok = ok and all(np.array_equal(Rq[r].view(np.uint32), v.view(np.uint32)) for r, v in hits)
        print(json.dumps(dict(base, call="search vs search_and_reconstruct", search_ms=t_s, search_and_reconstruct_ms=t_sr,
                              ratio=t_sr / t_s, slot_table_bytes=8 * a.n, parity_ok=ok,
                              parity="D, I equal search's; 32 queries' rows equal reconstruct_batch and, for %d results in "
                                     "8 sampled lists, the CPU decode" % len(hits))), flush=True)

        # reconstruct_n(0, N) into a device buffer
        outn = torch.empty((a.n, d), dtype=torch.float32, device="cuda")

        def rnall():
            fb.check(fb.lib.faiss_Index_reconstruct_n(idx._h, fb.ctypes.c_int64(0), fb.ctypes.c_int64(a.n),
                                                      fb._ptr(outn, fb._c_f)))

        t_n = median_ms(torch, rnall, a.reps)
        # arena slots >= stored rows; the ids pass reads the arena's ids (counted at N here: a lower bound)
        nbytes = a.n * (8 + 8 + 8 + cs + 4 * d)
        keys = np.array(sorted(truth), dtype=np.int64)
        ok = np.array_equal(outn[torch.from_numpy(keys).cuda()].cpu().numpy().view(np.uint32),
                            np.stack([truth[int(i)] for i in keys]).view(np.uint32))
        del outn
        print(json.dumps(dict(base, call="reconstruct_n(0, N)", ms=t_n, bytes=nbytes, tb_per_s=nbytes / t_n / 1e9,
                              frac_of_hbm_datasheet=nbytes / t_n / 1e9 / HBM_TBPS, parity_ok=bool(ok),
                              parity="rows of the %d ids of 8 sampled lists equal the CPU decode" % keys.size)), flush=True)

        # reconstruct_batch of random ids, ids -> slots included
        kb = torch.from_numpy(rs.randint(0, a.n, a.batch).astype(np.int64)).cuda()
        outb = torch.empty((a.batch, d), dtype=torch.float32, device="cuda")

        def rb():
            fb.check(fb.lib.faiss_Index_reconstruct_batch(idx._h, fb.ctypes.c_int64(a.batch), fb._ptr(kb, fb._c_i64),
                                                          fb._ptr(outb, fb._c_f)))

        t_b = median_ms(torch, rb, a.reps)
        kbh = kb.cpu().numpy()
        sel = np.array([int(i) in truth for i in kbh])
        ok = np.array_equal(outb[torch.from_numpy(np.nonzero(sel)[0]).cuda()].cpu().numpy().view(np.uint32),
                            np.stack([truth[int(i)] for i in kbh[sel]]).reshape(-1, d).view(np.uint32)) if sel.any() else False
        print(json.dumps(dict(base, call="reconstruct_batch", keys=a.batch, ms=t_b, keys_per_s=a.batch / t_b * 1e3,
                              parity_ok=bool(ok),
                              parity="%d keys in 8 sampled lists equal the CPU decode" % int(sel.sum()))), flush=True)
        del idx, outb, kb
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
