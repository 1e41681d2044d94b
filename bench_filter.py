"""Benchmark of filtered search (SearchParameters::sel) on GpuIndexFlat and the IVF indexes.

    python bench_filter.py [--n 10000000] [--nq 10000] [--k 100] [--reps 3] [--ivf-n 10000000] [--no-ivf]

Flat: N = 10M rows, d = 128, nq = 10k, k = 100, queries and rows resident on the device.  Selectivity 1, 0.5, 0.1,
0.01 and 0.001, as an IDSelectorRange [0, s N) and as a random IDSelectorBitmap.  The index picks the route from the
selected count: the masked tensor-core search, or -- at most 1 row in 32 selected -- the compacted route (the
selected rows gathered and searched with the exact kernel).  To show where that choice should fall, every line also
times the two routes' costs apart: the unfiltered tensor-core search (what the masked route costs: the same kernel
over all N rows) and the exact kernel over an index that holds only the selected rows (what the compacted route
costs, before the gather).

IVF: IVF-Flat (nlist = 4096, nprobe = 64) and IVF-PQ (M = 32, nlist = 4096, nprobe = 32; the shape of bench_ivf.py's
configs[3]) over --ivf-n rows, each with a random 10 % IDSelectorBatch, against the same search unfiltered.

Per workload, one JSON line: the median of --reps timed calls after a warm-up call (CUDA events), QPS, the
selector's mask-build kernel time (KernelTiming "sel_mask"), the tensor-core kernel time and launches ("flat_tc":
0 launches means the compacted route ran), and a parity check.  Flat parity: 64 queries against the reference CPU
IndexFlat with the same selector (oracle/_ref) where it was built; IVF: every returned label is selected.  The card's
name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_metrics import gpu_identity, timed  # noqa: E402


def kernel_ms(fb, name):
    ms, n = ctypes.c_double(), ctypes.c_int()
    fb.lib.faiss_b200_kernel_timing_collect(name.encode(), ctypes.byref(ms), ctypes.byref(n))
    return ms.value, n.value


def run(torch, fb, idx, xq, k, reps, params=None):
    """median ms of reps calls after a warm-up, kernel timings of the last call"""
    idx.search(xq, k, params=params)
    times = []
    for r in range(reps):
        if r == reps - 1:
            fb.lib.faiss_b200_kernel_timing(1)
            for name in ("sel_mask", "flat_tc"):
                kernel_ms(fb, name)
        times.append(timed(torch, lambda: idx.search(xq, k, params=params)))
    mask, _ = kernel_ms(fb, "sel_mask")
    tc, tcn = kernel_ms(fb, "flat_tc")
    fb.lib.faiss_b200_kernel_timing(0)
    return float(np.median(times)), {"mask_ms": mask, "flat_tc_ms": tc, "flat_tc_launches": tcn}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ivf-n", type=int, default=10_000_000)
    ap.add_argument("--no-ivf", action="store_true")
    ap.add_argument("--no-parity", action="store_true")
    a = ap.parse_args()

    import torch

    import faiss_b200 as fb
    from oracle import oracle_sel_np as osel

    assert torch.cuda.is_available(), "bench_filter.py needs a GPU"
    gpu = gpu_identity()
    res = fb.StandardGpuResources()
    gen = torch.Generator(device="cuda").manual_seed(0)
    N, d, nq, k = a.n, a.d, a.nq, a.k
    xb = torch.rand((N, d), generator=gen, device="cuda")
    xq = torch.rand((nq, d), generator=gen, device="cuda")
    idx = fb.GpuIndexFlatL2(res, d)
    idx.add(xb)
    t_unf, info_unf = run(torch, fb, idx, xq, k, a.reps)
    ref_idx = None
    if not a.no_parity:
        from oracle import ref, ref_sel

        if ref_sel.available():
            ref_idx = ref.IndexFlat(d, 1)
            ref_idx.add(xb.cpu().numpy())
    rs = np.random.RandomState(1)
    for sel_kind in ("range", "bitmap"):
        for s in (1.0, 0.5, 0.1, 0.01, 0.001):
            if sel_kind == "range":
                spec = ("range", 0, int(s * N))
                rows = np.arange(int(s * N))
            else:
                keep = rs.rand(N) < s
                spec = ("bitmap", np.packbits(keep, bitorder="little"))
                rows = np.nonzero(keep)[0]
            sel = fb.IDSelectorRange(spec[1], spec[2]) if sel_kind == "range" else fb.IDSelectorBitmap(spec[1])
            t, info = run(torch, fb, idx, xq, k, a.reps, fb.SearchParameters(sel=sel))
            line = {"bench": "flat", "selector": sel_kind, "selectivity": s, "selected": int(rows.size), "N": N, "d": d,
                    "nq": nq, "k": k, "ms": t, "qps": nq / t * 1e3, **info,
                    "route": "masked_tensor_cores" if info["flat_tc_launches"] else "compacted",
                    "unfiltered_ms": t_unf, "unfiltered_qps": nq / t_unf * 1e3}
            if s <= 0.1:  # the compacted route's search: the exact kernel over the selected rows only
                sub = fb.GpuIndexFlatL2(res, d, use_tensor_cores=False)
                sub.add(xb[torch.from_numpy(rows).cuda()].contiguous())
                line["exact_over_selected_ms"], _ = run(torch, fb, sub, xq, k, a.reps)
                del sub
            D, I = idx.search(xq[:64], k, params=fb.SearchParameters(sel=sel))
            if ref_idx is not None:
                from oracle import oracle_np as o
                from oracle import ref_sel

                rD, rI = ref_sel.search(ref_idx, xq[:64].cpu().numpy(), k, spec)
                try:
                    o.compare_lists(rD, rI, D.cpu().numpy(), I.cpu().numpy(), eps=1e-4, pct_max_diff1=0.02, pct_max_diffN=0.01)
                    line["parity"] = "ok (reference IndexFlat, 64 queries)"
                except AssertionError as e:
                    line["parity"] = "FAIL " + str(e)[:200]
            else:
                got = I.cpu().numpy()
                line["parity"] = "labels selected" if osel.is_member(spec, got[got >= 0]).all() else "FAIL: unselected label"
            line["gpu"] = gpu
            print(json.dumps(line), flush=True)
    del idx, xb
    torch.cuda.empty_cache()
    if a.no_ivf:
        return
    n = a.ivf_n
    xb = torch.rand((n, d), generator=gen, device="cuda")
    batch = np.random.RandomState(2).choice(n, n // 10, replace=False)
    for name, make, nprobe in (
        ("ivfflat", lambda: fb.GpuIndexIVFFlat(res, d, 4096), 64),
        ("ivfpq", lambda: fb.GpuIndexIVFPQ(res, d, 4096, 32, 8), 32),
    ):
        ivf = make()
        ivf.train(xb[: 4096 * 64])
        ivf.add(xb)
        t_unf, _ = run(torch, fb, ivf, xq, k, a.reps, fb.SearchParametersIVF(nprobe=nprobe))
        sel = fb.IDSelectorBatch(batch)
        t, info = run(torch, fb, ivf, xq, k, a.reps, fb.SearchParametersIVF(nprobe=nprobe, sel=sel))
        D, I = ivf.search(xq[:64], k, params=fb.SearchParametersIVF(nprobe=nprobe, sel=sel))
        got = I.cpu().numpy()
        ok = osel.is_member(("batch", batch), got[got >= 0]).all()
        print(json.dumps({"bench": name, "selector": "batch", "selectivity": 0.1, "N": n, "nlist": 4096, "nprobe": nprobe,
                          "nq": nq, "k": k, "ms": t, "qps": nq / t * 1e3, "mask_ms": info["mask_ms"],
                          "unfiltered_ms": t_unf, "unfiltered_qps": nq / t_unf * 1e3,
                          "parity": "labels selected (64 queries)" if ok else "FAIL: unselected label", "gpu": gpu}), flush=True)
        del ivf
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
