"""Benchmark of all-pairs distances (pairwise_distance_gpu / bfKnn with k = -1) and of knn_gpu's input formats.

    python bench_pairwise.py [--nq 10000] [--n 1000000] [--dims 16,64,128] [--reps 5]

Pairwise lines: L2 and L1 at nq x N for every d, queries, database and the [nq, N] fp32 output resident on the device
(40 GB at the default shape).  Each timed call alternates with the exact k-NN kernel (GpuIndexFlat with
use_tensor_cores=False, k = 100) on the same inputs: the same arithmetic with selection instead of stores, the
yardstick for components/s.  Reported: the median of --reps CUDA-event timed calls after a warm-up call,
components/s (nq * N * d / t), output bytes/s and its share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s),
the k-NN kernel's ms and components/s, and torch.cdist (p = 2 / p = 1) on the same inputs for its time only: its
values differ (the norm expansion for p = 2).  Each line checks 4 sampled rows against knn_gpu's distances.

Format lines: knn_gpu at N = --n, d = 128, k = 100, nq = --nq, device-resident, per input format (fp32 / fp16 / bf16
x row / column-major vectors): the conversion's cost over the fp32 row-major call.

The card's name, power limit and SM clock are read in the same run and printed first.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3


def gpu_identity(gpu_index=0):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        name, plim, smax, sm = [x.strip() for x in r.stdout.strip().split(",")[:4]]
        return {"name": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax), "sm_mhz_now": float(sm)}
    except Exception as e:
        return {"error": str(e)[:100]}


def timed(torch, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def median_alternating(torch, fns, reps):
    for f in fns:  # warm-up: every shape of the timed window
        f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            ts[i].append(timed(torch, f))
    return [float(np.median(t)) for t in ts], ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--dims", default="16,64,128")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--skip-formats", action="store_true")
    args = ap.parse_args()

    import torch

    import faiss_b200 as fb

    if not torch.cuda.is_available():
        sys.exit("bench_pairwise.py needs a CUDA device")
    dev = torch.cuda.current_device()
    print(json.dumps({"card": gpu_identity(dev), "nq": args.nq, "n": args.n, "reps": args.reps}), flush=True)
    res = fb.StandardGpuResources()
    res.setDefaultStream(dev, torch.cuda.current_stream(dev).cuda_stream)
    nq, n, k = args.nq, args.n, args.k
    gen = torch.Generator(device="cuda")

    for d in [int(x) for x in args.dims.split(",")]:
        gen.manual_seed(d)
        xb = torch.rand((n, d), generator=gen, device="cuda")
        xq = torch.rand((nq, d), generator=gen, device="cuda")
        for name, metric, p in (("L2", fb.METRIC_L2, 2.0), ("L1", fb.METRIC_L1, 1.0)):
            idx = fb.GpuIndexFlat(res, d, metric, use_tensor_cores=False)
            idx.add(xb)
            Dk = torch.empty((nq, k), dtype=torch.float32, device="cuda")
            Ik = torch.empty((nq, k), dtype=torch.int64, device="cuda")
            out = torch.empty((nq, n), dtype=torch.float32, device="cuda")
            run = lambda: fb.pairwise_distance_gpu(res, xq, xb, D=out, metric=metric)  # noqa: E731
            run_knn = lambda: idx.search(xq, k, Dk, Ik)  # noqa: E731
            (t, tk), (ts, tks) = median_alternating(torch, [run, run_knn], args.reps)
            # check: sampled rows of the matrix at knn's ids equal knn's distances
            rows = [0, 1, nq // 2, nq - 1]
            ok = bool(torch.equal(torch.gather(out[rows], 1, Ik[rows]), Dk[rows]))
            # cdist: time only, with our output freed (it allocates its own [nq, n] matrix)
            del out
            torch.cuda.empty_cache()
            cdist_err = None
            try:
                (tc,), _ = median_alternating(torch, [lambda: torch.cdist(xq, xb, p=p)], args.reps)
            except RuntimeError as e:
                tc, cdist_err = None, str(e)[:80]
            torch.cuda.empty_cache()
            comps = float(nq) * n * d
            line = {
                "bench": "pairwise", "metric": name, "nq": nq, "n": n, "d": d,
                "ms_median": round(t, 3), "ms_all": [round(v, 3) for v in ts],
                "component_evals_per_s": comps / (t * 1e-3),
                "output_bytes_per_s": 4.0 * nq * n / (t * 1e-3),
                "output_share_of_hbm": 4.0 * nq * n / (t * 1e-3) / HBM_BYTES_PER_S,
                "knn_exact_k": k, "knn_exact_ms_median": round(tk, 3), "knn_exact_ms_all": [round(v, 3) for v in tks],
                "knn_exact_component_evals_per_s": comps / (tk * 1e-3),
                "ratio_vs_knn_components_per_s": tk / t,
                "torch_cdist_ms_median": None if tc is None else round(tc, 3),
                "knn_consistency": "ok" if ok else "FAIL",
            }
            if cdist_err:
                line["torch_cdist_error"] = cdist_err
            print(json.dumps(line), flush=True)
            del idx

    if args.skip_formats:
        return
    d = 128
    gen.manual_seed(7)
    xb32 = torch.rand((n, d), generator=gen, device="cuda")
    xq32 = torch.rand((nq, d), generator=gen, device="cuda")
    formats = []
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        for col in (False, True):
            xb = xb32.to(dt)
            xb = xb.t().contiguous().t() if col else xb
            formats.append(("%s_%s" % (str(dt).split(".")[-1], "col" if col else "row"), xq32.to(dt), xb))
    fns = [lambda xq=xq, xb=xb: fb.knn_gpu(res, xq, xb, k) for _, xq, xb in formats]
    meds, alls = median_alternating(torch, fns, args.reps)
    for (name, _, _), t, ts in zip(formats, meds, alls):
        print(json.dumps({"bench": "knn_gpu_format", "format": name, "nq": nq, "n": n, "d": d, "k": k,
                          "ms_median": round(t, 3), "ms_all": [round(v, 3) for v in ts],
                          "over_f32_row_ms": round(t - meds[0], 3)}), flush=True)


if __name__ == "__main__":
    main()
