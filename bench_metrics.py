"""Benchmark of GpuIndexFlat's extra metrics (L1, Linf, Lp, Canberra, BrayCurtis, JensenShannon, Jaccard, Gower)
on the exact SIMT kernel, against the exact L2 kernel of the same build as a yardstick.

    python bench_metrics.py [--n 1000000] [--d 128] [--k 100] [--reps 5] [--metrics L1,Linf,...]

Shape: N database rows, d = 128, k = 100, queries and outputs resident on the device.  L1, Linf, BrayCurtis
and Jaccard run nq = 10000 queries; the ops with a transcendental or a division per component (Lp with p = 3,
Canberra, JensenShannon) and Gower's branches run nq = 1000.  Each metric's timed calls alternate with calls of
the exact L2 kernel (use_tensor_cores=False) at the same nq.

Per metric, one JSON line: the median of --reps timed calls after a warm-up call (CUDA events around
index.search: the exact kernel plus the merge of the database split), component evaluations per second
(nq * N * d / t), and for L1 and the L2 yardstick -- the two ops whose instruction count is known, two FP32
instructions per component -- the share of the data-sheet FP32 issue rate (67 TFLOP/s = 33.5e12 FP32
instructions/s on the H100 SXM at 700 W).  The card's name and power limit are read in the same run.  Each line
checks its own result on 32 queries against the reference CPU IndexFlat of the same metric (oracle/_ref, or the
numpy restatement where it was not built) with compare_lists.
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

FP32_INSTR_PER_S = 33.5e12  # H100 SXM data sheet: 67 TFLOP/s FP32 = 33.5e12 FMA-pipe instructions/s

# name -> (metric, metric_arg, nq, FP32 instructions per component or None)
METRICS = {
    "L1": (2, 0.0, 10000, 2),
    "Linf": (3, 0.0, 10000, None),
    "Lp3": (4, 3.0, 1000, None),
    "Canberra": (20, 0.0, 1000, None),
    "BrayCurtis": (21, 0.0, 10000, None),
    "JensenShannon": (22, 0.0, 1000, None),
    "Jaccard": (23, 0.0, 10000, None),
    "Gower": (25, 0.0, 1000, None),
}


def gpu_identity(gpu_index=0):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        name, plim, smax = [x.strip() for x in r.stdout.strip().split(",")[:3]]
        return {"name": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax)}
    except Exception as e:
        return {"error": str(e)[:100]}


def make_rows(torch, n, d, metric, gen):
    """positive floats in [0.05, 1.05) (every metric's domain); Gower: even columns numeric in [0, 1), odd columns
    categorical in {-1, -2, -3}"""
    x = torch.rand((n, d), generator=gen, device="cuda") + 0.05
    if metric == 25:
        x[:, 0::2] -= 0.05
        x[:, 1::2] = -torch.floor(x[:, 1::2] * 2.9 + 1)
    return x.contiguous()


def timed(torch, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def parity(fb_metric, arg, xb, xq, D, I, k):
    from oracle import oracle_metrics_np as m
    from oracle import oracle_np as o
    from oracle import ref_metrics

    if ref_metrics.available():
        idx = ref_metrics.IndexFlat(xb.shape[1], fb_metric, arg)
        idx.add(xb)
        rD, rI = idx.search(xq, k)
        src = "oracle/_ref IndexFlat"
    else:
        rD, rI = m.knn_extra(xq, xb, k, fb_metric, arg, block=4)
        src = "numpy knn_extra"
    try:
        st = o.compare_lists(rD, rI, D, I, eps=1e-4, pct_max_diff1=0.01, pct_max_diffN=0.002)
        return {"parity": "ok", "parity_vs": src, "max_rel_err": st["max_rel_err"]}
    except AssertionError as e:
        return {"parity": "FAIL: %s" % e, "parity_vs": src}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--metrics", default=",".join(METRICS))
    ap.add_argument("--nq-scale", type=float, default=1.0, help="multiply every nq (smaller dry runs)")
    args = ap.parse_args()

    import torch

    import faiss_b200 as fb

    if not torch.cuda.is_available():
        sys.exit("bench_metrics.py needs a CUDA device")
    card = gpu_identity(torch.cuda.current_device())
    print(json.dumps({"card": card, "n": args.n, "d": args.d, "k": args.k, "reps": args.reps}), flush=True)
    res = fb.StandardGpuResources()
    dev = torch.cuda.current_device()
    res.setDefaultStream(dev, torch.cuda.current_stream(dev).cuda_stream)
    n, d, k = args.n, args.d, args.k
    gen = torch.Generator(device="cuda")

    for name in args.metrics.split(","):
        metric, arg, nq, instr = METRICS[name]
        nq = max(32, int(nq * args.nq_scale))
        gen.manual_seed(1234)
        xb = make_rows(torch, n, d, metric, gen)
        xq = make_rows(torch, nq, d, metric, gen)
        idx = fb.GpuIndexFlat(res, d, metric, use_tensor_cores=False)
        idx.metric_arg = arg
        idx.add(xb)
        # the yardstick: the exact L2 SIMT kernel over the same rows and queries
        l2 = fb.GpuIndexFlat(res, d, fb.METRIC_L2, use_tensor_cores=False)
        l2.add(xb)
        D = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        I = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        D2, I2 = torch.empty_like(D), torch.empty_like(I)
        run = lambda: idx.search(xq, k, D, I)  # noqa: E731
        run_l2 = lambda: l2.search(xq, k, D2, I2)  # noqa: E731
        run()  # warm-up, every shape of the timed window
        run_l2()
        torch.cuda.synchronize()
        ts, ts_l2 = [], []
        for _ in range(args.reps):
            ts.append(timed(torch, run))
            ts_l2.append(timed(torch, run_l2))
        assert idx.lastSearchInfo()["tensor_cores"] == 0 and l2.lastSearchInfo()["tensor_cores"] == 0
        t, t2 = float(np.median(ts)), float(np.median(ts_l2))
        evals = float(nq) * n * d
        line = {
            "metric": name, "nq": nq, "n": n, "d": d, "k": k,
            "ms_median": round(t, 3), "ms_all": [round(v, 3) for v in ts],
            "component_evals_per_s": evals / (t * 1e-3),
            "l2_exact_ms_median": round(t2, 3), "l2_exact_ms_all": [round(v, 3) for v in ts_l2],
            "ratio_to_l2_exact": round(t / t2, 4),
            "l2_exact_fp32_share": round(2 * evals / (t2 * 1e-3) / FP32_INSTR_PER_S, 4),
        }
        if instr is not None:
            line["fp32_share"] = round(instr * evals / (t * 1e-3) / FP32_INSTR_PER_S, 4)
        line.update(parity(metric, arg, xb.cpu().numpy(), xq[:32].cpu().numpy(), D[:32].cpu().numpy(),
                           I[:32].cpu().numpy(), k))
        line["card"] = card.get("name")
        line["power_limit_w"] = card.get("power_limit_w")
        print(json.dumps(line), flush=True)
        del idx, l2, xb, xq
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
