"""GpuIndexCagra benchmark: build time by stage, then search QPS, recall@10, distance evaluations and gathered bytes
per second at itopk_size 32 ... 256, beside GpuIndexIVFPQ / GpuIndexIVFFlat on the same data, in one call.

    python bench_cagra.py [--n 1000000] [--d 128] [--nq 10000] [--k 10]

Data: bench.synthetic_dataset (SyntheticDataset restated).  Ground truth: GpuIndexFlatL2.  Queries and results stay
on the device during the timed searches.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

import faiss_b200 as fb
from bench import synthetic_dataset


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _recall(I, gt, k):
    I = I[:, :k]
    gt = gt[:, :k]
    return float(np.mean([len(np.intersect1d(a, b)) for a, b in zip(I, gt)]) / k)


def _timed(fn, min_seconds=1.0):
    fn()  # warm-up of the shape
    torch.cuda.synchronize()
    reps, t = 0, 0.0
    t0 = time.perf_counter()
    while t < min_seconds:
        out = fn()
        torch.cuda.synchronize()
        reps += 1
        t = time.perf_counter() - t0
    return t / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_cagra.py needs a GPU"
    out = {"card": _card(), "n": a.n, "d": a.d, "nq": a.nq, "k": a.k}

    _, xb, xq = synthetic_dataset(a.d, 0, a.n, a.nq)
    res = fb.StandardGpuResources()
    xb_t = torch.from_numpy(xb).cuda()
    xq_t = torch.from_numpy(xq).cuda()

    flat = fb.GpuIndexFlatL2(res, a.d)
    flat.add(xb_t)
    _, gt = flat.search(xq_t, a.k)
    gt = gt.cpu().numpy()
    del flat

    index = fb.GpuIndexCagra(res, a.d, fb.METRIC_L2)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    index.train(xb_t)
    torch.cuda.synchronize()
    out["build_s"] = time.perf_counter() - t0
    out["build_stages_s"] = index.lastBuildSeconds()
    out["graph_degree"] = index.graph_degree

    out["cagra"] = []
    for itopk in (32, 64, 128, 256):
        p = fb.SearchParametersCagra(itopk_size=itopk)
        dt, (_, I) = _timed(lambda: index.search(xq_t, a.k, params=p))
        evals = index.lastSearchDistanceCount()
        out["cagra"].append({
            "itopk_size": itopk,
            "qps": a.nq / dt,
            "recall@10": _recall(I.cpu().numpy(), gt, a.k),
            "distances_per_query": evals / a.nq,
            "gathered_GB_per_s": evals * a.d * 4 / dt / 1e9,
        })

    nlist = 4096
    for name, make in (("ivfpq_M32", lambda: fb.GpuIndexIVFPQ(res, a.d, nlist, 32, 8)),
                       ("ivfflat", lambda: fb.GpuIndexIVFFlat(res, a.d, nlist))):
        ivf = make()
        ivf.train(xb_t)
        ivf.add(xb_t)
        rows = []
        for nprobe in (16, 64):
            ivf.nprobe = nprobe
            dt, (_, I) = _timed(lambda: ivf.search(xq_t, a.k))
            rows.append({"nprobe": nprobe, "qps": a.nq / dt, "recall@10": _recall(I.cpu().numpy(), gt, a.k)})
        out[name] = rows
        del ivf
    print(json.dumps(out))


if __name__ == "__main__":
    main()
