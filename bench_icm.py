"""GpuIcmEncoder benchmark: LocalSearchQuantizer's ICM encoding of n = 100k and 1M SyntheticDataset rows at d = 128,
M = 8, K = 256, encode_ils_iters = 16, icm_iters = 4, nperts = 4 (the reference's defaults), in one call.

    python bench_icm.py [--n 100000 1000000] [--subset 4000]

Per n it reports the host draws (std::mt19937 through the reference shim), the device precompute (x·Cᵀ) and the fused
kernel from CUDA events, vectors/s of the whole encode, and the rate at which the kernel gathers binary-term rows
(n·ils·icm_iters·M·(M-1)·K·4 bytes over kernel time; the C·Cᵀ table is 16 MB, so this is an L2 rate, not an HBM rate).
The reference CPU encoder runs on a subset at several OpenMP thread counts, scaled to n.  The parity line compares the
subset's codes with the CPU encoder's, fed the same draws.  Prints one JSON line; writes nothing.
"""
import argparse
import ctypes
import json
import os
import subprocess
import time

import numpy as np
import torch

import faiss_b200 as fb
from bench import synthetic_dataset
from oracle import oracle_lsq_np as lo
from oracle import ref_lsq

M, K, D, ILS, ICM, NPERTS, SEED = 8, 256, 128, 16, 4, 4, 0x12345


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _collect(name):
    ms, cnt = ctypes.c_double(), ctypes.c_int()
    fb.check(fb.lib.faiss_b200_kernel_timing_collect(name.encode(), ctypes.byref(ms), ctypes.byref(cnt)))
    return ms.value / 1e3


def _codebooks(xt):
    # additive codebooks: each level is K rows of the previous level's residuals, assigned with one matmul
    rs = np.random.RandomState(0)
    r = torch.from_numpy(xt).cuda()
    cbs = []
    for _ in range(M):
        c = r[torch.from_numpy(rs.choice(r.shape[0], K, replace=False)).cuda()]
        a = ((c * c).sum(1)[None] - 2 * r @ c.T).argmin(1)
        r = r - c[a]
        cbs.append(c)
    return torch.stack(cbs).cpu().numpy()


def _draws(n, seed):
    if ref_lsq.available():
        return ref_lsq.draws(M, K, NPERTS, n, ILS, seed)[0]
    return lo.draws(lo.MT19937(seed), M, K, NPERTS, n, ILS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--subset", type=int, default=4000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_icm.py needs a GPU"
    out = {"card": _card(), "d": D, "M": M, "K": K, "ils_iters": ILS, "icm_iters": ICM, "nperts": NPERTS,
           "draws_from": "reference std::mt19937" if ref_lsq.available() else "numpy restatement"}
    nmax = max(a.n)
    xt, xb, _ = synthetic_dataset(D, 20000, nmax, 0)
    cb = _codebooks(xt)
    res = fb.StandardGpuResources()
    enc = fb.GpuIcmEncoder(M, K, D, res)
    enc.setBinaryTerm(cb)
    codes_all = np.random.RandomState(1).randint(0, K, (nmax, M)).astype(np.int32)

    # warm-up of every shape the timed runs use
    w = 2000
    enc.encode(torch.from_numpy(codes_all[:w]).cuda(), torch.from_numpy(xb[:w]).cuda(), torch.from_numpy(_draws(w, 1)).cuda(), icm_iters=ICM)
    torch.cuda.synchronize()

    out["runs"] = []
    for n in a.n:
        t0 = time.perf_counter()
        perts = _draws(n, SEED)
        t_draws = time.perf_counter() - t0
        x_t = torch.from_numpy(xb[:n]).cuda()
        c_t = torch.from_numpy(codes_all[:n]).cuda()
        p_t = torch.from_numpy(perts).cuda()
        del perts
        torch.cuda.synchronize()
        fb.lib.faiss_b200_kernel_timing(1)
        t0 = time.perf_counter()
        got = enc.encode(c_t, x_t, p_t, icm_iters=ICM)
        torch.cuda.synchronize()
        t_enc = time.perf_counter() - t0
        fb.lib.faiss_b200_kernel_timing(0)
        t_pre, t_ker = _collect("icm_unary"), _collect("icm_encode")
        gather = n * ILS * ICM * M * (M - 1) * K * 4
        out["runs"].append({
            "n": n, "host_draws_s": t_draws, "precompute_s": t_pre, "kernel_s": t_ker, "encode_s": t_enc,
            "vectors_per_s": n / t_enc, "binary_gather_L2_GB_per_s": gather / t_ker / 1e9,
        })
        del x_t, c_t, p_t, got
        torch.cuda.empty_cache()

    # the reference CPU encoder on a subset, fed the same draws (std::mt19937(SEED)), at several thread counts
    s = a.subset
    xs, cs = xb[:s], codes_all[:s]
    gpu = enc.encode(cs, xs, _draws(s, SEED), icm_iters=ICM)
    err_gpu = float(lo.evaluate(cb, gpu, xs).astype(np.float64).sum())
    if ref_lsq.available():
        q = ref_lsq.LSQ(cb, nperts=NPERTS, icm_iters=ICM)
        cpu_rows = []
        for th in sorted({1, 8, os.cpu_count() or 1}):
            ref_lsq.set_threads(th)
            t0 = time.perf_counter()
            cpu, _ = q.icm_encode(cs, xs, ILS, SEED)
            dt = time.perf_counter() - t0
            cpu_rows.append({"threads": th, "subset": s, "subset_s": dt, "scaled_to_1M_s": dt * 1e6 / s})
        out["cpu_reference"] = cpu_rows
        err_cpu = float(lo.evaluate(cb, cpu, xs).astype(np.float64).sum())
        same = float((gpu == cpu).all(1).mean())
        ratio = err_gpu / err_cpu
        out["parity"] = {"subset": s, "identical_code_rows": same, "error_ratio_gpu_over_cpu": ratio,
                         "ok": bool(abs(ratio - 1) <= 1e-3)}
    else:
        out["parity"] = {"ok": False, "reason": "reference shim not built"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
