"""GpuRqEncoder benchmark: ResidualQuantizer's compute_codes (beam search + pack) of n = 1M SyntheticDataset rows at
d = 128, M = 8, nbits = 8, with max_beam_size 5 and 32, in both distance modes, in one call each.

    python bench_rq.py [--n 1000000] [--subset 2000]

Per (mode, beam) it reports, from CUDA events, the precompute (the runFlatPairwise inner products and runL2Norms),
the beam kernels (rq_beam_step_kernel in mode 0, rq_beam_lut_kernel in mode 1) and rq_pack_kernel, the whole encode
and vectors/s.  Work is computed from shapes:
  mode 0  GEMM FLOPs 2·n·Σ B_in·K·d (fp32 SIMT: bound by the 67 TFLOP/s fp32 rate) and step-kernel bytes
          n·Σ (B_in·K + 2·B_out·d)·4 (the inner-product matrix and the residuals: an HBM stream);
  mode 1  GEMM FLOPs 2·n·total_K·d, and the LUT kernel's cross-table reads n·Σ B_in·K·m·4 (an L2 rate: the table is
          7.3 MB).
The codebooks are greedy residual codebooks built on the device (each level: K random rows of the previous level's
residuals), which is enough to time the encoder.  The reference CPU encoder runs on a subset at several OpenMP thread
counts, scaled to n; the parity line is the share of subset rows whose packed codes equal the CPU's.  Prints one JSON
line; writes nothing.
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
from oracle import ref_rq

D, M, NBITS, K = 128, 8, 8, 256


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _collect(name):
    ms, cnt = ctypes.c_double(), ctypes.c_int()
    fb.check(fb.lib.faiss_b200_kernel_timing_collect(name.encode(), ctypes.byref(ms), ctypes.byref(cnt)))
    return ms.value / 1e3


def _codebooks(xt):
    rs = np.random.RandomState(0)
    r = torch.from_numpy(xt).cuda()
    cbs = []
    for _ in range(M):
        c = r[torch.from_numpy(rs.choice(r.shape[0], K, replace=False)).cuda()]
        a = ((c * c).sum(1)[None] - 2 * r @ c.T).argmin(1)
        r = r - c[a]
        cbs.append(c)
    return torch.cat(cbs).cpu().numpy()


def _work(n, lut, beam):
    flops, step_bytes, lut_bytes, b = 0, 0, 0, 1
    for m in range(M):
        bo = min(b * K, beam)
        if lut:
            lut_bytes += n * b * K * m * 4
        else:
            flops += 2 * n * b * K * D
            step_bytes += n * (b * K + 2 * bo * D) * 4
        b = bo
    if lut:
        flops = 2 * n * M * K * D
    return flops, step_bytes, lut_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--subset", type=int, default=2000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rq.py needs a GPU"
    n = a.n
    out = {"card": _card(), "d": D, "M": M, "nbits": NBITS, "n": n, "runs": []}
    xt, xb, _ = synthetic_dataset(D, 20000, n, 0)
    cb = _codebooks(xt)
    res = fb.StandardGpuResources()
    enc = fb.GpuRqEncoder(D, [NBITS] * M, res)
    enc.setCodebooks(cb)
    x_t = torch.from_numpy(xb).cuda()
    for lut in (0, 1):
        for beam in (5, 32):
            enc.computeCodes(x_t[:2000], lut, beam)  # warm-up of the shapes the timed call uses
            torch.cuda.synchronize()
            fb.lib.faiss_b200_kernel_timing(1)
            t0 = time.perf_counter()
            got = enc.computeCodes(x_t, lut, beam)
            torch.cuda.synchronize()
            t_enc = time.perf_counter() - t0
            fb.lib.faiss_b200_kernel_timing(0)
            t_gemm, t_step, t_lut, t_pack = (_collect(k) for k in ("rq_gemm", "rq_step", "rq_lut", "rq_pack"))
            flops, step_bytes, lut_bytes = _work(n, lut, beam)
            run = {"use_beam_LUT": lut, "max_beam_size": beam, "precompute_s": t_gemm, "beam_kernel_s": t_lut if lut else t_step,
                   "pack_s": t_pack, "encode_s": t_enc, "vectors_per_s": n / t_enc,
                   "precompute_TFLOP_per_s": flops / t_gemm / 1e12}
            if lut:
                run["lut_cross_reads_L2_TB_per_s"] = lut_bytes / t_lut / 1e12
            else:
                run["step_HBM_TB_per_s"] = step_bytes / t_step / 1e12
            out["runs"].append(run)
            del got

    # the reference CPU encoder on a subset, on the same codebooks, at several thread counts
    s = a.subset
    xs = xb[:s]
    if ref_rq.available():
        cpu_rows, parity = [], []
        for lut in (0, 1):
            for beam in (5, 32):
                q = ref_rq.RQ(D, [NBITS] * M, cb, max_beam_size=beam, use_beam_LUT=lut)
                for th in sorted({1, 8, os.cpu_count() or 1}):
                    ref_rq.set_threads(th)
                    t0 = time.perf_counter()
                    cpu = q.compute_codes(xs)
                    dt = time.perf_counter() - t0
                    cpu_rows.append({"use_beam_LUT": lut, "max_beam_size": beam, "threads": th, "subset": s,
                                     "scaled_to_n_s": dt * n / s})
                gpu = enc.computeCodes(xs, lut, beam)
                parity.append({"use_beam_LUT": lut, "max_beam_size": beam,
                               "identical_code_rows": float((gpu == cpu).all(1).mean())})
        out["cpu_reference"] = cpu_rows
        out["parity"] = parity
    else:
        out["parity"] = {"reason": "reference shim not built"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
