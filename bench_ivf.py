#!/usr/bin/env python
"""bench_ivf.py -- secondary benchmark lines for the IVF rows of the hot path (not the driver's
headline; bench.py is).  BASELINE.json configs[3]: GpuIndexIVFPQ N=100M d=128 nlist=4096 m=32
nbits=8 nprobe=32 nq=10k k=100; configs[2]: GpuIndexIVFFlat N=10M nlist=4096 nprobe=64.

  python bench_ivf.py --index ivfpq  [--n 100000000] [--steps 5] [--nbits 4 --m 64]
  python bench_ivf.py --index ivfflat [--n 10000000]
  python bench_ivf.py --index ivfsq --qtype 8bit   (IVF-Flat config; --qtype one of QTYPES)

--nbits 4/5/6 builds the IVF-PQ index with interleaved_layout (4-bit with M in {32, 64}: the nibble-pair scan,
kernel "ivfpq_scan"; other shapes: the packed scan, kernel "ivfpq_scan_packed").  --dump-outputs DIR writes the
last timed step's result (distances.npy, labels.npy), as bench.py does.

Prints one JSON line: QPS (device-resident queries), e2e QPS (host buffers), and the HBM roofline of
the scan kernel: algorithmic bytes = sum over (query, probe) of listLen * code_size, divided by the
scan kernel's CUDA-event time, against MEASURED_PEAKS.json hbm_gbs.  Queries share probed lists, so
L2 reuse can push the achieved rate past 100% of the HBM peak.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


QTYPES = {"8bit": 0, "4bit": 1, "8bit_uniform": 2, "4bit_uniform": 3, "fp16": 4, "8bit_direct": 5, "6bit": 6}


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--index", default="ivfpq", choices=["ivfpq", "ivfflat", "ivfsq"])
    ap.add_argument("--qtype", default="8bit", choices=sorted(QTYPES), help="ScalarQuantizer type (--index ivfsq)")
    ap.add_argument("--n", type=int, default=None)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--m", type=int, default=32)
    ap.add_argument("--nbits", type=int, default=8, help="bits per PQ code (--index ivfpq)")
    ap.add_argument("--nprobe", type=int, default=None)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ntrain", type=int, default=1 << 20)
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's distances and labels as DIR/<name>.npy")
    ap.add_argument("--recall-queries", type=int, default=100, help="queries checked against exact fp32 ground truth (0 = skip)")
    args = ap.parse_args()
    N = args.n or (100_000_000 if args.index == "ivfpq" else 10_000_000)
    nprobe = args.nprobe or (32 if args.index == "ivfpq" else 64)
    d, nq, k = args.d, args.nq, args.k

    import torch

    import faiss_b200 as fb
    from bench import ClockSampler, peaks

    assert torch.cuda.is_available()
    dev = torch.device("cuda", 0)
    res = fb.StandardGpuResources()
    res.setDefaultStream(0, torch.cuda.current_stream(dev).cuda_stream)

    def gen(n, seed):
        g = torch.Generator(device=dev)
        g.manual_seed(seed)
        return torch.rand((n, d), dtype=torch.float32, device=dev, generator=g)

    if args.index == "ivfpq":
        if args.nbits == 8:
            index = fb.GpuIndexIVFPQ(res, d, args.nlist, args.m, 8, fb.METRIC_L2)
        else:
            index = fb.GpuIndexIVFPQ(res, d, args.nlist, args.m, args.nbits, fb.METRIC_L2, interleaved_layout=True)
        code_size = (args.m * args.nbits + 7) // 8
        nibble_pairs = args.nbits == 4 and args.m in (32, 64)
        kname = b"ivfpq_scan" if args.nbits == 8 or nibble_pairs else b"ivfpq_scan_packed"
    elif args.index == "ivfflat":
        index = fb.GpuIndexIVFFlat(res, d, args.nlist, fb.METRIC_L2)
        code_size = 4 * d
        kname = b"ivfflat_scan"
    elif args.index == "ivfsq":
        index = fb.GpuIndexIVFScalarQuantizer(res, d, args.nlist, QTYPES[args.qtype], fb.METRIC_L2)
        code_size = index.code_size
        kname = b"ivfsq_scan"
    t0 = time.time()
    xt = gen(min(args.ntrain, N), 4321)
    index.train(xt)
    del xt
    torch.cuda.synchronize()
    t_train = time.time() - t0
    log("trained in %.1f s" % t_train)
    t0 = time.time()
    index.reserveMemory(N + N // 8)
    CH = 1_000_000
    for c0 in range(0, N, CH):
        xb = gen(min(CH, N - c0), 1234 + c0 // CH)
        index.add(xb)
        del xb
    torch.cuda.synchronize()
    t_add = time.time() - t0
    log("added %d vectors in %.1f s (%.0f vec/s)" % (N, t_add, N / t_add))
    index.nprobe = nprobe
    xq = gen(nq, 1235)
    xq_pin = torch.empty((nq, d), dtype=torch.float32, pin_memory=True)
    xq_pin.copy_(xq)
    D_pin = torch.empty((nq, k), dtype=torch.float32, pin_memory=True)
    I_pin = torch.empty((nq, k), dtype=torch.int64, pin_memory=True)

    lens = np.array([index.getListLength(l) for l in range(args.nlist)], dtype=np.int64)

    for _ in range(max(3, args.warmup)):
        D, I = index.search(xq, k)
    torch.cuda.synchronize()
    # algorithmic bytes of one step: probed list lengths x code size
    cent = torch.from_numpy(index.getCoarseCentroids()).to(dev)
    probes = torch.cdist(xq, cent).topk(nprobe, dim=1, largest=False).indices.cpu().numpy()
    scanned = int(lens[probes].sum())
    alg_bytes = scanned * code_size

    sampler = ClockSampler(0)
    sampler.start()
    fb.lib.faiss_b200_kernel_timing(1)
    l0 = fb.lib.faiss_b200_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.steps):
        D, I = index.search(xq, k)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    launches = fb.lib.faiss_b200_launch_count() - l0
    kms, kn = ctypes.c_double(), ctypes.c_int()
    fb.lib.faiss_b200_kernel_timing_collect(kname, ctypes.byref(kms), ctypes.byref(kn))
    fb.lib.faiss_b200_kernel_timing(0)
    clocks = sampler.stop()
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "distances.npy"), D.cpu().numpy().astype(np.float32))
        np.save(os.path.join(args.dump_outputs, "labels.npy"), I.cpu().numpy().astype(np.float64))  # ids < 2^53: exact

    for _ in range(2):
        index.search(xq_pin.numpy(), k, D=D_pin.numpy(), I=I_pin.numpy())
    t0 = time.time()
    for _ in range(args.steps):
        index.search(xq_pin.numpy(), k, D=D_pin.numpy(), I=I_pin.numpy())
    e2e_ms = (time.time() - t0) * 1e3 / args.steps

    # recall vs exact ground truth on a query subset: the database is regenerated chunk by chunk (same
    # seeds as the add loop), each chunk searched exactly (fp32 SIMT kernel), chunk results merged
    recall = None
    if args.recall_queries > 0:
        nr = min(args.recall_queries, nq)
        bestD = torch.full((nr, k), float("inf"), device=dev)
        bestI = torch.full((nr, k), -1, dtype=torch.int64, device=dev)
        for c0 in range(0, N, CH):
            xb = gen(min(CH, N - c0), 1234 + c0 // CH)
            cD, cI = fb.flat_search_exact(res, xb, xq[:nr].contiguous(), k)
            allD = torch.cat([bestD, cD], dim=1)
            allI = torch.cat([bestI, cI + c0], dim=1)
            o_ = torch.argsort(allD, dim=1, stable=True)[:, :k]
            bestD, bestI = torch.gather(allD, 1, o_), torch.gather(allI, 1, o_)
            del xb
        D, I = index.search(xq[:nr].contiguous(), k)
        inter = sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(I.cpu().numpy(), bestI.cpu().numpy()))
        r1 = float((I[:, :k] == bestI[:, :1]).any(dim=1).float().mean())
        recall = {"queries": nr, "intersection_recall_at_k": inter / float(nr * k), "recall_1_at_k": r1,
                  "note": "vs exact fp32 ground truth; uniform random d=%d data is a worst case for IVF/PQ recall (SURVEY 8d)" % d}

    pk, src = peaks()
    roof = {"bound": "hbm", "unit": "GB/s", "peak": float(pk["hbm_gbs"]), "peak_source": src + " copy bandwidth (MEASURED_PEAKS.json)",
            "traffic": None, "algorithmic_bytes_per_step": alg_bytes, "vectors_scanned_per_step": scanned}
    if kn.value:
        kms_step = kms.value / args.steps
        roof.update({"achieved": alg_bytes / (kms_step * 1e-3) / 1e9, "kernel_ms_per_step": kms_step, "kernel_share_of_step": kms_step / ms})
        roof["frac"] = roof["achieved"] / roof["peak"]
    out = {"metric": "queries/sec (%s)" % args.index, "value": nq / (ms * 1e-3), "unit": "queries/s", "n_gpus": 1, "steps": args.steps,
           "warmup": max(3, args.warmup), "ms_per_step": ms, "higher_is_better": True, "dtype": {"ivfpq": "%d-bit codes, f32 LUT" % args.nbits if args.nbits != 8 else "u8 codes, f32 LUT", "ivfflat": "f32", "ivfsq": "SQ %s codes" % args.qtype}[args.index],
           "data": "synthetic", "config": {"workload": "%s N=%d d=%d nlist=%d %snprobe=%d nq=%d k=%d" % (
               args.index, N, d, args.nlist, ("M=%d nbits=%d " % (args.m, args.nbits)) if args.index == "ivfpq" else ("qtype=%s " % args.qtype) if args.index == "ivfsq" else "", nprobe, nq, k),
               "list_len_mean": float(lens.mean()), "list_len_max": int(lens.max()), "train_s": t_train, "add_s": t_add, "add_vec_per_s": N / t_add},
           "clocks": clocks, "e2e": {"value": nq / (e2e_ms * 1e-3), "unit": "queries/s", "ms_per_step": e2e_ms,
                                     "h2d_bytes_per_step": nq * d * 4, "d2h_bytes_per_step": nq * k * 12},
           "gpu_launches": int(launches), "roofline": roof, "recall": recall}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
