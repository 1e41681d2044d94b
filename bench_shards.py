#!/usr/bin/env python
"""bench_shards.py -- BASELINE configs[4] in the shape the box allows: IVFPQ sharded over the GPUs of
one node (IndexShards semantics), coarse quantiser trained by sharded k-means.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
      bench_shards.py --gpus N [--ntotal 1000000000 --d 96 --nlist 65536 --m 32 --nprobe 32]

One process per GPU.  Per rank: its contiguous slice of the database and of the training set.
  * train: `faiss_b200.kmeans_sharded` (C++, faiss_b200_kmeans_sharded) -- Flat k=1 assignment on the wgmma
    streaming path against the replicated centroid table, deterministic local partial sums, ONE packed NCCL
    all-reduce per iteration (k*d sums | k counts | objective); PQ codebooks trained on rank 0's residuals and broadcast.
  * add: device-side assign -> residual -> PQ encode -> append, shard-local ids.
  * search: every query to every shard, ONE all-gather of the per-shard [nq, k] (fp32 | int64) + device
    merge (`DistributedIndexShards`, NCCL communicator owned by the C++ resources), ids translated like successive_ids.
Prints one JSON line (rank 0).  configs[4] itself is N=1e9 on 8 GPUs (125M vectors per GPU); the defaults
here are sized per GPU the same way (--ntotal defaults to 125M x world).
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


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--ntotal", type=int, default=None)
    ap.add_argument("--d", type=int, default=96)
    ap.add_argument("--nlist", type=int, default=65536)
    ap.add_argument("--m", type=int, default=32)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--niter", type=int, default=10)
    ap.add_argument("--ppc", type=int, default=256, help="training points per centroid (reference max_points_per_centroid)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    # NCCL prints its version banner to stdout when the first communicator is created: keep stdout to
    # the one JSON line by creating it with fd 1 -> fd 2
    sys.stdout.flush()
    saved = os.dup(1)
    os.dup2(2, 1)
    try:
        dist.init_process_group("nccl", device_id=dev)
        dist.all_reduce(torch.zeros(1, device=dev))
        torch.cuda.synchronize()
    finally:
        os.dup2(saved, 1)
        os.close(saved)

    import faiss_b200 as fb
    from bench import ClockSampler, peaks
    from faiss_b200.distributed import merge_host, shard_bounds

    N = args.ntotal or 125_000_000 * world
    d, nlist, M, nq, k = args.d, args.nlist, args.m, args.nq, args.k
    res = fb.StandardGpuResources()
    res.setDefaultStream(local_rank, torch.cuda.current_stream(dev).cuda_stream)
    # the search path's NCCL communicator belongs to the library's resources object (C++); torch.distributed hands
    # the 128-byte id around and serves the Python-level k-means all-reduce
    ids = [fb.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0, device=dev)
    res.ncclInitRank(local_rank, world, rank, ids[0])

    CH = 1_000_000

    def gen(r0, r1, seed0):
        """rows [r0, r1) of a stream generated in seeded 1M-row chunks (independent of the world size)"""
        out = torch.empty((r1 - r0, d), dtype=torch.float32, device=dev)
        c = r0 // CH
        while c * CH < r1:
            g = torch.Generator(device=dev)
            g.manual_seed(seed0 + c)
            chunk = torch.rand((CH, d), dtype=torch.float32, device=dev, generator=g)
            a, b = max(r0, c * CH), min(r1, (c + 1) * CH)
            out[a - r0 : b - r0] = chunk[a - c * CH : b - c * CH]
            del chunk
            c += 1
        return out

    # ---------------------------------------------------------------- sharded k-means (coarse quantiser)
    n_train = min(N, nlist * args.ppc)
    t0, t1 = shard_bounds(n_train, rank, world)
    xt = gen(t0, t1, 500_000)
    torch.cuda.synchronize()
    dist.barrier()
    tt = time.time()
    # C++ sharded k-means behind the C ABI: local wgmma k=1 assignment (streaming mode), deterministic local
    # partial sums, ONE packed ncclAllReduce per iteration on the library's own communicator
    cent_np, objs, kstats = fb.kmeans_sharded(res, xt, nlist, niter=args.niter, seed=1234, device=local_rank)
    cent = torch.from_numpy(cent_np).to(dev)
    torch.cuda.synchronize()
    dist.barrier()
    train_s = time.time() - tt
    if rank == 0:
        log("[rank %d] k-means %d x %d-d on %d points (%d local): %.2f s, objective %.4g -> %.4g, %s" % (
            rank, nlist, d, n_train, t1 - t0, train_s, objs[0], objs[-1], kstats))
    assert all(objs[i + 1] <= objs[i] * 1.0001 for i in range(len(objs) - 1)), "objective must not increase"

    # ---------------------------------------------------------------- PQ codebooks: rank 0 trains, broadcast
    index = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, fb.METRIC_L2, device=local_rank)
    index.setCoarseCentroids(cent.cpu().numpy())
    pq = torch.empty((M, 256, d // M), dtype=torch.float32, device=dev)
    if rank == 0:
        index.setPQClustering(niter=10)
        index.train(xt[: min(xt.shape[0], 1 << 18)])
        pq.copy_(torch.from_numpy(index.getPQCentroids().reshape(M, 256, d // M)))
    dist.broadcast(pq, src=0)
    if rank != 0:
        index.setPQCentroids(pq.cpu().numpy())
        index.setIsTrained(True)
    del xt

    # ---------------------------------------------------------------- add this rank's shard
    r0, r1 = shard_bounds(N, rank, world)
    torch.cuda.synchronize()
    ta = time.time()
    index.reserveMemory((r1 - r0) + (r1 - r0) // 8)
    for c0 in range(r0, r1, 2 * CH):
        xb = gen(c0, min(r1, c0 + 2 * CH), 1234)
        index.add(xb)
        del xb
    torch.cuda.synchronize()
    add_s = time.time() - ta
    dist.barrier()
    log("[rank %d] added rows [%d,%d) in %.1f s (%.1f M vec/s)" % (rank, r0, r1, add_s, (r1 - r0) / add_s / 1e6))
    index.nprobe = args.nprobe

    g = torch.Generator(device=dev)
    g.manual_seed(1235)
    xq = torch.rand((nq, d), dtype=torch.float32, device=dev, generator=g)
    # IndexShards with one shard per rank behind the C ABI: ONE grouped ncclAllGather + device merge
    searcher = fb.DistributedIndexShards(res, index, successive_ids=True)
    assert searcher.ntotal == N, (searcher.ntotal, N)

    for _ in range(max(3, args.warmup)):
        D, I = searcher.search(xq, k)
    torch.cuda.synchronize()
    assert bool((D[:, 1:] >= D[:, :-1]).all()) and bool(((I >= 0) & (I < N)).all())

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    fb.lib.faiss_b200_kernel_timing(1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dist.barrier()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.steps):
        D, I = searcher.search(xq, k)
    e1.record()
    torch.cuda.synchronize()
    dist.barrier()
    ms = e0.elapsed_time(e1) / args.steps
    kms, kn = ctypes.c_double(), ctypes.c_int()
    fb.lib.faiss_b200_kernel_timing_collect(b"ivfpq_scan", ctypes.byref(kms), ctypes.byref(kn))
    fb.lib.faiss_b200_kernel_timing(0)
    t = torch.tensor([ms, kms.value / args.steps], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, scan_ms = float(t[0]), float(t[1])
    # algorithmic bytes of this rank's scan: probed list lengths x M
    lens = np.array([index.getListLength(l) for l in range(nlist)], dtype=np.int64)
    cent_d = cent
    probes = torch.cdist(xq, cent_d).topk(args.nprobe, dim=1, largest=False).indices.cpu().numpy()
    scanned = torch.tensor([float(lens[probes].sum())], dtype=torch.float64, device=dev)
    dist.all_reduce(scanned, op=dist.ReduceOp.SUM)
    # ---- parity of the collective path (outside the timed region): the merged result of a query sample must equal
    # the reference merge rule (merge_knn_results semantics, host) applied to every rank's LOCAL result
    ns = min(nq, 256)
    lD, lI = index.search(xq[:ns].contiguous(), k)
    lI = torch.where(lI >= 0, lI + r0, lI)
    gD = [torch.empty_like(lD) for _ in range(world)]
    gI = [torch.empty_like(lI) for _ in range(world)]
    dist.all_gather(gD, lD)
    dist.all_gather(gI, lI)
    parity = None
    if rank == 0:
        hD, hI = merge_host(torch.stack(gD).cpu().numpy(), torch.stack(gI).cpu().numpy(), k, fb.METRIC_L2)
        parity = {"queries": ns, "ids_equal": bool(np.array_equal(hI, I[:ns].cpu().numpy())),
                  "distances_equal": bool(np.array_equal(hD, D[:ns].cpu().numpy())),
                  "what": "NCCL all-gather + device merge == host merge_knn_results of the %d per-rank results" % world}
        parity["ok"] = parity["ids_equal"] and parity["distances_equal"]
    if rank == 0:
        clocks = sampler.stop()
        pk, src = peaks()
        alg = float(scanned[0]) * M
        out = {"metric": "queries/sec (IVFPQ, IndexShards over %d GPUs)" % world, "value": nq / (ms * 1e-3), "unit": "queries/s",
               "n_gpus": world, "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms, "higher_is_better": True,
               "scaling": "weak", "dtype": "u8 codes, f32 LUT", "data": "synthetic",
               "config": {"workload": "IndexShards x%d of GpuIndexIVFPQ: N=%d (%d per GPU) d=%d nlist=%d M=%d nbits=8 nprobe=%d nq=%d k=%d (BASELINE configs[4] per-GPU shape)" % (
                   world, N, N // world, d, nlist, M, args.nprobe, nq, k),
                   "kmeans": {"points": n_train, "niter": args.niter, "train_s": train_s, "s_per_iter": train_s / args.niter,
                              "allreduce_bytes_per_iter": 4 * (nlist * d + nlist + 1), "objective_first_last": [float(objs[0]), float(objs[-1])], "stats": kstats},
                   "add_s": add_s, "add_vec_per_s_per_gpu": (r1 - r0) / add_s, "allgather_bytes_per_rank_per_step": nq * k * 12},
               "clocks": clocks, "parity_check": parity,
               "roofline": {"bound": "hbm", "unit": "GB/s", "peak": float(pk["hbm_gbs"]) * world, "peak_source": src + " copy bandwidth x n_gpus",
                            "algorithmic_bytes_per_step": alg, "scan_ms_per_step_max_over_ranks": scan_ms,
                            "achieved": alg / (scan_ms * 1e-3) / 1e9 if scan_ms > 0 else None,
                            "frac": alg / (scan_ms * 1e-3) / 1e9 / (float(pk["hbm_gbs"]) * world) if scan_ms > 0 else None, "traffic": None}}
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
