"""Worker for tests/test_multigpu.py: one process per GPU (launched with torch.distributed.run), the database
sharded over the ranks behind faiss_b200.DistributedIndexShards (NCCL communicator owned by the resources
object, id handed over through the launcher's process group).  Rank 0 checks the merged result against an
UNSHARDED index over the same rows and prints one JSON line.  Model: faiss/gpu/test/test_multi_gpu.py:23-43."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist

    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")  # only to hand the 128-byte NCCL id around (plumbing)
    import faiss_b200 as fb

    res = fb.StandardGpuResources()
    ids = [fb.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    res.ncclInitRank(local, world, rank, ids[0])
    assert res.ncclRank(local) == (rank, world)
    out = {"world": world}
    rs = np.random.RandomState(123)

    # ---- Flat, tensor-core path with pooled thresholds (N large enough for the tensor-core path), floats and integers
    N, d, nq, k = 300_000, 64, 700, 50
    xb = rs.rand(N, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    for name, tb, tq in (("flat_float", xb, xq), ("flat_int", np.floor(xb * 16), np.floor(xq * 16))):
        r0, r1 = rank * N // world, (rank + 1) * N // world
        shard = fb.GpuIndexFlatL2(res, d, device=local)
        sh = fb.DistributedIndexShards(res, shard, successive_ids=True)
        sh.add(tb[r0:r1])
        assert sh.ntotal == N and sh.info()["id_offset"] == r0
        D, I = sh.search(tq, k)
        tc = shard.lastSearchInfo()["tensor_cores"]
        Dd, Id = sh.search(torch.from_numpy(tq).cuda(local), k)  # device-resident queries
        if rank == 0:
            full = fb.GpuIndexFlatL2(res, d, device=local, use_tensor_cores=False)
            full.add(tb)
            uD, uI = full.search(tq, k)
            out[name] = {"ids_equal": bool(np.array_equal(I, uI)), "distances_equal": bool(np.array_equal(D, uD)),
                         "device_queries_equal": bool(np.array_equal(Id.cpu().numpy(), uI) and np.array_equal(Dd.cpu().numpy(), uD)),
                         "tensor_cores": tc}
        del sh, shard

    # ---- small Flat shards (exact SIMT path on every rank: no pooling), inner product, k > shard size
    N2, k2 = 90, 64
    xs = rs.rand(N2, 16).astype(np.float32)
    r0, r1 = rank * N2 // world, (rank + 1) * N2 // world
    shard = fb.GpuIndexFlatIP(res, 16, device=local)
    sh = fb.DistributedIndexShards(res, shard)
    sh.add(xs[r0:r1])
    D, I = sh.search(xs[:7], k2)
    if rank == 0:
        full = fb.GpuIndexFlatIP(res, 16, device=local)
        full.add(xs)
        uD, uI = full.search(xs[:7], k2)
        out["flat_ip_small"] = {"ids_equal": bool(np.array_equal(I, uI)), "distances_equal": bool(np.array_equal(D, uD))}
    del sh, shard

    # ---- IVF-Flat shards with explicit ids (id mod world), one coarse quantiser everywhere
    N3, d3, nlist, nprobe, k3 = 40_000, 32, 64, 8, 20
    x3 = rs.rand(N3, d3).astype(np.float32)
    q3 = rs.rand(200, d3).astype(np.float32)
    cent = x3[rs.permutation(N3)[:nlist]].copy()
    ivf = fb.GpuIndexIVFFlat(res, d3, nlist, fb.METRIC_L2, device=local)
    ivf.setCoarseCentroids(cent)
    ivf.setIsTrained(True)
    ivf.nprobe = nprobe
    sh = fb.DistributedIndexShards(res, ivf, successive_ids=False)
    mine = np.arange(rank, N3, world)
    sh.add_with_ids(x3[mine], mine.astype(np.int64))
    assert sh.ntotal == N3
    D, I = sh.search(q3, k3)
    if rank == 0:
        full = fb.GpuIndexIVFFlat(res, d3, nlist, fb.METRIC_L2, device=local)
        full.setCoarseCentroids(cent)
        full.setIsTrained(True)
        full.nprobe = nprobe
        full.add(x3)
        uD, uI = full.search(q3, k3)
        out["ivfflat_idmod"] = {"ids_equal": bool(np.array_equal(I, uI)), "distances_equal": bool(np.array_equal(D, uD))}
    del sh, ivf
    # ---- sharded k-means (C++, one packed all-reduce per iteration) == the single-process algorithm on the
    # concatenated set: integer-valued points make every partial sum exact, so the centroids must be identical
    xk = np.floor(rs.rand(24_000, 16) * 32).astype(np.float32)
    r0, r1 = rank * 24_000 // world, (rank + 1) * 24_000 // world
    cent, obj, st = fb.kmeans_sharded(res, xk[r0:r1], 50, niter=6, seed=321, device=local)
    if rank == 0:
        c1, o1 = fb.kmeans(res, xk, 50, niter=6, seed=321, max_points_per_centroid=1 << 20, device=local)
        out["kmeans_sharded"] = {"ids_equal": bool(np.array_equal(cent, c1)), "distances_equal": bool(np.allclose(obj, o1, rtol=1e-5)),
                                 "max_abs_diff": float(np.abs(cent - c1).max())}
    dist.barrier()
    if rank == 0:
        print("RESULT " + json.dumps(out), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
