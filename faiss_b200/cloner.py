"""Cloner helpers at payload level: the host format either side of the hot path.

The reference clones a CPU index to GPUs with `index_cpu_to_gpu[_multiple]` (faiss/gpu/GpuCloner.cpp:
124-498): coarse centroids, PQ centroids and every `ArrayInvertedLists` list (codes bytes + int64 ids)
are copied verbatim; with `GpuMultipleClonerOptions.shard` the inverted lists are split over the GPUs
by `shard_type` (GpuCloner.cpp:287-322, `IndexIVF::copy_subset_to`, faiss/IndexIVF.cpp).  These
helpers work on that payload (numpy arrays), so any producer of the format -- the reference CPU index,
a file reader -- can feed them; nothing here depends on the reference's classes.

    payload = {"d", "nlist", "metric", "centroids" [nlist, d] f32,
               "pq" [M, 2^nbits, dsub] f32 (IVFPQ only; nbits != 8 builds the index with interleaved_layout),
               "sq" {"qtype", "by_residual", "trained" f32} (IVF scalar quantiser only: ScalarQuantizer::trained),
               "codes": [nlist] uint8 arrays, "ids": [nlist] int64 arrays}

    cagra payload = {"d", "metric", "xb" [n, d] f32, "graph" [n, degree] int64}   (GpuIndexCagra <-> IndexHNSWCagra)
"""
import numpy as np

SHARD_BY_ID_MOD = 1      # id % nshard == i          (the reference's default)
SHARD_BY_ID_RANGE = 2    # i*ntotal/nshard <= id < (i+1)*ntotal/nshard
SHARD_BY_LIST_RANGE = 4  # whole lists  i*nlist/nshard <= l < (i+1)*nlist/nshard


def shard_ivf_lists(codes, ids, code_size, nshard, shard_type=SHARD_BY_ID_MOD, ntotal=None):
    """Split inverted lists over `nshard` sub-indexes with the reference's rules
    (ToGpuClonerMultiple::copy_ivf_shard, GpuCloner.cpp:287-322).  Entry order inside a list is kept
    (copy_subset_to appends in list order).  Returns [(codes_i, ids_i)] * nshard, each a list over all
    nlist lists (empty arrays where a shard holds nothing of a list)."""
    nlist = len(ids)
    assert len(codes) == nlist and nshard >= 1
    ids = [np.ascontiguousarray(a, dtype=np.int64).reshape(-1) for a in ids]
    codes = [np.ascontiguousarray(c, dtype=np.uint8).reshape(-1, code_size) for c in codes]
    for c, a in zip(codes, ids):
        assert c.shape[0] == a.size, "codes / ids length mismatch"
    if ntotal is None:
        ntotal = int(sum(a.size for a in ids))
    out = []
    for i in range(nshard):
        ci, ii = [], []
        if shard_type == SHARD_BY_ID_RANGE:
            i0, i1 = i * ntotal // nshard, (i + 1) * ntotal // nshard
        elif shard_type == SHARD_BY_LIST_RANGE:
            l0, l1 = i * nlist // nshard, (i + 1) * nlist // nshard
        elif shard_type != SHARD_BY_ID_MOD:
            raise ValueError("shard_type %d not implemented" % shard_type)  # as the reference
        for l in range(nlist):
            if shard_type == SHARD_BY_ID_MOD:
                keep = (ids[l] % nshard) == i
            elif shard_type == SHARD_BY_ID_RANGE:
                keep = (ids[l] >= i0) & (ids[l] < i1)
            else:
                keep = np.full(ids[l].shape, l0 <= l < l1)
            ci.append(np.ascontiguousarray(codes[l][keep]).reshape(-1))
            ii.append(np.ascontiguousarray(ids[l][keep]))
        out.append((ci, ii))
    return out


def _pq_nbits(pq):
    """nbits of PQ centroids [M, 2^nbits, dsub]"""
    ksub = int(pq.shape[1])
    nbits = ksub.bit_length() - 1
    if ksub != 1 << nbits:
        raise ValueError("PQ centroids: %d centroids per sub-quantizer is not a power of two" % ksub)
    return nbits


def gpu_ivf_from_payload(res, payload, device=0):
    """GpuIndexIVFFlat / GpuIndexIVFPQ / GpuIndexIVFScalarQuantizer holding exactly the payload (the role of
    copyFrom, faiss/gpu/GpuIndexIVFPQ.cu:105-217, GpuIndexIVFFlat.cu:89-150, GpuIndexIVFScalarQuantizer.cu:126-210)."""
    import faiss_b200 as fb

    d, nlist, metric = int(payload["d"]), int(payload["nlist"]), int(payload.get("metric", fb.METRIC_L2))
    if payload.get("sq") is not None:
        sq = payload["sq"]
        index = fb.GpuIndexIVFScalarQuantizer(
            res, d, nlist, int(sq["qtype"]), metric, bool(sq.get("by_residual", True)), device=device
        )
        index.setCoarseCentroids(payload["centroids"])
        index.setTrained(np.asarray(sq.get("trained", []), dtype=np.float32))
    elif "pq" in payload and payload["pq"] is not None:
        pq = np.ascontiguousarray(payload["pq"], dtype=np.float32)
        M, nbits = int(pq.shape[0]), _pq_nbits(pq)
        if nbits == 8:
            index = fb.GpuIndexIVFPQ(res, d, nlist, M, 8, metric, device=device)
        else:  # the reference GPU index takes 4-, 5- and 6-bit codes only with GpuIndexIVFPQConfig::interleavedLayout
            index = fb.GpuIndexIVFPQ(res, d, nlist, M, nbits, metric, device=device, interleaved_layout=True)
        index.setCoarseCentroids(payload["centroids"])
        index.setPQCentroids(pq)
    else:
        index = fb.GpuIndexIVFFlat(res, d, nlist, metric, device=device)
        index.setCoarseCentroids(payload["centroids"])
    # all list lengths are known up front: ONE arena relayout with exact capacities, then plain copies
    # (per-list growth would re-layout the whole arena once per list: quadratic in nlist)
    index.setListSizes(np.array([len(payload["ids"][l]) for l in range(nlist)], dtype=np.int64))
    for l in range(nlist):
        if len(payload["ids"][l]):
            index.setList(l, payload["codes"][l], payload["ids"][l])
    index.setIsTrained(True)
    return index


def gpu_ivf_shards_from_payload(resources, payload, shard_type=SHARD_BY_ID_MOD, devices=None, threaded=True):
    """index_cpu_to_gpu_multiple(..., shard=True): one sub-index per resources object, the same coarse
    quantiser (and PQ) everywhere, lists split by `shard_type`, wrapped in IndexShards with explicit ids
    (successive_ids=False, GpuCloner.cpp:417)."""
    import faiss_b200 as fb

    n = len(resources)
    devices = list(devices) if devices is not None else [0] * n
    if payload.get("sq") is not None:
        # the code size is the index's own (ScalarQuantizer::code_size): build the shards first, then fill them
        empty = dict(payload)
        empty["codes"] = [np.zeros(0, np.uint8)] * int(payload["nlist"])
        empty["ids"] = [np.zeros(0, np.int64)] * int(payload["nlist"])
        subs = [gpu_ivf_from_payload(r, empty, device=dev) for r, dev in zip(resources, devices)]
        parts = shard_ivf_lists(payload["codes"], payload["ids"], subs[0]._code_size(), n, shard_type)
        shards = fb.IndexShards(int(payload["d"]), threaded=threaded, successive_ids=False)
        for sub_index, (ci, ii) in zip(subs, parts):
            sub_index.setListSizes(np.array([len(a) for a in ii], dtype=np.int64))
            for l in range(len(ii)):
                if len(ii[l]):
                    sub_index.setList(l, ci[l], ii[l])
            shards.add_shard(sub_index)
        return shards
    if payload.get("pq") is not None:
        pq = payload["pq"]
        code_size = (int(pq.shape[0]) * _pq_nbits(pq) + 7) // 8  # ProductQuantizer::code_size
    else:
        code_size = 4 * int(payload["d"])
    parts = shard_ivf_lists(payload["codes"], payload["ids"], code_size, n, shard_type)
    shards = fb.IndexShards(int(payload["d"]), threaded=threaded, successive_ids=False)
    for r, dev, (ci, ii) in zip(resources, devices, parts):
        sub = dict(payload)
        sub["codes"], sub["ids"] = ci, ii
        shards.add_shard(gpu_ivf_from_payload(r, sub, device=dev))
    return shards


# ------------------------------------------------------------------------------------------------
# GpuIndexCagra <-> IndexHNSWCagra: the "cagra" payload {"d", "metric", "xb" [n, d] f32, "graph" [n, degree] int64}
# is what GpuIndexCagra::copyFrom(IndexHNSWCagra*) and copyTo move (faiss/gpu/GpuIndexCagra.cu copyFrom_ex / copyTo):
# the stored vectors and the level-0 neighbour table (-1: no edge).
# ------------------------------------------------------------------------------------------------
def cagra_payload(index):
    """the payload of a built GpuIndexCagra"""
    xb, graph = index.copyTo()
    return {"d": int(index.d), "metric": int(index.metric_type), "xb": xb, "graph": graph}


def gpu_cagra_from_payload(res, payload, device=0):
    """a GpuIndexCagra holding exactly the payload's vectors and graph"""
    import faiss_b200 as fb

    cfg = fb.GpuIndexCagraConfig()
    cfg.device = int(device)
    index = fb.GpuIndexCagra(res, int(payload["d"]), int(payload.get("metric", fb.METRIC_L2)), cfg)
    index.copyFrom(payload["xb"], payload["graph"])
    return index
