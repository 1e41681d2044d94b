#!/usr/bin/env python
"""bench_flat_rounds.py -- where the tensor-core Flat kernel's time goes, round by round, at bench.py's headline shape.

The search runs its database tiles in rounds of growing size (faiss_b200/csrc/flat_tc_schedule.h), one
flat_tc_kernel launch each; later rounds filter against tighter thresholds.  This script builds bench.py's seeded
index (N=10M, d=128, nq=10k, k=100; BENCH_N / BENCH_D / BENCH_NQ / BENCH_K override), warms it, then profiles
--searches searches with torch.profiler (CUDA activities only) while nvidia-smi samples the SM clock.  For each round
it prints the median kernel time, the largest number of tiles one CTA walks in it (from the schedule, compiled here
with the host C++ compiler) and so the clocks per tile at the median SM clock, and how many queries were searched again
because their estimated thresholds overshot (those repairs add launches outside the table).  The last line is one
JSON object.

  python bench_flat_rounds.py [--searches 5] [--warmup 3]

Writes nothing but stdout / stderr: the schedule driver is compiled in a temporary directory.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the headline shape, its seeded generators, the clock sampler and the card's identity)

CSRC = os.path.join(ROOT, "faiss_b200", "csrc")

DRIVER = r"""
#include <cstdio>
#include "flat_tc_schedule.h"
using namespace fb200::tc;
int main() {
    long long n, nq;
    int k, sms, int8;
    if (scanf("%lld %d %d %lld %d", &n, &k, &sms, &nq, &int8) != 5)
        return 1;
    const FlatTcSchedule s = planFlatTcSchedule(n, k, sms, 0, 0, int8 != 0);
    const char* sep = "";
    printf("[");
    for (long long qb = 0; qb < nq; qb += s.qBatch) {
        const long long b = nq - qb < s.qBatch ? nq - qb : s.qBatch;
        const long long qPairs = (b + kUnitM - 1) / kUnitM;
        const FlatTcRounds r = s.rounds(qPairs);
        for (size_t i = 0; i < r.rounds.size(); i++) {
            const FlatTcRound& x = r.rounds[i];
            printf("%s[%lld, %d, %d, %d, %d]", sep, qPairs, x.begin, x.end, x.slices, x.tilesPerSlice);
            sep = ", ";
        }
    }
    printf("]\n");
}
"""


def schedule(n, k, sms, nq, int8):
    """[(qPairs, begin, end, slices, tilesPerSlice)] of every flat_tc_kernel launch of one search, in launch order"""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        raise RuntimeError("no host C++ compiler (g++) for the schedule driver")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "sched.cpp"), os.path.join(d, "sched")
        with open(src, "w") as f:
            f.write(DRIVER)
        subprocess.run([cxx, "-std=c++17", "-O1", "-I", CSRC, src, "-o", exe], check=True)
        out = subprocess.run([exe], input="%d %d %d %d %d\n" % (n, k, sms, nq, int(int8)), capture_output=True,
                             text=True, check=True).stdout
    return [tuple(r) for r in json.loads(out)]


def tiles_per_cta(qpairs, begin, end, slices, tps, sms):
    """the most tiles one CTA walks in a launch: unit u = slice * qPairs + query unit, CTA c takes u = c, c + grid, ..."""
    units = qpairs * slices
    grid = min(units, sms)
    most = 0
    for c in range(grid):
        t = 0
        for u in range(c, units, grid):
            sl = u // qpairs
            b = begin + sl * tps
            t += max(0, min(end, b + tps) - b)
        most = max(most, t)
    return most, grid


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--searches", type=int, default=5, help="profiled searches (the median per round is reported)")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    assert torch.cuda.is_available(), "bench_flat_rounds.py needs a GPU"
    import faiss_b200 as fb

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    res = fb.StandardGpuResources()
    stream = torch.cuda.current_stream(device)
    res.setDefaultStream(0, stream.cuda_stream)
    sms = torch.cuda.get_device_properties(device).multi_processor_count

    xb = bench.gen_rows(torch, device, 0, bench.N_TOTAL, bench.DIM)
    index = fb.GpuIndexFlatL2(res, bench.DIM, device=0)
    index.add(xb)
    del xb
    xq = bench.gen_queries(torch, device, bench.NQ, bench.DIM)
    torch.cuda.synchronize()

    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.7)  # nvidia-smi start-up
    sampler.mark_load()
    for _ in range(max(1, args.warmup)):
        index.search(xq, bench.K)
    torch.cuda.synchronize()
    bits = index.lastSearchOperandBits()
    repaired = index.lastSearchRepairedQueries()
    sched = schedule(bench.N_TOTAL, bench.K, sms, bench.NQ, bits == 8)

    sampler.mark_begin()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.searches):
            index.search(xq, bench.K)
        torch.cuda.synchronize()
    sampler.mark_end()
    clocks = sampler.stop()

    kern = sorted((e for e in prof.events() if "flat_tc_kernel" in e.name), key=lambda e: e.time_range.start)
    per_search = len(sched)
    if len(kern) != per_search * args.searches:
        raise RuntimeError("profiled %d flat_tc_kernel launches, the schedule has %d per search x %d searches "
                           "(%d queries repaired per search)" % (len(kern), per_search, args.searches, repaired))
    ms = np.array([e.time_range.elapsed_us() * 1e-3 for e in kern]).reshape(args.searches, per_search)
    mhz = clocks.get("sm_mhz")
    rows = []
    for i, (qp, b, e, sl, tps) in enumerate(sched):
        tiles, grid = tiles_per_cta(qp, b, e, sl, tps, sms)
        med = float(np.median(ms[:, i]))
        rows.append({"round": i, "tiles": [b, e], "slices": sl, "tiles_per_slice": tps, "grid": grid,
                     "tiles_per_cta": tiles, "ms": med, "ms_min": float(ms[:, i].min()), "ms_max": float(ms[:, i].max()),
                     "clocks_per_tile": (med * 1e-3 * mhz * 1e6 / tiles) if mhz else None})
    total_ms = float(np.median(ms.sum(axis=1)))
    total_tiles = sum(r["tiles_per_cta"] for r in rows)
    gpu = bench.gpu_identity(0)

    print("%s, power limit %s W, median SM clock %s MHz (%s), operand bits %d, repaired queries %d"
          % (gpu.get("name"), gpu.get("power_limit_w"), mhz, clocks.get("window", clocks.get("reasons")), bits, repaired))
    print("%5s %15s %6s %5s %6s %10s %9s %12s" % ("round", "tiles", "slices", "grid", "tps", "tiles/CTA", "ms", "clocks/tile"))
    for r in rows:
        cpt = "%12.0f" % r["clocks_per_tile"] if r["clocks_per_tile"] else "%12s" % "-"
        print("%5d %15s %6d %5d %6d %10d %9.3f %s" % (r["round"], "%d-%d" % tuple(r["tiles"]), r["slices"], r["grid"],
                                                    r["tiles_per_slice"], r["tiles_per_cta"], r["ms"], cpt))
    cpt_all = total_ms * 1e-3 * mhz * 1e6 / total_tiles if mhz else None
    print("%5s %15s %6s %5s %6s %10d %9.3f %s" % ("all", "", "", "", "", total_tiles, total_ms,
                                                  ("%12.0f" % cpt_all) if cpt_all else "-"))
    print(json.dumps({"gpu": gpu, "clocks": clocks, "operand_bits": bits, "repaired_queries": repaired,
                      "searches": args.searches,
                      "flat_tc_ms": total_ms, "tiles_per_cta": total_tiles, "clocks_per_tile": cpt_all, "rounds": rows}),
          flush=True)


if __name__ == "__main__":
    main()
