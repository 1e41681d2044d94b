"""The round schedule of the tensor-core Flat search (faiss_b200/csrc/flat_tc_schedule.h), on the CPU.

The header is pure host arithmetic: it is compiled here with the host C++ compiler and a small driver.  The pinned
table below is the schedule the search has always computed for these shapes (batch size, first round, tile
permutation, every round and the scratch sizes); a change to it changes which kernels run with which grids."""
import json
import os
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "faiss_b200", "csrc")

DRIVER = r"""
#include <cstdio>
#include "flat_tc_schedule.h"
using namespace fb200::tc;
int main() {
    long long n, nq, maxTiles;
    int k, sms, ranks;
    while (scanf("%lld %d %d %lld %d %lld", &n, &k, &sms, &nq, &ranks, &maxTiles) == 6) {
        const FlatTcSchedule s = planFlatTcSchedule(n, k, sms, ranks, maxTiles);
        printf("{\"qBatch\": %lld, \"r0\": %d, \"A\": %llu, \"B\": %llu, \"LIST\": %d, \"KL\": %d, \"bisect\": %d, "
               "\"streaming\": %d, \"T\": %lld, \"Tsched\": %lld, \"batches\": [",
               (long long)s.qBatch, s.r0Tiles, s.permA, s.permB, s.LIST, s.KL, (int)s.useBisect, (int)s.streaming,
               (long long)s.T, (long long)s.Tsched);
        const char* sep = "";
        for (long long qb = 0; qb < nq; qb += s.qBatch) {
            const long long b = nq - qb < s.qBatch ? nq - qb : s.qBatch;
            const long long qPairs = (b + kUnitM - 1) / kUnitM;
            const FlatTcRounds r = s.rounds(qPairs);
            printf("%s[%lld, [", sep, qPairs);
            for (size_t i = 0; i < r.rounds.size(); i++) {
                const FlatTcRound& x = r.rounds[i];
                printf("%s[%d, %d, %d, %d, %d]", i ? ", " : "", x.begin, x.end, x.slices, x.tilesPerSlice, x.cap);
            }
            printf("], %zu, %zu]", r.arenaBytes, r.countBytes);
            sep = ", ";
        }
        printf("]}\n");
    }
}
"""

# name: (n, k, SMs, nq, shard ranks (0: not sharded), largest shard's tiles)
SHAPES = {
    "n10m_k100": (10_000_000, 100, 132, 10_000, 0, 0),
    "n10m_k100_2shards": (4_999_000, 100, 132, 10_000, 2, 19532),
    "n10m_k100_8shards": (1_249_000, 100, 132, 10_000, 8, 4883),
    "k1_stream_nlist4096": (4096, 1, 132, 1_000_000, 0, 0),
    "k128": (10_000_000, 128, 132, 10_000, 0, 0),
    "k129": (10_000_000, 129, 132, 10_000, 0, 0),
    "k2048": (10_000_000, 2048, 132, 10_000, 0, 0),
    "n32769": (32769, 100, 132, 10_000, 0, 0),
}

# (qBatch, r0, A, B, LIST, KL, bisect, streaming, distinct batches: [(qPairs, rounds (begin, end, slices, tiles per
# slice, cap), arena bytes, count bytes)])
PINNED = {
    "n10m_k100": (65536, 4, 24142, 13021, 256, 128, 1, 0, [
        (79, [(0, 4, 1, 4, 256), (4, 16, 1, 12, 512), (16, 64, 3, 16, 256), (64, 256, 5, 39, 128),
              (256, 1024, 5, 154, 128), (1024, 4096, 5, 615, 128), (4096, 16384, 5, 2458, 128),
              (16384, 39063, 5, 4536, 128)], 248512512, 808960)]),
    "n10m_k100_2shards": (65536, 4, 12069, 6509, 256, 128, 1, 0, [
        (79, [(0, 4, 1, 4, 256), (4, 16, 1, 12, 512), (16, 64, 3, 16, 256), (64, 256, 5, 39, 128),
              (256, 1024, 5, 154, 128), (1024, 4096, 5, 615, 128), (4096, 19532, 5, 3088, 256)], 414187520, 808960)]),
    "n10m_k100_8shards": (131072, 2, 3015, 1626, 256, 128, 1, 0, [
        (79, [(0, 2, 1, 2, 128), (2, 16, 1, 14, 2048), (16, 128, 5, 23, 256), (128, 1024, 5, 180, 256),
              (1024, 4883, 5, 772, 256)], 662700032, 808960)]),
    "k1_stream_nlist4096": (67584, 2, 9, 5, 128, 64, 1, 1, [
        (528, [(0, 16, 1, 16, 64)], 138412032, 1081344),
        (421, [(0, 16, 1, 16, 64)], 110362624, 862208)]),
    "k128": (65536, 4, 24142, 13021, 256, 128, 1, 0, [
        (79, [(0, 4, 1, 4, 256), (4, 16, 1, 12, 1024), (16, 64, 3, 16, 256), (64, 256, 5, 39, 256),
              (256, 1024, 5, 154, 256), (1024, 4096, 5, 615, 256), (4096, 16384, 5, 2458, 256),
              (16384, 39063, 5, 4536, 128)], 414187520, 808960)]),
    "k129": (16384, 21, 24142, 13021, 512, 256, 0, 0, [
        (79, [(0, 21, 1, 21, 1344), (21, 84, 3, 21, 256), (84, 336, 5, 51, 256), (336, 1344, 5, 202, 256),
              (1344, 5376, 5, 807, 256), (5376, 21504, 5, 3226, 256), (21504, 39063, 5, 3512, 64)],
         434896896, 808960)]),
    "k2048": (2048, 320, 24142, 13021, 4096, 2048, 0, 0, [
        (16, [(0, 320, 8, 40, 2560), (320, 1280, 8, 120, 2048), (1280, 5120, 8, 480, 2048),
              (5120, 20480, 33, 466, 512), (20480, 39063, 33, 564, 128)], 1342177280, 1081344),
        (15, [(0, 320, 8, 40, 2560), (320, 1280, 8, 120, 2048), (1280, 5120, 26, 148, 512),
              (5120, 20480, 35, 439, 512), (20480, 39063, 44, 423, 128)], 1258291200, 1351680)]),
    "n32769": (65536, 4, 79, 43, 256, 128, 1, 0, [
        (79, [(0, 4, 1, 4, 256), (4, 16, 1, 12, 512), (16, 64, 3, 16, 256), (64, 129, 3, 22, 128)],
         248512512, 485376)]),
}

K_TILE_N, K_PARTS = 256, 4


@pytest.fixture(scope="module")
def schedules(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no host C++ compiler (g++)")
    d = tmp_path_factory.mktemp("flat_tc_schedule")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text(DRIVER)
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    names = list(SHAPES)
    stdin = "".join("%d %d %d %d %d %d\n" % SHAPES[nm] for nm in names)
    out = subprocess.run([str(exe)], input=stdin, capture_output=True, text=True, check=True).stdout
    lines = out.strip().splitlines()
    assert len(lines) == len(names)
    return {nm: json.loads(line) for nm, line in zip(names, lines)}


def distinct_batches(s):
    """the batches of a schedule, consecutive repeats of the same qPairs dropped"""
    out = []
    for qp, rounds, arena, counts in s["batches"]:
        b = (qp, [tuple(r) for r in rounds], arena, counts)
        if not out or out[-1][0] != qp:
            out.append(b)
    return out


@pytest.mark.parametrize("name", list(SHAPES))
def test_schedule_pinned(schedules, name):
    s = schedules[name]
    got = (s["qBatch"], s["r0"], s["A"], s["B"], s["LIST"], s["KL"], s["bisect"], s["streaming"], distinct_batches(s))
    assert got == PINNED[name]


@pytest.mark.parametrize("name", list(SHAPES))
def test_schedule_invariants(schedules, name):
    s = schedules[name]
    n, k, sms, nq, ranks, max_tiles = SHAPES[name]
    assert s["T"] == (n + K_TILE_N - 1) // K_TILE_N
    assert s["Tsched"] == (max(s["T"], max_tiles) if ranks else s["T"])
    assert sum(min(s["qBatch"], nq - q) for q in range(0, nq, s["qBatch"])) == nq
    for _, rounds, _, _ in s["batches"]:
        # the rounds tile [0, Tsched) contiguously, every slice within its round
        assert rounds[0][0] == 0 and rounds[-1][1] == s["Tsched"]
        for (b0, e0, _, _, _), (b1, _, _, _, _) in zip(rounds, rounds[1:]):
            assert e0 == b1 and b0 < e0
        for b, e, slices, tps, _ in rounds:
            assert slices * tps >= e - b > (slices - 1) * tps
        if s["streaming"]:
            assert len(rounds) == 1 and rounds[0][4] == 64
        else:
            tps0 = rounds[0][3]
            assert rounds[0][4] == tps0 * K_TILE_N // K_PARTS  # every score of round 0 is a candidate
