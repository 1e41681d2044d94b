"""The estimated-threshold rule of the tensor-core Flat search (flat_tc_schedule.h flatTcEstRank), on the CPU.

After `seen` of T tiles the selection may raise a query's threshold to its j-th best score so far; the rule picks the
smallest j whose miss probability under the header's model -- the query's top-k rows in pairs, X = 2 Y with
Y ~ Hypergeometric(T, ceil(k / 2), seen) -- is at most delta.  Pinned here against scipy's hypergeometric tail, with
the per-round share of the miss budget the schedule gives each round and the searches that must not estimate."""
import json
import os
import shutil
import subprocess

import pytest
from scipy.stats import hypergeom

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "faiss_b200", "csrc")

DRIVER = r"""
#include <cstdio>
#include "flat_tc_schedule.h"
using namespace fb200::tc;
int main() {
    char mode[8];
    while (scanf("%7s", mode) == 1) {
        if (mode[0] == 'r') { // rank: T k seen delta
            long long T, seen;
            int k;
            double delta;
            if (scanf("%lld %d %lld %lf", &T, &k, &seen, &delta) != 4)
                return 1;
            printf("%d\n", flatTcEstRank(T, k, seen, delta));
        } else { // schedule: n k ranks maxTiles nq -> T, budget and [end, estRank] of every round
            long long n, maxTiles, nq;
            int k, ranks;
            if (scanf("%lld %d %d %lld %lld", &n, &k, &ranks, &maxTiles, &nq) != 5)
                return 1;
            const FlatTcSchedule s = planFlatTcSchedule(n, k, 132, ranks, maxTiles);
            const FlatTcRounds r = s.rounds((nq + kUnitM - 1) / kUnitM);
            printf("{\"T\": %lld, \"budget\": %.17g, \"rounds\": [", (long long)s.T, kEstMissBudget);
            for (size_t i = 0; i < r.rounds.size(); i++)
                printf("%s[%d, %d]", i ? ", " : "", r.rounds[i].end, r.rounds[i].estRank);
            printf("]}\n");
        }
    }
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    d = tmp_path_factory.mktemp("est")
    src, exe = str(d / "est.cpp"), str(d / "est")
    with open(src, "w") as f:
        f.write(DRIVER)
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", CSRC, src, "-o", exe], check=True)

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return out.split("\n")[:-1]

    return run


def _tail(T, k, seen, y):
    """P(Y >= y), Y ~ Hypergeometric(T tiles, ceil(k / 2) pairs, seen draws)"""
    return float(hypergeom(T, (k + 1) // 2, min(seen, T)).sf(y - 1))


CASES = [(T, k, seen, delta)
         for T in (128, 782, 7813, 39063, 1 << 20)
         for k in (2, 10, 100, 128, 1024)
         for seen in (1, 4, 16, 64, 256, 1024, 4096, 16384, 65536)
         for delta in (1e-4 / 7, 1e-3)
         if seen < T]


def test_rank_is_the_smallest_within_the_tail_bound(driver):
    got = driver(["r %d %d %d %.17g" % c for c in CASES])
    assert len(got) == len(CASES)
    for (T, k, seen, delta), j in zip(CASES, map(int, got)):
        assert 0 <= j < k
        if (k + 1) // 2 >= T:  # a pair in every tile: no estimate
            assert j == 0
            continue
        if j > 0:
            assert j % 2 == 1  # X = 2 Y >= j  <=>  Y >= (j + 1) / 2
            y = (j + 1) // 2
            assert _tail(T, k, seen, y) <= delta * (1 + 1e-9), (T, k, seen, delta, j)
            assert y == 1 or _tail(T, k, seen, y - 1) > delta * (1 - 1e-9), (T, k, seen, delta, j)
        else:  # no j < k meets delta: the largest odd j < k does not
            y = k // 2 if k % 2 == 0 else (k - 1) // 2
            assert y < 1 or _tail(T, k, seen, y) > delta * (1 - 1e-9), (T, k, seen, delta)


@pytest.mark.parametrize("n,k,nq", [(10_000_000, 100, 10_000), (2_000_000, 10, 300), (400_000, 1024, 5000),
                                    (65536, 10, 64)])
def test_schedule_splits_the_budget_over_the_rounds(driver, n, k, nq):
    s = json.loads(driver(["s %d %d 0 0 %d" % (n, k, nq)])[0])
    rounds = s["rounds"]
    assert rounds[-1][1] == 0  # the last selection sets the final, provable threshold
    delta = s["budget"] / (len(rounds) - 1)
    want = driver(["r %d %d %d %.17g" % (s["T"], k, end, delta) for end, _ in rounds[:-1]])
    assert [r[1] for r in rounds[:-1]] == [int(j) for j in want]
    assert any(r[1] > 0 for r in rounds)


def test_sharded_and_streaming_searches_stay_provable(driver):
    sharded = json.loads(driver(["s 4000000 100 4 4000 10000"])[0])
    streaming = json.loads(driver(["s 4000000 1 0 0 10000"])[0])
    assert all(r[1] == 0 for r in sharded["rounds"] + streaming["rounds"])
