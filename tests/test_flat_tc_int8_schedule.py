"""The schedule of an int8-scored tensor-core Flat search (flat_tc_schedule.h, int8 = true): a base list of
max(128, nextpow2(4k)) entries, selection by bisection for every k <= 128, and candidate caps that hold the rounds at
the int8 margin.  Compiled with the host compiler, no GPU needed."""
import json
import os
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "faiss_b200", "csrc")

SRC = r"""
#include <cstdio>
#include "flat_tc_schedule.h"
using namespace fb200::tc;
int main() {
    long long n; int k, sms;
    while (scanf("%lld %d %d", &n, &k, &sms) == 3) {
        const FlatTcSchedule s = planFlatTcSchedule(n, k, sms, 0, 0, true);
        const FlatTcRounds r = s.rounds((s.qBatch + kUnitM - 1) / kUnitM);
        printf("{\"LIST\": %d, \"KL\": %d, \"bisect\": %d, \"r0\": %d, \"rounds\": [", s.LIST, s.KL, (int)s.useBisect, s.r0Tiles);
        for (size_t i = 0; i < r.rounds.size(); i++)
            printf("%s[%d, %d, %d, %d, %d]", i ? ", " : "", r.rounds[i].begin, r.rounds[i].end, r.rounds[i].slices,
                   r.rounds[i].tilesPerSlice, r.rounds[i].cap);
        printf("]}\n");
    }
}
"""

SHAPES = [(n, k) for n in (32768, 1_000_000, 10_000_000) for k in (2, 10, 64, 100, 128)]
# entries within 2 eps of the k-th best under the int8 certificate, per k (median of a CPU simulation on uniform
# data at d = 128, N = 10M, k = 100: 274 entries)
MARGIN = 2.74
K_SEL_CAP = 1536  # tc_select_bisect_kernel's per-query buffer (kSelCap)


@pytest.fixture(scope="module")
def plans(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no host C++ compiler (g++)")
    d = tmp_path_factory.mktemp("int8sched")
    src, exe = d / "s.cpp", d / "s"
    src.write_text(SRC)
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    stdin = "".join("%d %d 132\n" % s for s in SHAPES)
    out = subprocess.run([str(exe)], input=stdin, capture_output=True, text=True, check=True).stdout
    return dict(zip(SHAPES, (json.loads(l) for l in out.splitlines())))


@pytest.mark.parametrize("shape", SHAPES)
def test_list_and_selection(plans, shape):
    n, k = shape
    p = plans[shape]
    assert p["LIST"] == max(128, 1 << (4 * k - 1).bit_length())
    assert p["LIST"] <= 512 and p["bisect"] == 1


@pytest.mark.parametrize("shape", SHAPES)
def test_rounds_hold_the_int8_margin(plans, shape):
    """every round after the first: the mean count of a segment stays under half its cap, and the base list plus the
    round's expected candidates fit the selection buffer"""
    n, k = shape
    for begin, end, slices, tps, cap in plans[shape]["rounds"]:
        if begin == 0:
            assert slices * tps * 256 <= K_SEL_CAP  # the all-pass first round
            continue
        mean = MARGIN * k * tps / begin / 4
        assert mean <= cap / 2, (begin, end, tps, cap, mean)
        assert MARGIN * k * (1 + (end - begin) / begin) <= K_SEL_CAP, (begin, end)

