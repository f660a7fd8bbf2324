"""When a forward sorts its depth strata lazily (gs_bin_policy.h: BinPlan.lazy_strata) and when the shape's "strata
needed" table must be reset to "all": a small C++ driver replays call sequences the way gs_forward consumes the plan and
the verdict.  No GPU."""
import shutil
import subprocess

import pytest

from tests.test_bin_policy_cpu import CSRC

MERGE_SORT, FWD_WS, ALL_STRATA, NO_TILE_STRATA = 64, 32, 524288, 16384

DRIVER = r"""
#include <cstdio>
#include "gs_bin_policy.h"

int main(int argc, char **argv) {
    if (argc > 1) {  // capacity check of the compositor's stage
        unsigned cap;
        while (scanf("%u", &cap) == 1) printf("%d\n", (int)lazy_stratum_fits(cap));
        return 0;
    }
    ShapeSlot slots[4];
    bool table[4] = {};
    uint64_t clock = 0;
    int V, nt, P;
    unsigned tuning, ov, w2, x2;
    while (scanf("%d %d %d %u %u %u %u", &V, &nt, &P, &tuning, &ov, &w2, &x2) == 7) {
        const BinShape sh{V, nt, P, 1};
        const size_t n = (size_t)V * P;
        const int k = pick_slot(slots, 4, clock, sh);
        SpecState &s = slots[k].spec;
        const BinPlan p = plan_binning(s, sh, n, table[k], tuning);
        bool exact = !p.speculate;
        if (p.speculate) {
            const uint32_t words[4] = {0, 300, w2, ov};
            bool release = false;
            exact = !learn_speculative(s, sh, p, words, 1u << 30, tuning, &release);
            printf("spec strata=%d tile=%d lazy=%d reset=%d %s", (int)p.strata, p.per_tile, (int)p.lazy_strata,
                   (int)p.reset_need, exact ? "redo" : "commit");
        }
        if (exact) {
            if (learn_exact(s, sh, n, 300, x2, true, tuning) != LEARN_NONE) {
                table[k] = true;
                start_trial(s);
            }
            printf("%sexact", p.speculate ? " " : "");
        }
        printf(" | learned=%d\n", (int)s.need_learned);
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.fail("no host C++ compiler")
    d = tmp_path_factory.mktemp("lazy_policy")
    src = d / "driver.cpp"
    src.write_text(DRIVER)
    exe = d / "driver"
    subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    return str(exe)


def replay(driver, calls, args=()):
    text = "".join(" ".join(str(v) for v in c) + "\n" for c in calls)
    return subprocess.run([driver, *args], input=text, capture_output=True, text=True, check=True).stdout.splitlines()


A = (2, 100, 1000)


def call(tuning=0, overflow=0, max_sub=50, exact_sub=60):
    return (*A, tuning, overflow, max_sub, exact_sub)


def test_table_is_reset_on_first_use_after_exact_and_after_overflow(driver):
    assert replay(driver, [call(), call(), call(), call(), call(overflow=1), call(), call()]) == [
        "exact | learned=0",                                   # first call of the shape
        "spec strata=1 tile=0 lazy=1 reset=1 commit | learned=1",   # trial: the table starts at "all"
        "spec strata=1 tile=0 lazy=1 reset=0 commit | learned=1",   # steady state reads what the last call wrote
        "spec strata=1 tile=0 lazy=1 reset=0 commit | learned=1",
        "spec strata=1 tile=0 lazy=1 reset=0 redo exact | learned=0",  # overflow: the redo's exact call forgets it
        "spec strata=1 tile=0 lazy=1 reset=1 commit | learned=1",
        "spec strata=1 tile=0 lazy=1 reset=0 commit | learned=1",
    ]


@pytest.mark.parametrize("tuning", [MERGE_SORT, FWD_WS, ALL_STRATA])
def test_merge_sort_ws_compositor_and_all_strata_never_skip(driver, tuning):
    got = replay(driver, [call(), call(tuning=tuning), call(tuning=tuning), call()])
    assert got == [
        "exact | learned=0",
        "spec strata=1 tile=0 lazy=0 reset=0 commit | learned=0",
        "spec strata=1 tile=0 lazy=0 reset=0 commit | learned=0",
        "spec strata=1 tile=0 lazy=1 reset=1 commit | learned=1",  # a table the compositor did not write is reset
    ]


def test_per_tile_strata_never_skip(driver):
    got = replay(driver, [call(), call(overflow=1), call(), call()])
    assert got == [
        "exact | learned=0",
        "spec strata=1 tile=0 lazy=1 reset=1 redo exact | learned=0",   # the per-view trial overflows: per-tile from here
        "spec strata=1 tile=1 lazy=0 reset=0 commit | learned=0",
        "spec strata=1 tile=1 lazy=0 reset=0 commit | learned=0",
    ]


def test_whole_tile_speculation_never_skips(driver):
    assert replay(driver, [call(tuning=8), call(tuning=8)]) == ["exact | learned=0",
                                                                "spec strata=0 tile=0 lazy=0 reset=0 commit | learned=0"]


def test_stratum_too_large_for_the_compositor_stage_never_skips(driver):
    # the stage holds 2 x 256 records of 48 bytes: 3072 keys of 8 bytes
    assert replay(driver, [(64,), (2048,), (3072,), (3073,), (4096,)], args=("fits",)) == ["1", "1", "1", "0", "0"]
