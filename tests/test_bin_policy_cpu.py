"""The forward's binning policy (pf3plat_b200/csrc/gs_bin_policy.h) on the host: a small C++ driver replays scripted
call sequences -- the verdict words a speculative call would read back, the counts an exact call would scan -- the way
gs_forward consumes them, and prints the plan and the shape's state after each call.  No GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pf3plat_b200", "csrc")

FORCE_RADIX, NO_SPEC, SEPARATE_EMIT, NO_STRATA, NO_TILE_STRATA = 1, 2, 4, 8, 16384

# One call per input line: shape (V, tiles, P, S), tuning, the speculative verdict (overflow, longest list, largest
# sub-counter) and the exact path's counts (longest list, largest sub-counter).  Like gs_forward, the driver runs the
# exact path after a plan that does not speculate and after an overflow, allocates a slot's boundary table on its
# first learn and keeps it when the slot is evicted, and grows the sort scratch to the speculative buckets.
DRIVER = r"""
#include <cstdio>
#include "gs_bin_policy.h"

static const char *NAMES[] = {"UNKNOWN", "TRIAL", "ON", "OFF"};

int main() {
    ShapeSlot slots[4];
    bool table[4] = {};
    uint64_t clock = 0;
    size_t sort_bytes = 0;
    int V, nt, P, S;
    unsigned tuning, ov, w1, w2, x1, x2;
    while (scanf("%d %d %d %d %u %u %u %u %u %u", &V, &nt, &P, &S, &tuning, &ov, &w1, &w2, &x1, &x2) == 10) {
        const BinShape sh{V, nt, P, S};
        const size_t n = (size_t)V * P;
        const int k = pick_slot(slots, 4, clock, sh);
        SpecState &s = slots[k].spec;
        const BinPlan p = plan_binning(s, sh, n, table[k], tuning);
        printf("s%d", k);
        bool exact = !p.speculate;
        if (p.speculate) {
            const size_t need = (size_t)V * nt * BIN_SUB * p.sub_cap * 8;
            if (need > sort_bytes) sort_bytes = need + 256;
            const uint32_t words[4] = {0, w1, w2, ov};
            bool release = false;
            const bool committed = learn_speculative(s, sh, p, words, sort_bytes, tuning, &release);
            if (release) sort_bytes = 0;
            printf(" spec strata=%d tile=%d cap=%u read=%d write=%d fused=%d %s release=%d", (int)p.strata, p.per_tile,
                   p.sub_cap, p.read_tab, p.write_tab, (int)p.fused_emit, committed ? "commit" : "redo", (int)release);
            exact = !committed;
        }
        if (exact) {
            const bool smem_sort = x1 <= BIN_SMEM_CAP && !(tuning & GS_TUNE_FORCE_RADIX_BINNING);
            const int learn = learn_exact(s, sh, n, x1, x2, smem_sort, tuning);
            if (learn != LEARN_NONE) {
                table[k] = true;
                start_trial(s);
            }
            printf(" exact learn=%s", learn == LEARN_NONE ? "none" : learn == LEARN_PER_TILE ? "tile" : "view");
        }
        printf(" | %s cap=%u limit=%u tile=%d tab=%d\n", NAMES[s.strata_state], s.sub_cap, s.tile_limit,
               s.per_tile, s.tile_tab);
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.fail("no host C++ compiler")
    d = tmp_path_factory.mktemp("bin_policy")
    src = d / "driver.cpp"
    src.write_text(DRIVER)
    exe = d / "driver"
    subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    return str(exe)


def call(shape, spec=(0, 0, 0), exact=(0, 0), tuning=0):
    return (*shape, tuning, *spec, *exact)


def replay(driver, calls):
    text = "".join(" ".join(str(v) for v in c) + "\n" for c in calls)
    out = subprocess.run([driver], input=text, capture_output=True, text=True, check=True).stdout
    return out.splitlines()


A = (2, 100, 1000, 1)          # 200 (view, tile) pairs: 1 600 sub-buckets


def test_fresh_shape_exact_then_per_view_trial_then_sticky_on(driver):
    got = replay(driver, [
        call(A, exact=(300, 60)),              # exact: capacities 94 -> 128, limit 362 -> 384; per-view boundaries
        call(A, spec=(0, 280, 50)),            # trial on doubled capacities
        call(A, spec=(0, 280, 60)),            # needs 94 -> 128: kept
        call(A, spec=(0, 280, 40)),            # needs 68 -> 128: kept
        call(A, spec=(0, 280, 20)),            # needs 42 -> 64: 128 > 1.5 x 64, re-derived
        call(A, spec=(0, 280, 200)),           # needs 276 -> 320: 64 no longer fits
        call(A, spec=(0, 280, 180)),           # needs 250 -> 256: 320 <= 1.5 x 256, kept
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=256 read=0 write=-1 fused=1 commit release=0 | ON cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=128 read=0 write=-1 fused=1 commit release=0 | ON cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=128 read=0 write=-1 fused=1 commit release=0 | ON cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=128 read=0 write=-1 fused=1 commit release=0 | ON cap=64 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=64 read=0 write=-1 fused=1 commit release=0 | ON cap=320 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=320 read=0 write=-1 fused=1 commit release=0 | ON cap=320 limit=384 tile=0 tab=0",
    ]


def test_trial_capacity_is_clamped_and_its_buckets_released(driver):
    got = replay(driver, [
        call(A, exact=(3000, 1100)),           # 1 446 -> 1 472 per sub-bucket: the trial's 2 944 is clamped to 2 048
        call(A, spec=(0, 2000, 100)),          # 26 MB of trial buckets against 2 x 2.4 MB + 8 MB needed: given back
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=1472 limit=3392 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=2048 read=0 write=-1 fused=1 commit release=1 | ON cap=192 limit=3392 tile=0 tab=0",
    ]
    got = replay(driver, [
        call(A, exact=(3000, 1100)),
        call(A, spec=(0, 2000, 900)),          # next capacity 1 216: 2 x 15.6 MB + 8 MB exceeds the 26 MB, kept
        call(A, spec=(0, 2000, 100)),          # ON: only a trial's buckets are given back
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=1472 limit=3392 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=2048 read=0 write=-1 fused=1 commit release=0 | ON cap=1216 limit=3392 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=1216 read=0 write=-1 fused=1 commit release=0 | ON cap=192 limit=3392 tile=0 tab=0",
    ]


def test_trial_beyond_32_bit_offsets_runs_whole_tile_and_stays_in_trial(driver):
    big = (8, 40000, 1000, 1)                  # 2 560 000 sub-buckets: 1 024 each fits 32-bit offsets, 2 048 does not
    got = replay(driver, [
        call(big, exact=(2000, 760)),
        call(big, spec=(0, 2000, 760)),
        call(big, spec=(0, 2000, 760)),
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=1024 limit=2240 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=1024 read=-1 write=-1 fused=0 commit release=0 | TRIAL cap=1024 limit=2240 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=1024 read=-1 write=-1 fused=0 commit release=0 | TRIAL cap=1024 limit=2240 tile=0 tab=0",
    ]
    # 1 706 -> 1 728 per sub-bucket puts offsets beyond 32 bits even undoubled: exact, no boundaries, call after call
    assert replay(driver, [call(big, exact=(2000, 1300))] * 2) == ["s0 exact learn=none | UNKNOWN cap=0 limit=0 tile=0 tab=0"] * 2


def test_stratum_beyond_2048_turns_strata_off_for_good_unless_headroom_fits(driver):
    got = replay(driver, [
        call(A, exact=(3000, 1100)),
        call(A, spec=(0, 2000, 1800)),         # 2 356 -> 2 368 > 2 048, but 1 800 + 10 % fits: capacity 2 048
        call(A, spec=(0, 2000, 1900)),         # 2 496 > 2 048 and 1 900 + 10 % does not fit: OFF
        call(A, exact=(3000, 1100)),           # OFF is sticky: no boundaries learned
        call(A, spec=(0, 3000, 1100)),         # whole-tile speculation
        call(A, spec=(1, 0, 0), exact=(3000, 1100)),   # a whole-tile overflow leaves OFF alone
        call(A, spec=(0, 3000, 1100)),
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=1472 limit=3392 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=2048 read=0 write=-1 fused=1 commit release=0 | ON cap=2048 limit=3392 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=2048 read=0 write=-1 fused=1 commit release=0 | OFF cap=0 limit=3392 tile=0 tab=0",
        "s0 exact learn=none | OFF cap=1472 limit=3392 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=1472 read=-1 write=-1 fused=1 commit release=0 | OFF cap=1472 limit=3392 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=1472 read=-1 write=-1 fused=1 redo release=0 exact learn=none | OFF cap=1472 limit=3392 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=1472 read=-1 write=-1 fused=1 commit release=0 | OFF cap=1472 limit=3392 tile=0 tab=0",
    ]


def test_per_view_trial_overflow_moves_to_per_tile_boundaries(driver):
    got = replay(driver, [
        call(A, exact=(300, 60)),
        call(A, spec=(1, 0, 0), exact=(300, 60)),   # per-view trial overflows: the exact redo learns per-tile boundaries
        call(A, spec=(0, 280, 50)),                 # per-tile trial: reads table 0, the sort writes table 1
        call(A, spec=(0, 280, 50)),                 # and the tables swap on every success
        call(A, spec=(0, 280, 50)),
        call(A, spec=(1, 0, 0), exact=(300, 60)),   # ON overflows reading table 1: the redo learns into table 0
        call(A, spec=(0, 280, 50)),                 # the new per-tile trial reads table 0
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=256 read=0 write=-1 fused=1 redo release=0 exact learn=tile | TRIAL cap=128 limit=384 tile=1 tab=0",
        "s0 spec strata=1 tile=1 cap=256 read=0 write=1 fused=1 commit release=0 | ON cap=128 limit=384 tile=1 tab=1",
        "s0 spec strata=1 tile=1 cap=128 read=1 write=0 fused=1 commit release=0 | ON cap=128 limit=384 tile=1 tab=0",
        "s0 spec strata=1 tile=1 cap=128 read=0 write=1 fused=1 commit release=0 | ON cap=128 limit=384 tile=1 tab=1",
        "s0 spec strata=1 tile=1 cap=128 read=1 write=0 fused=1 redo release=0 exact learn=tile | TRIAL cap=128 limit=384 tile=1 tab=0",
        "s0 spec strata=1 tile=1 cap=256 read=0 write=1 fused=1 commit release=0 | ON cap=128 limit=384 tile=1 tab=1",
    ]


def test_per_view_trial_overflow_without_tile_strata_turns_strata_off(driver):
    got = replay(driver, [
        call(A, exact=(300, 60), tuning=NO_TILE_STRATA),
        call(A, spec=(1, 0, 0), exact=(300, 60), tuning=NO_TILE_STRATA),
        call(A, spec=(0, 280, 60), tuning=NO_TILE_STRATA),
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=256 read=0 write=-1 fused=1 redo release=0 exact learn=none | OFF cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | OFF cap=128 limit=384 tile=0 tab=0",
    ]


def test_per_tile_trial_overflow_turns_strata_off(driver):
    got = replay(driver, [
        call(A, exact=(300, 60)),
        call(A, spec=(1, 0, 0), exact=(300, 60)),
        call(A, spec=(1, 0, 0), exact=(300, 60)),   # the per-tile trial overflows too
        call(A, spec=(0, 280, 60)),
    ])
    assert got[2:] == [
        "s0 spec strata=1 tile=1 cap=256 read=0 write=1 fused=1 redo release=0 exact learn=none | OFF cap=128 limit=384 tile=1 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | OFF cap=128 limit=384 tile=1 tab=0",
    ]


def test_overflow_while_on_goes_back_to_unknown_then_exact_then_a_new_trial(driver):
    got = replay(driver, [
        call(A, exact=(300, 60)),
        call(A, spec=(0, 280, 50)),
        call(A, spec=(1, 0, 0), exact=(9000, 60)),  # ON overflows; the redo's lists exceed the shared-memory sort
        call(A, exact=(300, 60)),                   # UNKNOWN: exact, learns per-view boundaries again
        call(A, spec=(0, 280, 50)),                 # a new trial
        call(A, spec=(1, 0, 0), exact=(300, 60)),   # ON overflows, the redo learns at once
    ])
    assert got == [
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=256 read=0 write=-1 fused=1 commit release=0 | ON cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=128 read=0 write=-1 fused=1 redo release=0 exact learn=none | UNKNOWN cap=0 limit=384 tile=0 tab=0",
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=256 read=0 write=-1 fused=1 commit release=0 | ON cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=1 tile=0 cap=128 read=0 write=-1 fused=1 redo release=0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
    ]


def test_sticky_tile_limit_and_lists_too_long_for_speculation(driver):
    got = replay(driver, [
        call(A, exact=(300, 60), tuning=NO_STRATA),
        call(A, spec=(0, 320, 60), tuning=NO_STRATA),    # 384 -> 384: kept
        call(A, spec=(0, 200, 60), tuning=NO_STRATA),    # 252 -> 256: 384 <= 1.5 x 256, kept
        call(A, spec=(0, 140, 60), tuning=NO_STRATA),    # 186 -> 192: 384 > 1.5 x 192, re-derived
        call(A, spec=(0, 400, 60), tuning=NO_STRATA),    # 472 -> 512: 192 no longer fits
        call(A, spec=(0, 7400, 60), tuning=NO_STRATA),   # 8 172 -> 8 192: still the shared-memory sort
        call(A, spec=(0, 7500, 60), tuning=NO_STRATA),   # 8 282 -> 8 320: lists too long, exact from now on
        call(A, exact=(7500, 60), tuning=NO_STRATA),
        call(A, exact=(300, 60), tuning=NO_STRATA),
    ])
    assert got == [
        "s0 exact learn=none | UNKNOWN cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=128 limit=192 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=128 limit=512 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=128 limit=8192 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=0 limit=8192 tile=0 tab=0",
        "s0 exact learn=none | UNKNOWN cap=0 limit=8192 tile=0 tab=0",
        "s0 exact learn=none | UNKNOWN cap=128 limit=384 tile=0 tab=0",
    ]


def test_tuning_bits(driver):
    # GS_TUNE_FORCE_RADIX_BINNING: never speculates, and the radix sort learns no boundaries
    assert replay(driver, [call(A, exact=(300, 60), tuning=FORCE_RADIX)] * 2 + [call(A, spec=(0, 300, 60))]) == [
        "s0 exact learn=none | UNKNOWN cap=128 limit=384 tile=0 tab=0",
        "s0 exact learn=none | UNKNOWN cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=128 limit=384 tile=0 tab=0",
    ]
    # GS_TUNE_NO_SPECULATION: always exact (boundaries are still learned)
    assert replay(driver, [call(A, exact=(300, 60), tuning=NO_SPEC)] * 2) == [
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
    ]
    # GS_TUNE_NO_STRATA: whole-tile speculation on undoubled capacities, even with a trial pending
    assert replay(driver, [call(A, exact=(300, 60)), call(A, spec=(0, 300, 60), tuning=NO_STRATA)]) == [
        "s0 exact learn=view | TRIAL cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | TRIAL cap=128 limit=384 tile=0 tab=0",
    ]
    # GS_TUNE_SEPARATE_EMIT: k_emit_buckets fills the buckets
    assert replay(driver, [call(A, exact=(300, 60)), call(A, spec=(0, 300, 50), tuning=SEPARATE_EMIT)])[1] == (
        "s0 spec strata=1 tile=0 cap=256 read=0 write=-1 fused=0 commit release=0 | ON cap=128 limit=384 tile=0 tab=0")
    # no Gaussians: never speculates, learns nothing
    empty = (2, 100, 0, 1)
    assert replay(driver, [call(empty)] * 2) == ["s0 exact learn=none | UNKNOWN cap=64 limit=64 tile=0 tab=0"] * 2


def test_fused_emission_bound_is_96_mb_of_buckets(driver):
    wide = (4, 3072, 1000, 1)                  # 98 304 sub-buckets of 8-byte entries: 128 each is exactly 96 MB
    got = replay(driver, [
        call(wide, exact=(300, 60), tuning=NO_STRATA),
        call(wide, spec=(0, 300, 120), tuning=NO_STRATA),
        call(wide, spec=(0, 300, 120), tuning=NO_STRATA),
    ])
    assert got == [
        "s0 exact learn=none | UNKNOWN cap=128 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0 | UNKNOWN cap=192 limit=384 tile=0 tab=0",
        "s0 spec strata=0 tile=0 cap=192 read=-1 write=-1 fused=0 commit release=0 | UNKNOWN cap=192 limit=384 tile=0 tab=0",
    ]


def test_five_shapes_evict_the_least_recently_used_slot(driver):
    shapes = [(v, 100, 1000, 1) for v in (1, 2, 3, 4, 5)]
    got = replay(driver, [
        *[call(sh, exact=(300, 60), tuning=NO_STRATA) for sh in shapes[:4]],
        call(shapes[0], spec=(0, 300, 60), tuning=NO_STRATA),     # hit: keeps its capacities
        call(shapes[4], exact=(300, 60), tuning=NO_STRATA),       # miss: evicts shape 2, the least recently used
        call(shapes[1], exact=(300, 60), tuning=NO_STRATA),       # shape 2 starts over, in shape 3's slot
        call(shapes[0], spec=(0, 300, 60), tuning=NO_STRATA),
        call(shapes[3], spec=(0, 300, 60), tuning=NO_STRATA),
        call((1, 100, 1000, 2), exact=(300, 60), tuning=NO_STRATA),  # another scene count is another shape
    ])
    assert [line.split(" |")[0] for line in got] == [
        "s0 exact learn=none", "s1 exact learn=none", "s2 exact learn=none", "s3 exact learn=none",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0",
        "s1 exact learn=none",
        "s2 exact learn=none",
        "s0 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0",
        "s3 spec strata=0 tile=0 cap=128 read=-1 write=-1 fused=1 commit release=0",
        "s1 exact learn=none",
    ]
