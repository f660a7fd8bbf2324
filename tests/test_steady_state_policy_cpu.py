"""The call sequences tests/test_gpu_steady_state.py drives, replayed through gs_bin_policy.h on the CPU: which calls sort
their depth strata lazily (BinPlan.lazy_strata) and which reset the shape's "strata needed" table (BinPlan.reset_need).
The GPU tests' claim that their steady-state calls skip strata rests on these plans.  No GPU."""
import pytest

from tests.test_lazy_strata_policy_cpu import ALL_STRATA, FWD_WS, MERGE_SORT, call, driver, replay  # noqa: F401

EXACT = "exact | learned=0"
TRIAL = "spec strata=1 tile=0 lazy=1 reset=1 commit | learned=1"   # the table starts at "all"
LAZY = "spec strata=1 tile=0 lazy=1 reset=0 commit | learned=1"    # reads what the previous forward wrote
EAGER = "spec strata=1 tile=0 lazy=0 reset=0 commit | learned=0"   # sorts every stratum; the table is not written


def test_the_seven_call_sequence(driver):
    """dense x 4, moved, faint, dense: from the third call on every forward reads a learned table."""
    assert replay(driver, [call()] * 7) == [EXACT, TRIAL] + [LAZY] * 5


@pytest.mark.parametrize("tuning", [ALL_STRATA, FWD_WS, MERGE_SORT])
def test_an_eager_call_between_default_calls_resets_the_table(driver, tuning):
    got = replay(driver, [call()] * 4 + [call(tuning=tuning), call(), call(), call(tuning=tuning), call(tuning=tuning),
                                         call()])
    assert got == [EXACT, TRIAL, LAZY, LAZY, EAGER,
                   "spec strata=1 tile=0 lazy=1 reset=1 commit | learned=1", LAZY,
                   EAGER, EAGER, "spec strata=1 tile=0 lazy=1 reset=1 commit | learned=1"]


def test_interleaved_settings_of_the_gpu_sequence(driver):
    """Learned on defaults; anti-aliasing, a depth mode, and anti-aliasing on faint opacities are flags and inputs, not
    tunings: the same plan, the same table; then ALL_STRATA, FWD_WS and the default twice, the first of which resets."""
    got = replay(driver, [call()] * 4 + [call()] * 3 + [call(tuning=ALL_STRATA), call(tuning=FWD_WS), call(), call()])
    assert got == [EXACT, TRIAL, LAZY, LAZY, LAZY, LAZY, LAZY, EAGER, EAGER,
                   "spec strata=1 tile=0 lazy=1 reset=1 commit | learned=1", LAZY]


def test_overflow_at_call_five(driver):
    got = replay(driver, [call()] * 4 + [call(overflow=1), call(), call()])
    assert got == [EXACT, TRIAL, LAZY, LAZY,
                   "spec strata=1 tile=0 lazy=1 reset=0 redo exact | learned=0",   # the redo's exact call forgets it
                   TRIAL, LAZY]


def _shape(V, nt, P, **kw):
    return (V, nt, P) + call(**kw)[3:]


def test_eviction_by_four_other_shapes_then_a_return(driver):
    A = lambda: _shape(2, 100, 1000)
    others = [_shape(2, 100, 1001 + k) for k in range(4)]
    got = replay(driver, [A()] * 4 + others + [A(), A(), A()])
    assert got == [EXACT, TRIAL, LAZY, LAZY] + [EXACT] * 4 + [EXACT, TRIAL, LAZY]   # evicted: learned afresh


def test_three_other_shapes_keep_the_slot(driver):
    A = lambda: _shape(2, 100, 1000)
    others = [_shape(2, 100, 1001 + k) for k in range(3)]
    got = replay(driver, [A()] * 4 + others + [A(), A()])
    assert got == [EXACT, TRIAL, LAZY, LAZY] + [EXACT] * 3 + [LAZY, LAZY]


def test_two_frames_of_one_shape_key_share_one_slot_and_table(driver):
    """64 x 80 and 80 x 64 are both 20 tiles: the key (V, tiles, P, S) is the same, so they alternate on one slot, each
    reading the table the other frame wrote.  The policy sees only the key, so for it this is the one-shape sequence:
    what it pins is that the alternation never resets the table.  That the compositor's fallback makes a table written
    by the other frame correct is checked on the GPU only.  A frame of another tile count is a slot of its own and
    leaves the table alone."""
    a, b = _shape(2, 20, 5000), _shape(2, 20, 5000)
    other = _shape(2, 30, 5000)
    got = replay(driver, [a, b, a, b, a, b, a, b, other, a])
    assert got == [EXACT, TRIAL] + [LAZY] * 6 + [EXACT, LAZY]
