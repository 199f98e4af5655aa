"""The sweeps' restatement (sweep_ref) against the reference's known answers and the hand-computed edges
(golden/sweeps_golden.json), and its own rules at those edges (CPU only)."""
import json
import runpy

import pytest

import sweep_ref as W

SCENARIOS = W.load_golden()["scenarios"]


@pytest.mark.parametrize("sc", SCENARIOS, ids=[s["name"] for s in SCENARIOS])
def test_golden(sc):
    rows, records, groups = W.scenario_inputs(sc)
    for chk in sc["checks"]:
        now = chk["now"]
        linger = [t for t, _ in W.lingering(rows, now, chk["default_timeout_ms"], chk["max_timeout_ms"])]
        cancel = [t for t, _ in W.cancelled(rows)]
        strag = [[g, t] for g, t, _ in W.stragglers(rows, records, groups, now)]
        W.check_answers(chk, linger, cancel, strag)


def test_golden_is_what_the_generator_writes():
    ns = runpy.run_path(W.GOLDEN.replace("sweeps_golden.json", "make_sweeps_golden.py"), run_name="generator")
    assert json.loads(json.dumps(ns["scenarios"]())) == SCENARIOS


def test_reference_cases_are_pinned():
    names = {s["name"] for s in SCENARIOS}
    assert {"get-lingering-tasks", "kill-lingering-tasks", "find-stragglers: no straggler-handling",
            "find-stragglers: quantile deviation, no stragglers", "find-stragglers: quantile deviation, stragglers found",
            "find-stragglers: not enough complete"} <= names
    found = next(s for s in SCENARIOS if s["name"] == "find-stragglers: quantile deviation, stragglers found")
    assert found["groups"]["0"]["n_jobs"] == 9 and len(found["successes"]) == 6


def test_idx_truncation_and_counts():
    g = {0: dict(kind="quantile-deviation", quantile=0.3, multiplier=1.0, n_jobs=8)}
    assert int((8 - 1) * 0.3) == 2
    rows = [dict(task_id=1, start=0, groups=[0])]
    now = 100_000   # 100 s
    assert W.stragglers(rows, [(0, 10), (0, 20)], g, now) == []          # two successes: count == idx
    assert W.stragglers(rows, [(0, 10), (0, 20), (0, 30)], g, now) == [(0, 1, 0)]


def test_whole_seconds_truncate():
    assert W.runtime_s(0, 999) == 0 and W.runtime_s(0, 1000) == 1 and W.runtime_s(5, 3_600_004) == 3599
    with pytest.raises(ValueError):
        W.runtime_s(10, 9)


def test_start_after_now_throws_only_when_judged():
    g = {0: dict(kind="quantile-deviation", quantile=0.0, multiplier=1.0, n_jobs=1)}
    later = dict(task_id=1, start=2000, groups=[0])
    with pytest.raises(ValueError):
        W.stragglers([later], [(0, 1)], g, 1000)
    assert W.stragglers([dict(later, status="unknown")], [(0, 1)], g, 1000) == []
    with pytest.raises(ValueError):
        W.stragglers([later], [], g, 1000)            # without a success too: cook_state_sweep's rule


def test_orders_break_ties_by_pool():
    rows = [dict(task_id=5, start=0, pool=1, cancelled=True), dict(task_id=5, start=0, pool=0, cancelled=True),
            dict(task_id=2, start=0, pool=1, cancelled=True)]
    assert W.cancelled(rows) == [(2, 1), (5, 0), (5, 1)]
    assert W.lingering(rows, 10, 1, 1) == [(2, 1), (5, 0), (5, 1)]


def test_lingering_is_strict_and_int64():
    big = 2 ** 63 - 1
    rows = [dict(task_id=1, start=0, max_runtime=big), dict(task_id=2, start=0, max_runtime=30)]
    assert W.lingering(rows, 30, 10 ** 6, 10 ** 6) == []
    assert W.lingering(rows, 31, 10 ** 6, 10 ** 6) == [(2, 0)]
    assert W.lingering(rows, 10 ** 6 + 1, 10, 10 ** 6) == [(1, 0), (2, 0)]
