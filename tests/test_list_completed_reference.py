"""The completed-job listing's restatement (completed_ref) and cycle.list_jobs_response fed with it against the
reference's answers for the completed, success and failed states (golden/list_completed_golden.json), and the log's
rules on their own."""
import json
import os

import pytest

import completed_ref as CR
import list_ref as L
import test_list_jobs_reference as LJ
from cook_b200 import abi, cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                     "list_completed_golden.json")))
CASES = [(s, i) for s in GOLDEN["scenarios"] for i in range(len(s["queries"]))]
ACTIVE = {"waiting": L.WAITING, "running": L.RUNNING}


def logs(scenario):
    """Each handle's log after its seed and record batches."""
    out = []
    for h in scenario["handles"]:
        lg = CR.seed(h["since"], h["seed"])
        for b in h["record"]:
            CR.record(lg, b)
        out.append(lg)
    return out


def query(scenario, qd):
    """The query as list_ref.query, its waiting / running bits, and the completed-family states it asks for."""
    mask = 0
    for s in qd["states"]:
        mask |= ACTIVE.get(s, 0)
    q = L.query(qd["user"], mask, qd["start"], qd["end"], qd["lo"], qd["hi"], qd["pool"],
                [h["pool"] for h in scenario["handles"]], qd["include_custom_executor"], qd["limit"])
    return q, [s for s in qd["states"] if s in CR.NAMES]


def active_rows(scenario):
    return [{"pending": [(u, j, tuple(f) if f else None) for u, j, f in h["pending"]], "running": []}
            for h in scenario["handles"]]


def respond(qd, active_entries, completed):
    return cycle.list_jobs_response(LJ.answer_of(active_entries), states=qd["states"], limit=qd["limit"],
                                    completed=completed)


@pytest.mark.parametrize("scenario,i", CASES, ids=[f"{s['name']}-{i}" for s, i in CASES])
def test_golden(scenario, i):
    qd = scenario["queries"][i]
    q, done = query(scenario, qd)
    lgs = logs(scenario)
    if qd.get("refused"):
        assert CR.refused(lgs, q["start"])
        return
    assert not CR.refused(lgs, q["start"])
    entries = L.list_jobs(active_rows(scenario), q)[0] if q["states"] else []
    completed = {s: [(j, t) for j, t, _ in CR.list_completed(lgs, q, CR.NAMES[s])] for s in done}
    LJ.check(qd, respond(qd, entries, completed), None)


def test_abi_constants_match_the_restatement():
    assert (abi.CJ_SUCCESS, abi.CJ_FAILED, abi.CJ_REOPENED) == (CR.SUCCESS, CR.FAILED, CR.REOPENED)
    assert (abi.LC_SUCCESS, abi.LC_FAILED, abi.LC_COMPLETED) == (CR.L_SUCCESS, CR.L_FAILED, CR.L_COMPLETED)


def q0(**kw):
    return L.query(0, 0, 0, 1000, **kw)


def test_latest_record_wins_by_stamp_then_handle_then_row():
    """Equal stamps go to the greater handle index, then the later row; the latest record's handle is the entry's."""
    a = CR.seed(0, [(5, 10, 0, 1, -1, 0, CR.FAILED), (5, 10, 0, 1, -1, 0, CR.SUCCESS)])
    b = CR.seed(0, [(5, 9, 0, 1, -1, 0, CR.REOPENED)])
    assert CR.list_completed([a, b], q0(), CR.L_COMPLETED) == [(5, 1, 0)]
    assert CR.list_completed([a, b], q0(), CR.L_SUCCESS) == [(5, 1, 0)]   # the later row of handle 0
    b = CR.seed(0, [(5, 10, 0, 1, -1, 0, CR.REOPENED)])                    # same stamp, greater handle
    assert CR.list_completed([a, b], q0(), CR.L_COMPLETED) == []


def test_filters_apply_to_the_latest_record_and_the_cut_follows_them():
    rows = [(1, 1, 0, 5, -1, 0, CR.FAILED), (2, 1, 0, 6, -1, 0, CR.SUCCESS), (3, 1, 0, 7, -1, 0, CR.SUCCESS),
            (2, 2, 0, 6, -1, 0, CR.FAILED)]
    lg = CR.seed(0, rows)
    assert CR.list_completed([lg], q0(), CR.L_FAILED) == [(1, 5, 0), (2, 6, 0)]
    assert CR.list_completed([lg], q0(limit=1), CR.L_SUCCESS) == [(3, 7, 0)]


def test_record_skips_rows_before_the_horizon_and_advance_drops_them():
    lg = CR.seed(10, [])
    CR.record(lg, [(1, 1, 0, 9, -1, 0, CR.SUCCESS), (2, 1, 0, 10, -1, 0, CR.SUCCESS), (3, 1, 0, 12, -1, 0, CR.SUCCESS)])
    assert [r[0] for r in lg["rows"]] == [2, 3]
    CR.advance(lg, 11)
    assert [r[0] for r in lg["rows"]] == [3]
    assert CR.refused([lg], 10) and not CR.refused([lg], 11)
