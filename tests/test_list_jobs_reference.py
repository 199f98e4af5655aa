"""The job listing's restatement (list_ref) and cycle.list_jobs_response against the reference's answers for the
waiting and running states (golden/list_jobs_golden.json), and the per-state rules on their own."""
import json
import os

import numpy as np
import pytest

import list_ref as L
from cook_b200 import abi, cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "list_jobs_golden.json")))
CASES = [(s, i) for s in GOLDEN["scenarios"] for i in range(len(s["queries"]))]
STATE_BIT = {"waiting": L.WAITING, "running": L.RUNNING}


def handles(scenario):
    """The scenario's handles as list_ref rows, and each handle's pool code."""
    out = []
    for h in scenario["handles"]:
        run = [r["row"] if isinstance(r, dict) else r for r in h["running"]]
        out.append({"pending": [(u, j, tuple(f) if f else None) for u, j, f in h["pending"]],
                    "running": [(u, j, t, tuple(f) if f else None) for u, j, t, f in run]})
    return out, [h["pool"] for h in scenario["handles"]]


def ref_query(scenario, qd):
    hs, pools = handles(scenario)
    mask = 0
    for s in qd["states"]:
        mask |= STATE_BIT.get(s, 0)
    q = L.query(qd["user"], mask, qd["start"], qd["end"], qd["lo"], qd["hi"], qd["pool"], pools,
                qd["include_custom_executor"], qd["limit"])
    return hs, q


def answer_of(entries):
    cols = list(zip(*entries)) if entries else [(), (), (), ()]
    return {"state": np.array(cols[0], np.int32), "job_id": np.array(cols[1], np.int64),
            "submit_ms": np.array(cols[2], np.int64), "pool": np.array(cols[3], np.int32)}


def response(entries, qd):
    return cycle.list_jobs_response(answer_of(entries), states=qd["states"], limit=qd["limit"],
                                    completed={k: [tuple(e) for e in v] for k, v in qd.get("completed", {}).items()},
                                    uncommitted=[tuple(e) for e in qd.get("uncommitted", [])])


def check(qd, got, missing):
    if "response" in qd:
        assert got == qd["response"]
    if "get_jobs" in qd:
        assert list(reversed(got)) == qd["get_jobs"]
    if "count" in qd:
        assert len(got) == qd["count"]
    if "first" in qd:
        assert got[0] == qd["first"]
    if "second" in qd:
        assert got[1] == qd["second"]
    if "missing" in qd:
        assert missing == qd["missing"]


@pytest.mark.parametrize("scenario,i", CASES, ids=[f"{s['name']}-{i}" for s, i in CASES])
def test_golden(scenario, i):
    qd = scenario["queries"][i]
    hs, q = ref_query(scenario, qd)
    entries, missing = L.list_jobs(hs, q)
    check(qd, response(entries, qd), missing)


def test_abi_constants_match_the_restatement():
    assert (abi.LJ_WAITING, abi.LJ_RUNNING) == (L.WAITING, L.RUNNING)


def test_running_representative_is_the_greatest_task_id():
    """A job's running rows are one entry; its facts are its greatest task id's (another row's do not count)."""
    h = {"pending": [], "running": [(0, 7, 2, (100, -1, 0)), (0, 7, 5, None), (0, 8, 1, (50, -1, 0))]}
    q = L.query(0, L.RUNNING, 0, 1000)
    assert L.list_jobs([h], q) == ([(L.RUNNING, 8, 50, 0)], 1)
    h["running"][1] = (0, 7, 5, (100, -1, 1))
    assert L.list_jobs([h], L.query(0, L.RUNNING, 0, 1000, include_custom_executor=False)) == ([(L.RUNNING, 8, 50, 0)], 0)
    assert L.list_jobs([h], q)[0] == [(L.RUNNING, 7, 100, 0), (L.RUNNING, 8, 50, 0)]


def test_order_is_job_id_then_handle_and_each_state_is_cut():
    """One job id in two handles gives two entries, by handle; the cut applies per state before the merge."""
    f = (10, -1, 0)
    hs = [{"pending": [(0, 3, f), (0, 1, f)], "running": [(0, 2, 9, f)]},
          {"pending": [(0, 1, f)], "running": [(0, 2, 4, f), (0, 0, 1, f)]}]
    got, _ = L.list_jobs(hs, L.query(0, L.WAITING | L.RUNNING, 0, 100, limit=2))
    assert got == [(L.WAITING, 1, 10, 0), (L.WAITING, 1, 10, 1), (L.RUNNING, 0, 10, 1), (L.RUNNING, 2, 10, 0)]


def test_pool_check():
    """check-pool-for-listing: any pool (-1), the handle's pool, or the submit pool."""
    hs = [{"pending": [(0, 1, (5, -1, 0)), (0, 2, (5, 1, 0))], "running": []},
          {"pending": [(0, 3, (5, -1, 0)), (0, 4, (5, 0, 0))], "running": []}]
    ids = lambda pool: [e[1] for e in L.list_jobs(hs, L.query(0, L.WAITING, 0, 10, pool=pool, handle_pool=[0, 1]))[0]]
    assert ids(-1) == [1, 2, 3, 4]
    assert ids(0) == [1, 2, 4]
    assert ids(1) == [2, 3, 4]
    assert ids(2) == []


def test_response_merges_uncommitted_by_job_id_and_cuts():
    ans = answer_of([(L.WAITING, 5, 50, 0), (L.WAITING, 9, 10, 0)])
    got = cycle.list_jobs_response(ans, states=["waiting"], limit=2, uncommitted=[(7, 5)])
    # waiting by id [5, 7, 9] cut to [5, 7]; ascending submit [7, 5]; newest first
    assert got == [5, 7]
