"""CPU: the restatement of GET /usage (user_usage_ref) against the known answers (tests/golden/user_usage_golden.json),
and cycle.usage_response on answers taken from the restatement of cook_state_user_usage, for one device and several."""
import json
import os

import pytest

import user_usage_ref as U
from cook_b200 import abi, cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "user_usage_golden.json")))


def plain(x):
    """The response as JSON gives it back (user codes as keys become strings)."""
    return json.loads(json.dumps(x))


def routed(step):
    """The handles a shim keeps for an api step: one per pool (one default handle without pools), each job in its pool's
    handle or, without a pool, in the default pool's; returns (names, [{task id: row}])."""
    names = step["pools"] or [step["default_pool"]]
    handles = [{} for _ in names]
    for j in step["jobs"]:
        p = names.index(U.pool_of(j, step["default_pool"]) if step["pools"] else names[0])
        handles[p][j["task_id"]] = dict(j, groups=[])
    return names, handles


def response(names, handles, req, pools, groups=None, devices=None):
    """cycle.usage_response over the restated answers: the pool's handle alone with a pool, else every handle, split
    into devices (lists of handle indices) when given."""
    gb = req.get("group_breakdown", False)
    users = None if req.get("user") is None else [req["user"]]
    if req.get("pool") is not None:
        p = names.index(req["pool"])
        parts = [[p]]
    else:
        parts = devices or [list(range(len(names)))]
    per_pool = req.get("pool") is None and bool(pools)
    answers = [(U.engine_answer([handles[k] for k in part], users, per_pool, gb), [names[k] for k in part])
               for part in parts]
    info = (lambda g: tuple(groups[str(g)])) if groups else None
    return cycle.usage_response(answers, user=req.get("user"), pool=req.get("pool"), pools=pools, group_breakdown=gb,
                                group_info=info)


@pytest.mark.parametrize("k", range(len(GOLDEN["api"])))
def test_api_steps(k):
    step = GOLDEN["api"][k]
    req = step["request"]
    jobs = sorted(step["jobs"], key=lambda j: j["task_id"])
    got = U.get_user_usage(jobs, user=req.get("user"), pool=req.get("pool"), pools=step["pools"],
                           default_pool=step["default_pool"])
    assert plain(got) == step["want"]
    names, handles = routed(step)
    assert plain(response(names, handles, req, step["pools"])) == step["want"]


def edge_handles():
    names = list(GOLDEN["edges"]["handles"])
    return names, [{r["task_id"]: r for r in GOLDEN["edges"]["handles"][n]} for n in names]


@pytest.mark.parametrize("k", range(len(GOLDEN["edges"]["cases"])))
def test_edges(k):
    case = GOLDEN["edges"]["cases"][k]
    req, groups = case["request"], GOLDEN["edges"]["groups"]
    names, handles = edge_handles()
    ginfo = {int(g): tuple(v) for g, v in groups.items()}
    got = U.get_user_usage(U.jobs_of(handles, names), user=req.get("user"), pool=req.get("pool"),
                           group_breakdown=req.get("group_breakdown", False), pools=names, groups=ginfo)
    assert plain(got) == case["want"]
    assert plain(response(names, handles, req, names, groups)) == case["want"]
    # alpha and beta on one device, gamma on another: gamma's job folds last, so the host's addition is the fold
    if req.get("pool") is None:
        assert plain(response(names, handles, req, names, groups, devices=[[0, 1], [2]])) == case["want"]


def test_edge_answer():
    """The call's segments for alice over the three handles: representatives, first groups, order, lists, bytes."""
    names, handles = edge_handles()
    a = U.answer(handles, [0], per_pool=True, by_group=True)
    keys = [s[:3] for s in a]
    assert keys == sorted(keys) and keys[:4] == [(0, -1, U.TOTAL), (0, -1, U.UNGROUPED), (0, -1, 7), (0, -1, 9)]
    seg = {s[:3]: s for s in a}
    assert seg[(0, -1, U.TOTAL)][3:7] == (5, 1.9000000000000001, 190.0, 1.0)
    assert seg[(0, 0, 7)][7] == [100] and seg[(0, 0, 7)][4] == 0.3      # job 100's row 1005, not 1001 / 1002
    assert (0, 0, 8) not in seg
    assert seg[(0, 1, 9)][7] == [102] and (0, 1, 7) not in seg          # [9, 7]: the first entry
    assert seg[(0, -1, U.UNGROUPED)][7] == [101, 100]                   # job 100 of beta is a job of its own
    assert (0, 2, U.UNGROUPED) not in seg                               # no empty segment
    assert U.answer(handles, [2], True, True) == []
    assert U.rows_queried(handles, [0]) == 7 and U.rows_queried(handles) == 8
    assert U.d2h_bytes(a, True) == 8 + 48 * len(a) + 8 * sum(len(s[7]) for s in a if s[7] is not None)
    assert U.d2h_bytes(U.answer(handles, None), False) == 8 + 44 * 2
    assert (abi.UU_TOTAL, abi.UU_UNGROUPED) == (U.TOTAL, U.UNGROUPED)


def test_group_totals_add_up():
    """grouped + ungrouped jobs make the total (test_user_usage_grouped / _ungrouped), in every scope."""
    names, handles = edge_handles()
    for user in (0, 1):
        segs = U.answer(handles, [user], per_pool=True, by_group=True)
        for scope in {s[1] for s in segs}:
            ss = [s for s in segs if s[1] == scope]
            total = next(s for s in ss if s[2] == U.TOTAL)
            assert sum(s[3] for s in ss if s[2] != U.TOTAL) == total[3]
            assert sum(len(s[7]) for s in ss if s[2] != U.TOTAL) == total[3]
