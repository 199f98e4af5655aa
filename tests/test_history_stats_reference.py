"""CPU: the restatement of a finished-instance history and of GET /stats/instances for success and failed
(history_ref) and cycle.instance_stats_response against the known answers in tests/golden/history_stats_golden.json:
the reference's integration assertions transcribed, the hand-computed edges (a left fold on its last bit, end ==
start, the window's and the id bound's edges, the horizon, a tie at the tenth leader, zero cpus, a task id in two
handles), and the table's seed, finish and advance."""
import json
import os

import pytest

import history_ref as Hr
from cook_b200 import cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "history_stats_golden.json")))
REASONS = {int(k): v for k, v in GOLDEN["reasons"].items()}
LO, HI = -(1 << 63), (1 << 63) - 1


def plain(x):
    return json.loads(json.dumps(x))


def seeded(rows, since=GOLDEN["since"]):
    h = Hr.History()
    h.seed(since, rows)
    return h


def edge_histories():
    h = GOLDEN["edges"]["handles"]
    return [seeded(h[k]) for k in ("a", "b", "c")]


def response(hs, q):
    a = Hr.engine_answer(hs, q["status"], q["start"], q["end"], q.get("lo", LO), q.get("hi", HI))
    return cycle.instance_stats_response(a, user_name=str, reason_string=REASONS.get)


@pytest.mark.parametrize("k", range(len(GOLDEN["transcribed"])))
def test_transcribed(k):
    t = GOLDEN["transcribed"][k]
    q = t["request"]
    hs = [seeded(t["rows"], t["since"])]
    r = response(hs, q)
    key = t["reason"]
    assert r["overall"]["count"] == r["by-reason"][key]["count"] == t["count"]
    assert r["by-user-and-reason"][str(t["user"])][key]["count"] == t["count"]
    for m, chk in t["checks"].items():
        assert plain(r["overall"][m]["percentiles"]) == chk["percentiles"]
        assert r["overall"][m]["total"] == pytest.approx(chk["total_approx"], abs=1e-7)
    ref = Hr.get_stats(Hr.instances_of(hs, reason_of=lambda c: None if c == -1 else REASONS[c]), q["status"],
                       q["start"], q["end"], LO, HI)
    assert plain(r) == plain(Hr.I.response_keys(ref))


@pytest.mark.parametrize("k", range(len(GOLDEN["edges"]["cases"])))
def test_edges(k):
    case = GOLDEN["edges"]["cases"][k]
    q = case["request"]
    hs = edge_histories()
    got = Hr.get_stats(Hr.instances_of(hs, reason_of=lambda c: None if c == -1 else REASONS[c]), q["status"],
                       q["start"], q["end"], q["lo"], q["hi"])
    assert plain(Hr.I.response_keys(got)) == case["want"]
    r = response(hs, q)
    assert plain(r) == case["want"]
    for m in ("cpu-seconds", "mem-seconds"):   # the leaders' order, not only their map
        assert list(r["leaders"][m].items()) == list(case["want"]["leaders"][m].items())


def test_edge_facts():
    ex = GOLDEN["edges"]["expect"]
    cases = {c["name"]: c["want"] for c in GOLDEN["edges"]["cases"]}
    s, f = cases["success"], cases["failed"]
    assert s["overall"]["count"] == ex["success_count"]
    assert cases["alice's window"]["overall"]["cpu-seconds"]["total"] == ex["alice_cpu_total"] == 1.7
    assert list(f["leaders"]["cpu-seconds"].items())[9] == (str(ex["leader_10th"][0]), ex["leader_10th"][1])
    # a success's nil reason is the "" key; end == start is a zero run time; task id 500 counts twice
    assert set(s["by-reason"]) == {"", "Killed by user"} and s["by-reason"]["Killed by user"]["count"] == 1
    assert s["by-user-and-reason"]["1"][""]["run-time-seconds"]["percentiles"]["50"] == 0.0
    assert s["by-user-and-reason"]["4"][""]["count"] + s["by-user-and-reason"]["4"]["Killed by user"]["count"] == \
        ex["twice_count"]
    assert "Command exited non-zero" in f["by-reason"] and "Command exited non-zero" not in s["by-reason"]
    assert s["by-user-and-reason"]["2"][""]["cpu-seconds"]["total"] == 0.0
    # the window: 400 (start == start_ms) in; 401 (start == end_ms), 402 (before) and 950 (past the bound) out
    assert s["by-user-and-reason"]["3"][""]["count"] == 1
    assert cases["the horizon itself"]["overall"]["count"] == ex["success_count"] + 3   # 401, 402 and 950 come in
    assert cases["nothing selected"]["overall"] == {}


def test_table_ops():
    ops = GOLDEN["ops"]
    running = {int(k): v for k, v in ops["running"].items()}
    h = Hr.History()
    assert not h.on
    for s in ops["steps"]:
        if s["op"] == "seed":
            h.seed(s["since"], s["rows"])
        elif s["op"] == "finish":
            h.finish(running, s["task_id"], s["end"], s["success"], s["reason"])
        else:
            h.advance(s["since"])
        assert [[r["task_id"], r["reason"], int(r["success"])] for r in h.rows] == s["want"], s["op"]
    with pytest.raises(ValueError):
        h.advance(h.since - 1)
    with pytest.raises(ValueError):   # a window before the horizon is refused
        Hr.answer([h], "success", h.since - 1, h.since + 10)
    with pytest.raises(ValueError):   # end before start
        h.finish({1: dict(user=0, start_time=h.since + 5, cpus=1.0, mem=1.0)}, [1], [h.since + 4], [0])
    h.reset()
    assert not h.on and h.rows == []
    with pytest.raises(ValueError):
        h.advance(0)
    with pytest.raises(ValueError):
        Hr.answer([h], "success", 0, 1)
    # while off, a finish keeps nothing
    h.finish(running, [803], [GOLDEN["since"] + 400], [1])
    assert h.rows == []


def test_device_restatement_matches_reference_on_every_window():
    """`answer` (the device call's restatement) and get_stats agree on shifted windows and bounds of the edges."""
    hs = edge_histories()
    inst = Hr.instances_of(hs)
    T0 = GOLDEN["edges"]["cases"][0]["request"]["end"] + 500
    for status in ("success", "failed"):
        for start, end in ((T0 - 60000, T0), (T0 - 9000, T0 - 5000), (T0 - 5000, T0 - 4999)):
            for lo, hi in ((0, 10 ** 6), (101, 500), (500, 501)):
                want = Hr.I.response_keys(Hr.get_stats(inst, status, start, end, lo, hi))
                got = cycle.instance_stats_response(Hr.engine_answer(hs, status, start, end, lo, hi),
                                                    user_name=str, reason_string=str)
                assert plain(got) == plain(want), (status, start, end, lo, hi)


def test_task_id_twice_in_one_handle_keeps_table_order():
    """A caller's divergence: one handle holds task id 7 twice.  The fold runs in table order after (task id,
    handle)."""
    rows = [dict(task_id=7, user=0, start=10, end=10 + 1000, cpus=c, mem=1.0, reason=-1, success=True)
            for c in (0.1, 0.3, 1.1, 0.2)]
    segs, _, _ = Hr.answer([seeded(rows, 0)], "success", 0, 100)
    assert segs[0][4][1] == ((0.1 + 0.3) + 1.1) + 0.2 == 1.7
