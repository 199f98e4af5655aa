"""CPU: the restatement of GET /stats/instances (instance_stats_ref) and cycle.instance_stats_response against the known
answers in tests/golden/instance_stats_golden.json: the nearest-rank positions, the reference's integration assertions
transcribed on running rows, and the hand-computed edges (a left fold on its last bit, the window's and the entity-id
bound's edges, running and unknown rows, reasons, a tie at the tenth leader, zero cpus, a task id in two handles)."""
import json
import os

import pytest

import instance_stats_ref as I
from cook_b200 import cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instance_stats_golden.json")))
REASONS = {int(k): v for k, v in GOLDEN["reasons"].items()}


def plain(x):
    return json.loads(json.dumps(x))


def mirror(rows_by_handle):
    return [{r["task_id"]: r for r in rows} for rows in rows_by_handle]


def edge_mirror():
    h = GOLDEN["edges"]["handles"]
    return mirror([h[k] for k in ("a", "b", "c")])


def response(handles, q):
    a = I.engine_answer(handles, q["now"], q["status"], q["start"], q["end"], q.get("lo", -(1 << 63)),
                        q.get("hi", (1 << 63) - 1))
    return cycle.instance_stats_response(a, user_name=str, reason_string=REASONS.get)


def test_ranks():
    for n, want in GOLDEN["ranks"].items():
        assert [I.rank(int(n), p) for p in I.PCTS] == want, n
    # where ceil moves: p = 50 at odd and even n, p = 95 and 99 below and at n = 20 and 100
    assert GOLDEN["ranks"]["1"] == [0, 0, 0, 0, 0] and GOLDEN["ranks"]["2"] == [0, 1, 1, 1, 1]
    assert GOLDEN["ranks"]["20"] == [9, 14, 18, 19, 19] and GOLDEN["ranks"]["21"] == [10, 15, 19, 20, 20]
    assert GOLDEN["ranks"]["100"] == [49, 74, 94, 98, 99]
    assert I.percentile([], 50) is None and I.percentile([1.0], 0) is None and I.percentile([1.0], 101) is None


@pytest.mark.parametrize("k", range(len(GOLDEN["transcribed"])))
def test_transcribed(k):
    t = GOLDEN["transcribed"][k]
    q = t["request"]
    hs = mirror(t["handles"])
    got = I.get_stats(I.instances_of(hs), q["status"], q["start"], q["end"], -(1 << 63), (1 << 63) - 1, q["now"])
    assert got["overall"]["count"] == got["by-reason"][None]["count"] == t["count"]
    assert got["by-user-and-reason"][t["user"]][None]["count"] == t["count"]
    for key, chk in t.get("checks", {}).items():
        assert plain(got["overall"][key]["percentiles"]) == chk["percentiles"]
        assert got["overall"][key]["total"] == pytest.approx(chk["total_approx"], abs=1e-7)
    # the response built from the device call's restatement is the reference's, the nil reason under ""
    r = response(hs, q)
    assert plain(r) == plain(I.response_keys(got))
    assert r["by-reason"][""]["count"] == r["by-user-and-reason"][str(t["user"])][""]["count"] == t["count"]


@pytest.mark.parametrize("k", range(len(GOLDEN["edges"]["cases"])))
def test_edges(k):
    case = GOLDEN["edges"]["cases"][k]
    q = case["request"]
    hs = edge_mirror()
    got = I.get_stats(I.instances_of(hs, reason_of=lambda c: None if c == -1 else REASONS[c]), q["status"], q["start"],
                      q["end"], q["lo"], q["hi"], q["now"])
    assert plain(I.response_keys(got)) == case["want"]
    r = response(hs, q)
    assert plain(r) == case["want"]
    for m in ("cpu-seconds", "mem-seconds"):   # the leaders' order, not only their map
        assert [(str(u), t) for u, t in got["leaders"][m].items()] == list(r["leaders"][m].items())


def test_edge_facts():
    ex = GOLDEN["edges"]["expect"]
    cases = {c["name"]: c for c in GOLDEN["edges"]["cases"]}
    run, unk = cases["running"]["want"], cases["unknown"]["want"]
    assert run["overall"]["count"] == ex["count"]
    assert cases["alice's window"]["want"]["overall"]["cpu-seconds"]["total"] == ex["alice_cpu_total"] == 1.7
    assert list(run["leaders"]["cpu-seconds"].items())[9] == (str(ex["leader_10th"][0]), ex["leader_10th"][1])
    assert set(run["by-user-and-reason"]["1"]) == {"", "Killed by user", "Task max runtime exceeded"}
    assert run["by-user-and-reason"]["4"]["Killed by user"]["count"] + run["by-user-and-reason"]["4"][""]["count"] == \
        ex["twice_count"]
    # the unknown rows answer their status alone; the zero-cpus row is a zero product
    assert unk["overall"]["count"] == 2 and set(unk["by-user-and-reason"]) == {"2"}
    assert run["by-user-and-reason"]["2"][""]["cpu-seconds"]["total"] == 0.0
    # the window: 400 (start == start_ms) in; 401 (start == end_ms), 402 (before) and 950 (past the bound) out
    assert run["by-user-and-reason"]["3"][""]["count"] == 1
    assert cases["nothing selected"]["want"] == {"by-reason": {}, "by-user-and-reason": {}, "leaders": {
        "cpu-seconds": {}, "mem-seconds": {}}, "overall": {}}


def test_device_restatement_matches_reference_on_every_window():
    """`answer` (the device call's restatement) and get_stats agree on shifted windows and bounds of the edges."""
    hs = edge_mirror()
    inst = I.instances_of(hs)
    now = GOLDEN["edges"]["cases"][0]["request"]["now"]
    for status in ("running", "unknown"):
        for start, end in ((now - 60000, now), (now - 5000, now - 1000), (now - 2500, now - 2499)):
            for lo, hi in ((0, 10 ** 6), (101, 500), (500, 501)):
                want = I.response_keys(I.get_stats(inst, status, start, end, lo, hi, now))
                a = I.engine_answer(hs, now, status, start, end, lo, hi)
                got = cycle.instance_stats_response(a, user_name=str, reason_string=str)
                assert plain(got) == plain(want), (status, start, end, lo, hi)


def test_start_after_now():
    hs = edge_mirror()
    now = GOLDEN["edges"]["cases"][0]["request"]["now"]
    with pytest.raises(ValueError):
        I.answer(hs, now - 1500, "running", now - 60000, now)
    with pytest.raises(ValueError):
        I.get_stats(I.instances_of(hs), "running", now - 60000, now, 0, 10 ** 6, now - 1500)
    # a row that starts after now but is not selected does not matter
    assert I.answer(hs, now - 1500, "running", now - 60000, now - 2000)[0]
