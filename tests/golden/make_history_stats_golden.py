"""Writes tests/golden/history_stats_golden.json: the known answers of GET /stats/instances for success and failed
instances, answered from finished-instance histories.

"transcribed": the reference's integration tests test_instance_stats_failed and test_instance_stats_success
(integration/tests/cook/test_multi_user.py), without the name filter.  Three failed instances of cpus 0.1 / 0.2 / 0.4
and mem 32 / 64 / 128, all with the reason "Command exited non-zero" (not mea culpa); three successful ones of cpus
0.10 / 0.11 / 0.12 and mem 512 / 513 / 514 without a reason (the "" key).  The window is [first start, last start +
1 ms).  Run times are (end - start) / 1000 on off-grid milliseconds; the percentiles are util.percentile's nearest rank
(numpy's "higher" at n = 3) and the totals are checked to 7 places.

"edges": three handles (a, b, c) of finished rows, all seeded at horizon H0, and one request per case with the
reference's response, and facts computed by hand:
  fold     alice's successful cpu-seconds in ascending task id are 0.1, 0.3, 1.1, 0.2 (one second each): the left fold
           is 1.7, the pairwise sum 1.7000000000000002;
  instant  a row with end == start: run time 0.0;
  window   a row starts at start_ms (in), one at end_ms (out), one before; one inside has a task id past the bound;
  status   failed rows sit beside the successes and answer "failed" alone;
  leaders  twelve users of one failed second each: cpu totals 12 .. 7, then three tied at 6.5 (users 22, 21, 20 in
           task-id order), then 3, 2, 1; with users 3 (50), 1 (23) and 4 (13) leading, the tenth place is user 20's;
  zero     a row with zero cpus;
  twice    task id 500 is held by handles a and b (counted twice, a first).

"ops": one handle's table through seed, finish and advance: a finished row that started one ms before the horizon is
not kept, the one that started at it is; the reason of a finish is the given one or, when none is given, the running
row's fact; an advance to one ms past a row's start removes exactly that row.

Run from the repository root: python tests/golden/make_history_stats_golden.py
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import history_ref as Hr  # noqa: E402
import instance_stats_ref as I  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "history_stats_golden.json")
T0 = 1_700_000_000_000
H0 = T0 - 3_600_000
EXITED = 3001
REASONS = {1001: "Killed by user", 2003: "Task max runtime exceeded", EXITED: "Command exited non-zero"}


def row(t, user, start, run_ms, cpus, mem, success, reason=-1):
    return dict(task_id=t, user=user, start=start, end=start + run_ms, cpus=cpus, mem=mem, reason=reason,
                success=success)


def history(rows, since=H0):
    h = Hr.History()
    h.seed(since, rows)
    return h


def transcribed():
    failed = [row(10 + k, 0, T0 + 137 * k, ms, cpus, mem, False, EXITED)
              for k, (ms, cpus, mem) in enumerate(((353, 0.1, 32.0), (1421, 0.2, 64.0), (2467, 0.4, 128.0)))]
    success = [row(20 + k, 0, T0 + 211 * k, ms, 0.10 + 0.01 * k, 512.0 + k, True)
               for k, ms in enumerate((309, 1318, 2326))]
    out = []
    for name, rows, status, key in (("test_instance_stats_failed", failed, "failed", REASONS[EXITED]),
                                    ("test_instance_stats_success", success, "success", "")):
        rts = [(r["end"] - r["start"]) / 1000 for r in rows]
        checks = {}
        for k, m in ((None, "run-time-seconds"), ("cpus", "cpu-seconds"), ("mem", "mem-seconds")):
            xs = [t if k is None else t * r[k] for t, r in zip(rts, rows)]
            checks[m] = {"percentiles": {str(p): float(np.percentile(xs, p, method="higher")) for p in I.PCTS},
                         "total_approx": sum(xs)}
        req = dict(status=status, start=min(r["start"] for r in rows), end=max(r["start"] for r in rows) + 1)
        out.append({"name": name, "rows": rows, "since": H0, "request": req, "count": 3, "user": 0, "reason": key,
                    "checks": checks})
    return out


def edges():
    a, b, c = [], [], []
    for k, cpus in enumerate([0.1, 0.3, 1.1, 0.2]):                    # alice (0): the fold
        a.append(row(100 + k, 0, T0 - 5000, 1000, cpus, 100.0 * (k + 1), True))
    b.append(row(200, 1, T0 - 9000, 2500, 2.0, 64.0, True))             # bob (1): reasons
    b.append(row(201, 1, T0 - 8000, 4000, 1.0, 32.0, False, 1001))
    b.append(row(202, 1, T0 - 7000, 10000, 0.5, 16.0, False, 2003))
    b.append(row(203, 1, T0 - 6000, 0, 1.5, 8.0, True))                 # end == start
    c.append(row(300, 2, T0 - 7000, 7000, 0.5, 10.0, False, EXITED))    # carol (2)
    c.append(row(302, 2, T0 - 6000, 6000, 0.0, 30.0, True))             # zero cpus
    a.append(row(400, 3, T0 - 50000, 50000, 1.0, 1.0, True))            # start == start_ms: in
    a.append(row(401, 3, T0 - 500, 500, 1.0, 1.0, True))                # start == end_ms: out
    a.append(row(950, 3, T0 - 20000, 1000, 1.0, 1.0, True))             # past the bound: out
    a.append(row(402, 3, T0 - 50001, 1000, 1.0, 1.0, True))             # before the window: out
    a.append(row(500, 4, T0 - 3000, 1000, 3.0, 7.0, True))              # task id 500 in two handles
    b.append(row(500, 4, T0 - 4000, 2000, 5.0, 11.0, True, 1001))
    codes = [10, 11, 12, 13, 14, 15, 22, 21, 20, 23, 24, 25]
    for k, cpus in enumerate([12.0, 11.0, 10.0, 9.0, 8.0, 7.0, 6.5, 6.5, 6.5, 3.0, 2.0, 1.0]):
        c.append(row(600 + k, codes[k], T0 - 2000, 1000, cpus, float(2 * (k // 2) + 1), False))
    # the leaders' case: users 3 and 4 lead on failed rows too
    c.append(row(700, 3, T0 - 30000, 25000, 2.0, 1.0, False))
    c.append(row(701, 1, T0 - 30000, 14000, 1.0, 1.0, False))
    c.append(row(702, 4, T0 - 30000, 13000, 1.0, 1.0, False, 1001))
    handles = {"a": a, "b": b, "c": c}
    win = dict(start=T0 - 50000, end=T0 - 500, lo=0, hi=900)
    cases = [dict(name="success", request=dict(status="success", **win)),
             dict(name="failed", request=dict(status="failed", **win)),
             dict(name="alice's window", request=dict(status="success", start=T0 - 5000, end=T0 - 4999, lo=100, hi=104)),
             dict(name="the horizon itself", request=dict(status="success", start=H0, end=T0, lo=0, hi=1000)),
             dict(name="nothing selected", request=dict(status="failed", start=T0 - 1000, end=T0, lo=0, hi=900))]
    return handles, cases


def ops():
    """One handle: seed at H0, finish three running rows (one started at H0 - 1), advance past one row's start."""
    running = {800: dict(user=5, start_time=H0 - 1, cpus=1.0, mem=2.0, reason=-1),
               801: dict(user=5, start_time=H0, cpus=1.0, mem=2.0, reason=1001),
               802: dict(user=6, start_time=H0 + 10, cpus=0.5, mem=4.0, reason=1001),
               803: dict(user=6, start_time=H0 + 20, cpus=0.5, mem=4.0, reason=-1)}
    seed = [row(790, 5, H0 + 5, 100, 1.0, 1.0, True)]
    steps = [dict(op="seed", since=H0, rows=seed),
             dict(op="finish", task_id=[800, 801], end=[H0 + 100, H0 + 200], success=[0, 1], reason=None),
             dict(op="finish", task_id=[802, 803], end=[H0 + 300, H0 + 400], success=[0, 0], reason=[EXITED, -1]),
             dict(op="advance", since=H0 + 1)]
    h = Hr.History()
    for s in steps:
        if s["op"] == "seed":
            h.seed(s["since"], s["rows"])
        elif s["op"] == "finish":
            h.finish(running, s["task_id"], s["end"], s["success"], s["reason"])
        else:
            h.advance(s["since"])
        s["want"] = [[r["task_id"], r["reason"], int(r["success"])] for r in h.rows]
    # by hand: 800 started before the horizon; 801 keeps its fact 1001; 802 takes the given reason; the advance to
    # H0 + 1 removes exactly 801 (start H0)
    assert steps[1]["want"] == [[790, -1, 1], [801, 1001, 1]]
    assert steps[2]["want"] == [[790, -1, 1], [801, 1001, 1], [802, EXITED, 0], [803, -1, 0]]
    assert steps[3]["want"] == [[790, -1, 1], [802, EXITED, 0], [803, -1, 0]]
    return {"running": {str(k): v for k, v in running.items()}, "steps": steps}


def named(want):
    """The reference's response with the reason codes named, as the shim's dictionary names them."""
    name = lambda r: None if r is None else REASONS[r]
    return I.response_keys({**want, "by-reason": {name(r): s for r, s in want["by-reason"].items()},
                            "by-user-and-reason": {u: {name(r): s for r, s in m.items()}
                                                   for u, m in want["by-user-and-reason"].items()}})


def hand_checks(cases):
    w = {c["name"]: c["raw"] for c in cases}
    assert w["alice's window"]["overall"]["cpu-seconds"]["total"] == 1.7
    assert (0.1 + 0.3) + (1.1 + 0.2) == 1.7000000000000002
    s = w["success"]["overall"]
    # alice 4, bob's 200 and 203, carol's 302, 400, 500 twice
    assert s["count"] == 4 + 2 + 1 + 1 + 2
    assert w["success"]["by-user-and-reason"][1][None]["run-time-seconds"]["percentiles"][50] == 0.0
    assert w["success"]["by-user-and-reason"][2][None]["cpu-seconds"]["total"] == 0.0
    f = w["failed"]
    lc = list(f["leaders"]["cpu-seconds"].items())
    assert lc[:4] == [(3, 50.0), (1, 14.0 + 4.0 + 5.0), (4, 13.0), (10, 12.0)] and lc[9] == (20, 6.5)
    assert 21 not in dict(lc) and 22 not in dict(lc) and len(lc) == 10
    assert set(f["by-reason"]) == {None, 1001, 2003, EXITED}
    assert w["nothing selected"]["overall"] == {}
    return {"success_count": s["count"], "alice_cpu_total": 1.7, "leader_10th": [20, 6.5], "twice_count": 2}


def main():
    handles, cases = edges()
    hs = [history(handles[k]) for k in ("a", "b", "c")]
    inst = Hr.instances_of(hs)
    for case in cases:
        q = case["request"]
        case["raw"] = Hr.get_stats(inst, q["status"], q["start"], q["end"], q["lo"], q["hi"])
        case["want"] = named(case["raw"])
    expect = hand_checks(cases)
    for case in cases:
        del case["raw"]
    tr = transcribed()
    for t in tr:
        q = t["request"]
        got = Hr.get_stats(Hr.instances_of([history(t["rows"])]), q["status"], q["start"], q["end"], -(1 << 63),
                           (1 << 63) - 1)
        assert got["overall"]["count"] == t["count"]
        for key, chk in t["checks"].items():
            assert {str(p): v for p, v in got["overall"][key]["percentiles"].items()} == chk["percentiles"]
            assert round(got["overall"][key]["total"] - chk["total_approx"], 7) == 0
    out = {"transcribed": tr, "reasons": {str(k): v for k, v in REASONS.items()}, "since": H0,
           "edges": {"handles": handles, "cases": cases, "expect": expect}, "ops": ops()}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=False)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
