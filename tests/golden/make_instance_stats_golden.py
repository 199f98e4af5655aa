"""Writes tests/golden/instance_stats_golden.json: the known answers of GET /stats/instances for running and unknown
instances.

The reference has no unit test of task_stats.clj; its integration tests (integration/tests/cook/test_multi_user.py
test_instance_stats_running, test_instance_stats_success) assert the response's shape, and the success test the
percentiles (numpy's "higher" percentile, which is the nearest rank at n = 3) and totals (to 7 places).  Those
assertions are transcribed here on running rows ("transcribed"), next to hand-computed edges:

"ranks": the 0-based nearest-rank positions ceil(p/100 * n) - 1 for p = 50 75 95 99 100, n = 1 .. 21 and 100, computed
with exact fractions and math.ceil (the restatement computes them in integers).

"edges": three handles (a, b, c) of running rows with their user code, reason code (-1: none, 1001 "Killed by user",
2003 "Task max runtime exceeded") and unknown fact, and one request per case with the reference's response and the
facts computed by hand:
  fold     alice's cpu-seconds in ascending task id are 0.1, 0.3, 1.1, 0.2 (one second each): the left fold is 1.7, the
           pairwise sum (0.1 + 0.3) + (1.1 + 0.2) and the sorted fold are 1.7000000000000002;
  window   a row starts at start_ms (in) and one at end_ms (out); a row inside the window has a task id past the
           entity-id bound (out);
  status   unknown rows sit beside the running ones and answer the status "unknown" alone;
  reasons  bob has a row without a reason, one killed by user and one past its max runtime;
  leaders  twelve more users, one row each of one second: cpu totals 12 .. 7, then three tied at 6.5 (users 22, 21, 20
           in task-id order), then 3, 2, 1.  Users 3 (50), bob (14) and user 4 (13) lead, so the tie falls on the tenth
           place, which goes to user 20; mem totals tie pairwise;
  zero     a row with zero cpus;
  twice    task id 500 is held by handles a and b (counted twice, a first).

Run from the repository root: python tests/golden/make_instance_stats_golden.py
"""
import json
import math
import os
import sys
from fractions import Fraction

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import instance_stats_ref as I  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "instance_stats_golden.json")
NOW = 1_700_000_100_000
T0 = 1_700_000_000_000
REASONS = {1001: "Killed by user", 2003: "Task max runtime exceeded"}


def ranks():
    return {str(n): [math.ceil(Fraction(p, 100) * n) - 1 for p in I.PCTS] for n in list(range(1, 22)) + [100]}


def row(t, user, start, cpus, mem, reason=-1, unknown=False, job=None):
    return dict(task_id=t, job_id=job or t + 1, user=user, start_time=start, cpus=cpus, mem=mem, reason=reason,
                unknown=unknown)


def transcribed():
    """test_instance_stats_running: five running instances of one user, no reason, the window [first start, last start
    + 1 ms).  test_instance_stats_success's value checks on three instances of cpus 0.10 / 0.11 / 0.12 and mem base,
    base + 1, base + 2 (base 512 here), running 1, 2 and 3 s at `now`."""
    run = [row(10 + k, 0, T0 + 1000 * k, 1.0, 512.0) for k in range(5)]
    req = dict(status="running", start=T0, end=T0 + 4000 + 1, now=NOW)
    three = [row(20 + k, 0, NOW - 1000 * (k + 1), 0.10 + 0.01 * k, 512.0 + k) for k in range(3)]
    rts = [(NOW - r["start_time"]) / 1000 for r in three]
    checks = {}
    for k, key in ((None, "run-time-seconds"), ("cpus", "cpu-seconds"), ("mem", "mem-seconds")):
        xs = [t if k is None else t * r[k] for t, r in zip(rts, three)]
        checks[key] = {"percentiles": {str(p): float(np.percentile(xs, p, method="higher")) for p in I.PCTS},
                       "total_approx": sum(xs)}
    return [{"name": "test_instance_stats_running", "handles": [run], "request": req,
             "count": 5, "user": 0},
            {"name": "test_instance_stats_success (running)", "handles": [three],
             "request": dict(status="running", start=NOW - 3000, end=NOW - 999, now=NOW), "count": 3, "user": 0,
             "checks": checks}]


def edges():
    a, b, c = [], [], []
    # alice (0): the fold on its last bit; one second each, ascending task id 100 .. 103
    for k, cpus in enumerate([0.1, 0.3, 1.1, 0.2]):
        a.append(row(100 + k, 0, NOW - 1000, cpus, 100.0 * (k + 1)))
    # bob (1): three reasons, in handle b
    b.append(row(200, 1, NOW - 2500, 2.0, 64.0))
    b.append(row(201, 1, NOW - 4000, 1.0, 32.0, reason=1001))
    b.append(row(202, 1, NOW - 10000, 0.5, 16.0, reason=2003))
    # carol (2): unknown rows, one with a reason; a row with zero cpus
    c.append(row(300, 2, NOW - 7000, 1.5, 10.0, unknown=True))
    c.append(row(301, 2, NOW - 3000, 0.5, 20.0, reason=1001, unknown=True))
    c.append(row(302, 2, NOW - 6000, 0.0, 30.0))
    # the window's edges and the entity-id bound: start_ms = NOW - 50000, end_ms = NOW - 500, task ids < 900
    a.append(row(400, 3, NOW - 50000, 1.0, 1.0))      # start == start_ms: in
    a.append(row(401, 3, NOW - 500, 1.0, 1.0))        # start == end_ms: out
    a.append(row(950, 3, NOW - 20000, 1.0, 1.0))      # in the window, past the bound: out
    a.append(row(402, 3, NOW - 50001, 1.0, 1.0))      # before the window: out
    # the same task id in two handles
    a.append(row(500, 4, NOW - 1000, 3.0, 7.0))
    b.append(row(500, 4, NOW - 2000, 5.0, 11.0, reason=1001))
    # twelve users, one row each, one second: three of them tied at the tenth cpu total; mem in pairs of equal totals
    codes = [10, 11, 12, 13, 14, 15, 22, 21, 20, 23, 24, 25]
    for k, cpus in enumerate([12.0, 11.0, 10.0, 9.0, 8.0, 7.0, 6.5, 6.5, 6.5, 3.0, 2.0, 1.0]):
        c.append(row(600 + k, codes[k], NOW - 1000, cpus, float(2 * (k // 2) + 1)))
    handles = {"a": a, "b": b, "c": c}
    win = dict(start=NOW - 50000, end=NOW - 500, lo=0, hi=900, now=NOW)
    cases = [dict(name="running", request=dict(status="running", **win)),
             dict(name="unknown", request=dict(status="unknown", **win)),
             dict(name="alice's window", request=dict(status="running", start=NOW - 1000, end=NOW - 999, lo=100, hi=104,
                                                      now=NOW)),
             dict(name="nothing selected", request=dict(status="unknown", start=NOW - 1000, end=NOW, lo=0, hi=900,
                                                        now=NOW))]
    return handles, cases


def hand_checks(want_running, want_alice):
    """The facts computed by hand, asserted on the restatement before they are written."""
    alice = want_alice["overall"]["cpu-seconds"]["total"]
    assert alice == 1.7 and (0.1 + 0.3) + (1.1 + 0.2) == 1.7000000000000002 and ((0.1 + 0.2) + 0.3) + 1.1 != 1.7
    o = want_running["overall"]
    # selected running rows: alice 4, bob 3, carol's zero-cpus row, 400, 500 twice, twelve users
    assert o["count"] == 4 + 3 + 1 + 1 + 2 + 12
    assert set(want_running["by-reason"]) == {None, 1001, 2003}
    assert set(want_running["by-user-and-reason"][1]) == {None, 1001, 2003}
    lc = list(want_running["leaders"]["cpu-seconds"].items())
    assert lc[:4] == [(3, 50.0), (1, 14.0), (4, 13.0), (10, 12.0)] and lc[9] == (20, 6.5) and len(lc) == 10
    assert 21 not in dict(lc) and 22 not in dict(lc)
    return {"count": o["count"], "alice_cpu_total": alice, "leader_10th": [20, 6.5],
            "bob_reasons": [-1, 1001, 2003], "twice_count": 2}


def main():
    handles, cases = edges()
    mirror = [{r["task_id"]: r for r in handles[k]} for k in ("a", "b", "c")]
    inst = I.instances_of(mirror)
    for case in cases:
        q = case["request"]
        want = I.get_stats(inst, q["status"], q["start"], q["end"], q["lo"], q["hi"], q["now"])
        case["want_raw"] = want
        case["want"] = I.response_keys({**want, "by-reason": {None if r is None else REASONS[r]: s
                                                              for r, s in want["by-reason"].items()},
                                        "by-user-and-reason": {u: {None if r is None else REASONS[r]: s
                                                                   for r, s in m.items()}
                                                               for u, m in want["by-user-and-reason"].items()}})
    expect = hand_checks(cases[0]["want_raw"], cases[2]["want_raw"])
    for case in cases:
        del case["want_raw"]
    tr = transcribed()
    for t in tr:
        q = t["request"]
        inst_t = I.instances_of([{r["task_id"]: r for r in t["handles"][0]}])
        got = I.get_stats(inst_t, q["status"], q["start"], q["end"], -(1 << 63), (1 << 63) - 1, q["now"])
        assert got["overall"]["count"] == t["count"]
        assert got["by-reason"][None]["count"] == t["count"]
        assert got["by-user-and-reason"][t["user"]][None]["count"] == t["count"]
        for key, chk in t.get("checks", {}).items():
            assert {str(p): v for p, v in got["overall"][key]["percentiles"].items()} == chk["percentiles"]
            assert round(got["overall"][key]["total"] - chk["total_approx"], 7) == 0
    out = {"ranks": ranks(), "transcribed": tr, "reasons": {str(k): v for k, v in REASONS.items()},
           "edges": {"handles": handles, "cases": cases, "expect": expect}}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=False)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
