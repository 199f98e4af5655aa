"""Plain-Python restatement of GET /stats/instances (task-stats/get-stats, task_stats.clj) and of
cook_state_instance_stats.

The reference's functions over plain instance values {task_id, user, start (ms), cpus, mem, reason (None: none),
status}: get-tasks (the entity-id bound as [task_id_lo, task_id_hi), then the start window), task->task-entry with one
`now`, percentile / percentiles (nearest rank), generate-stats and generate-all-stats, in the JSON response's key names
with the percentiles keyed by int.  The nil reason stays None here; `response_keys` turns it into the "" key the JSON
encoder writes for it.  The leaders' order among equal totals is the reference's hash order; here, as in the device
call, it is ascending user.

`answer` is what cook_state_instance_stats returns over a host mirror of its handles' running rows, one {task id: row}
per handle with row {user, start_time, cpus, mem, reason (code, -1: none), unknown}: the selection in ascending (task
id, handle), per segment (kind, user, reason) the count, each metric's left fold from +0.0 in that order and its five
nearest-rank percentiles, and the leaders.
"""
import functools
import operator

PCTS = (50, 75, 95, 99, 100)
METRICS = ("run-time-seconds", "cpu-seconds", "mem-seconds")   # by abi.IS_RUN_TIME, IS_CPU, IS_MEM
OVERALL, REASON, USER_REASON = 0, 1, 2
LEADERS = 10
SEG_BYTES = 164   # kind, user, reason, count, three totals, fifteen percentiles
LEADER_BYTES = 24   # (user, total) for cpu and for mem


# ---- the reference ------------------------------------------------------------------------------------------------
def get_tasks(instances, status, start_ms, end_ms, task_id_lo, task_id_hi):
    """The instances of `status` in [task_id_lo, task_id_hi) in ascending task id (the avet seek), then the start
    window [start_ms, end_ms)."""
    sel = sorted((i for i in instances if i["status"] == status and task_id_lo <= i["task_id"] < task_id_hi),
                 key=lambda i: i["task_id"])
    return [i for i in sel if start_ms <= i["start"] < end_ms]


def task_entry(inst, now):
    """task->task-entry with the running instance's end = now.  Joda's interval throws when now < start."""
    if now < inst["start"]:
        raise ValueError("the interval's end is before its start")
    rt = (now - inst["start"]) / 1000.0
    return {"cpus": inst["cpus"], "mem": inst["mem"], "cpu-seconds": rt * inst["cpus"], "mem-seconds": rt * inst["mem"],
            "reason": inst.get("reason"), "run-time-seconds": rt, "user": inst["user"]}


def rank(n, p):
    """The 0-based position `percentile` reads: ceil(p/100 * n) - 1, the ratio exact."""
    return (p * n + 99) // 100 - 1


def percentile(coll, p):
    if not coll or p <= 0 or p > 100:
        return None
    return coll[rank(len(coll), p)]


def percentiles(coll, *ps):
    s = sorted(coll)
    return {p: percentile(s, p) for p in ps}


def generate_stats(entries):
    if not entries:
        return {}
    stats = lambda xs: {"percentiles": percentiles(xs, *PCTS), "total": functools.reduce(operator.add, xs)}
    out = {"count": len(entries)}
    for k in ("cpu-seconds", "mem-seconds", "run-time-seconds"):
        out[k] = stats([e[k] for e in entries])
    return out


def _group_by(entries, k):
    by = {}
    for e in entries:
        by.setdefault(e[k], []).append(e)
    return by


def generate_all_stats(tasks, now):
    entries = [task_entry(t, now) for t in tasks]
    by_user = _group_by(entries, "user")
    user_stats = {u: generate_stats(es) for u, es in by_user.items()}

    def leaders(k):
        ranked = sorted(((st[k]["total"], u) for u, st in user_stats.items()), key=lambda x: (-x[0], x[1]))
        return {u: n for n, u in ranked[:LEADERS]}

    return {"by-reason": {r: generate_stats(es) for r, es in _group_by(entries, "reason").items()},
            "by-user-and-reason": {u: {r: generate_stats(rs) for r, rs in _group_by(es, "reason").items()}
                                   for u, es in by_user.items()},
            "leaders": {"cpu-seconds": leaders("cpu-seconds"), "mem-seconds": leaders("mem-seconds")},
            "overall": generate_stats(entries)}


def get_stats(instances, status, start_ms, end_ms, task_id_lo, task_id_hi, now):
    return generate_all_stats(get_tasks(instances, status, start_ms, end_ms, task_id_lo, task_id_hi), now)


def response_keys(x):
    """The response as the JSON encoder writes it: the nil reason key becomes "", every key a string."""
    if isinstance(x, dict):
        return {("" if k is None else str(k)): response_keys(v) for k, v in x.items()}
    return x


# ---- cook_state_instance_stats over a host mirror -----------------------------------------------------------------
def selected(handles, now, status, start_ms, end_ms, task_id_lo, task_id_hi):
    """[(task id, handle index, row)] of the selected rows in ascending (task id, handle); ValueError when one starts
    after now (the call's COOK_E_BADARG)."""
    sel = sorted(((t, p, r) for p, run in enumerate(handles) for t, r in run.items()
                  if bool(r.get("unknown")) == (status == "unknown") and task_id_lo <= t < task_id_hi
                  and start_ms <= r["start_time"] < end_ms), key=lambda x: (x[0], x[1]))
    if any(r["start_time"] > now for _, _, r in sel):
        raise ValueError("a selected task starts after now")
    return sel


def metrics(r, now):
    rt = (now - r["start_time"]) / 1000.0
    return (rt, rt * r["cpus"], rt * r["mem"])


def answer(handles, now, status, start_ms, end_ms, task_id_lo=-(1 << 63), task_id_hi=(1 << 63) - 1):
    """([(kind, user, reason, count, totals (3), percentiles (3 x 5))], leaders_cpu, leaders_mem) in the call's
    order; leaders as [(user, total)].  status: "running" or "unknown"."""
    segs, users = {}, {}
    for t, p, r in selected(handles, now, status, start_ms, end_ms, task_id_lo, task_id_hi):
        m = metrics(r, now)
        reason = r.get("reason", -1)
        for key in ((OVERALL, -1, -1), (REASON, -1, reason), (USER_REASON, r["user"], reason)):
            segs.setdefault(key, []).append(m)
        users.setdefault(r["user"], []).append(m)
    out = []
    for key, ms in sorted(segs.items()):
        totals, pct = [], []
        for k in range(3):
            acc = 0.0
            for x in ms:   # the left fold, ascending (task id, handle)
                acc = acc + x[k]
            totals.append(acc)
            s = sorted(x[k] for x in ms)
            pct.append([s[rank(len(s), q)] for q in PCTS])
        out.append((*key, len(ms), totals, pct))

    def lead(k):
        tot = []
        for u, ms in users.items():
            acc = 0.0
            for x in ms:
                acc = acc + x[k]
            tot.append((u, acc))
        return sorted(tot, key=lambda x: (-x[1], x[0]))[:LEADERS]

    return out, lead(1), lead(2)


def d2h_bytes(segs, leaders, any_selected):
    return 8 + ((8 + SEG_BYTES * len(segs) + LEADER_BYTES * len(leaders)) if any_selected else 0)


def instances_of(handles, status_of=lambda r: "unknown" if r.get("unknown") else "running", reason_of=None):
    """The instances get_stats reads, from the mirror: one per row of every handle (a task id two handles hold counts
    twice, as the call counts it).  reason_of(code) gives the reason string (default: the code, None for -1)."""
    reason_of = reason_of or (lambda c: None if c == -1 else c)
    return [{"task_id": t, "user": r["user"], "start": r["start_time"], "cpus": r["cpus"], "mem": r["mem"],
             "reason": reason_of(r.get("reason", -1)), "status": status_of(r)}
            for run in handles for t, r in run.items()]


def engine_answer(handles, now, status, start_ms, end_ms, task_id_lo=-(1 << 63), task_id_hi=(1 << 63) - 1):
    """`answer` in engine.state_instance_stats' shape (numpy columns), for cycle.instance_stats_response on the CPU."""
    import numpy as np
    segs, lc, lm = answer(handles, now, status, start_ms, end_ms, task_id_lo, task_id_hi)
    col = lambda i, dt: np.array([s[i] for s in segs], dt)
    return {"kind": col(0, np.int32), "user": col(1, np.int32), "reason": col(2, np.int32), "count": col(3, np.int64),
            "total": np.array([s[4] for s in segs], np.float64).reshape(-1, 3),
            "pct": np.array([s[5] for s in segs], np.float64).reshape(-1, 3, 5), "leaders_cpu": lc, "leaders_mem": lm}
