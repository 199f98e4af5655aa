"""The three periodic killers' sweeps restated in plain Python over row lists (cook_state_sweep's reference).

A running row is a dict with task_id, start (ms), max_runtime (ms, or None / -1: none), status ("running" or
"unknown"), cancelled, groups (its job's group codes) and pool (the index of the handle that holds it; 0 when absent).
A record is (group code, runtime in whole seconds); `runtime_s` makes one of a success's start and end.  A group is a
dict with kind ("none" or "quantile-deviation"), quantile, multiplier and n_jobs.
"""
import json
import os

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sweeps_golden.json")


def runtime_s(start, end):
    """Joda's in-seconds of the interval [start, end] in ms: the whole seconds, truncated (the interval throws for
    end < start)."""
    if end < start:
        raise ValueError("an interval that ends before it starts")
    return (end - start) // 1000


def _key(r):
    return (r["task_id"], r.get("pool", 0))


def lingering(rows, now, default_timeout_ms, max_timeout_ms):
    """get-lingering-tasks: running or unknown rows with now > start + min(max-runtime or the default, the max timeout),
    as (task id, pool) in ascending order."""
    out = []
    for r in rows:
        m = r.get("max_runtime")
        m = default_timeout_ms if m is None or m == -1 else m
        if now - r["start"] > min(m, max_timeout_ms):
            out.append(_key(r))
    return sorted(out)


def cancelled(rows):
    """killable-cancelled-tasks: the cancelled rows, running or unknown, as (task id, pool) in ascending order."""
    return sorted(_key(r) for r in rows if r.get("cancelled"))


def stragglers(rows, records, groups, now):
    """find-stragglers :quantile-deviation for every group of `groups` ({code: group}), as (group, task id, pool) in
    ascending order.  Raises ValueError for a running row of a checked group that starts after now (the reference's
    interval throws there once the group has enough successes; cook_state_sweep rejects it whatever the count)."""
    out = []
    for g, p in groups.items():
        if p["kind"] != "quantile-deviation":
            continue
        judged = [r for r in rows if g in r.get("groups", ()) and r.get("status", "running") == "running"]
        runtimes = [runtime_s(r["start"], now) for r in judged]   # before the count: ours, see the header
        idx = int((p["n_jobs"] - 1) * p["quantile"])
        done = sorted(rt for c, rt in records if c == g)
        if idx < 0 or len(done) <= idx:
            continue
        limit = done[idx] * p["multiplier"]
        out += [(g,) + _key(r) for r, s in zip(judged, runtimes) if float(s) > limit]
    return sorted(out)


# ---- the golden scenarios --------------------------------------------------------------------------------------
def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)


def scenario_inputs(sc):
    """rows, records and groups ({int code: group}) of a golden scenario."""
    rows = [dict(t, max_runtime=-1 if t["max_runtime"] is None else t["max_runtime"]) for t in sc["tasks"]]
    records = [(s["group"], runtime_s(s["start"], s["end"])) for s in sc["successes"]]
    groups = {int(g): p for g, p in sc["groups"].items()}
    return rows, records, groups


def check_answers(chk, linger, cancel, strag):
    """A golden check against swept lists: linger and cancel as task ids, strag as [group, task id] pairs."""
    for k, got in (("linger", linger), ("cancel", cancel), ("straggler", strag)):
        if k in chk:
            assert got == chk[k], (k, got, chk[k])
    if "linger_has" in chk:
        assert set(chk["linger_has"]) <= set(linger)
    if "linger_lacks" in chk:
        assert not set(chk["linger_lacks"]) & set(linger)
