"""Writes sweeps_golden.json: the known answers of the reference scheduler's tests of its three periodic killers,
transcribed, and hand-computed cases at the edges of the same rules.

Each scenario lists running tasks (start time, the job's max-runtime or None, status, cancelled flag, group list),
successful instances (group, start, end) and groups (kind, quantile, multiplier, n_jobs: the group's jobs in every
state).  Each check gives now and the two lingering timeouts in ms, and what the reference returns there: a list given
exactly, or (`*_has` / `*_lacks`) the task ids a test only asserts membership of.  Run: python make_sweeps_golden.py
"""
import json
import os
from datetime import datetime, timezone

H, MIN, S = 3_600_000, 60_000, 1000
LONG_MAX = 2 ** 63 - 1


def ms(iso):
    return int(datetime.fromisoformat(iso).replace(tzinfo=timezone.utc).timestamp() * 1000)


def task(tid, start, max_runtime=None, status="running", cancelled=False, groups=()):
    return dict(task_id=tid, start=start, max_runtime=max_runtime, status=status, cancelled=cancelled,
                groups=list(groups))


def qd(quantile, multiplier, n_jobs):
    return dict(kind="quantile-deviation", quantile=quantile, multiplier=multiplier, n_jobs=n_jobs)


def check(now, timeout=None, default=None, maximum=None, **want):
    return dict(now=now, default_timeout_ms=default if default is not None else timeout,
                max_timeout_ms=maximum if maximum is not None else timeout, **want)


def scenarios():
    out = []
    # test-get-lingering-tasks (scheduler test): max-runtimes Long/MAX, 60 s, 30 s (its boundary is now), 10 s and
    # 64 days (past Integer/MAX ms)
    now = ms("2015-01-05T00:00:30")
    out.append(dict(name="get-lingering-tasks", tasks=[
        task(1, ms("2015-01-01T00:00:00"), LONG_MAX), task(2, ms("2015-01-04T00:00:00"), 60000),
        task(3, ms("2015-01-05T00:00:00"), 30000), task(4, ms("2015-01-05T00:00:00"), 10000),
        task(5, ms("2015-01-01T00:00:00"), 64 * 24 * H)], successes=[], groups={}, checks=[
        check(now, 120 * H, linger=[2, 4]),
        check(ms("2015-02-05T00:00:30"), 10 ** 4 * H, linger_lacks=[5]),   # next month, 1e4 hours
        check(ms("2016-01-05T00:00:30"), 10 ** 5 * H, linger_has=[5])]))  # next year, 1e5 hours
    # test-kill-lingering-tasks: timeout-hours 4 (both timeouts), no max-runtime; an unknown and a running task
    # started 5 h ago are killed, the one started 3 h ago is not
    now = ms("2020-06-01T12:00:00")
    out.append(dict(name="kill-lingering-tasks", tasks=[
        task(1, now - 5 * H, status="unknown"), task(2, now - 5 * H), task(3, now - 3 * H)],
        successes=[], groups={}, checks=[check(now, 4 * H, linger=[1, 2])]))
    # test-find-stragglers (group test), at a fixed now; a success ran from 3 h ago to 2 h ago
    now = ms("2020-06-01T12:00:00")
    ok = dict(start=now - 3 * H, end=now - 2 * H)
    out.append(dict(name="find-stragglers: no straggler-handling", tasks=[task(1, now - 30 * MIN, groups=[0])],
                    successes=[dict(group=0, **ok)], groups={0: dict(kind="none", n_jobs=2)},
                    checks=[check(now, 1000 * H, straggler=[])]))
    out.append(dict(name="find-stragglers: quantile deviation, no stragglers", tasks=[task(1, now - 90 * MIN, groups=[0])],
                    successes=[dict(group=0, **ok)], groups={0: qd(0.5, 2.0, 2)},
                    checks=[check(now, 1000 * H, straggler=[])]))
    out.append(dict(name="find-stragglers: quantile deviation, stragglers found", tasks=[
        task(7, now - 100 * MIN, groups=[0]), task(8, now - 190 * MIN, groups=[0]), task(9, now - 121 * MIN, groups=[0])],
        successes=[dict(group=0, **ok)] * 6, groups={0: qd(0.5, 2.0, 9)},
        checks=[check(now, 1000 * H, straggler=[[0, 8], [0, 9]])]))
    # jobs a (running 3 h), b (running 190 min, and a success) and c (no instance)
    out.append(dict(name="find-stragglers: not enough complete", tasks=[
        task(1, now - 3 * H, groups=[0]), task(2, now - 190 * MIN, groups=[0])],
        successes=[dict(group=0, **ok)], groups={0: qd(0.5, 2.0, 3)}, checks=[check(now, 1000 * H, straggler=[])]))
    # ---- hand-computed edges of the same rules
    succ = lambda g, *secs: [dict(group=g, start=now - 10 * H, end=now - 10 * H + s * S) for s in secs]
    # idx = (int)(7 * 0.3) = 2: the third smallest runtime (30 s) is the target, times 1.0
    out.append(dict(name="idx truncation", tasks=[task(1, now - 30 * S, groups=[0]), task(2, now - 31 * S, groups=[0])],
                    successes=succ(0, 40, 10, 30, 20), groups={0: qd(0.3, 1.0, 8)},
                    checks=[check(now, 1000 * H, straggler=[[0, 2]])]))
    # idx = (int)(4 * 0.5) = 2: two successes find nothing (group 0), three find the long runner (group 1)
    out.append(dict(name="success count at idx and idx + 1", tasks=[
        task(1, now - 5 * H, groups=[0, 1])], successes=succ(0, 60, 60) + succ(1, 60, 60, 60),
        groups={0: qd(0.5, 2.0, 5), 1: qd(0.5, 2.0, 5)}, checks=[check(now, 1000 * H, straggler=[[1, 1]])]))
    # limit 3600 * 2 = 7200 s: 7200 s is not a straggler, 7201 s is; 7200.999 s runs 7200 whole seconds, and a
    # success of 3600.999 s counts 3600
    out.append(dict(name="limit boundary and whole seconds", tasks=[
        task(1, now - 7200 * S, groups=[0]), task(2, now - 7201 * S, groups=[0]), task(3, now - 7200999, groups=[0])],
        successes=[dict(group=0, start=now - 10 * H, end=now - 10 * H + 3600999)], groups={0: qd(0.0, 2.0, 1)},
        checks=[check(now, 1000 * H, straggler=[[0, 2]])]))
    # limit 3601 * 2.5 = 9002.5 s
    out.append(dict(name="non-integer limit", tasks=[task(1, now - 9002 * S, groups=[0]), task(2, now - 9003 * S, groups=[0])],
                    successes=succ(0, 3601), groups={0: qd(1.0, 2.5, 1)},
                    checks=[check(now, 1000 * H, straggler=[[0, 2]])]))
    # an unknown task is not judged as a straggler, a running task in two checked groups is judged in each
    out.append(dict(name="status and several groups", tasks=[
        task(1, now - 5 * H, status="unknown", groups=[0]), task(2, now - 5 * H, groups=[0, 2]),
        task(3, now - 5 * H, groups=[1])], successes=succ(0, 60) + succ(2, 60) + succ(1, 60),
        groups={0: qd(0.0, 2.0, 1), 1: dict(kind="none", n_jobs=1), 2: qd(0.0, 2.0, 1)},
        checks=[check(now, 1000 * H, straggler=[[0, 2], [2, 2]])]))
    # max-runtime 10 h capped by a max timeout of 4 h; no max-runtime takes the default of 2 h
    out.append(dict(name="lingering caps and defaults", tasks=[
        task(1, now - 5 * H, 10 * H), task(2, now - 3 * H), task(3, now - 1 * H), task(4, now - 3 * H, 6 * H)],
        successes=[], groups={}, checks=[check(now, default=2 * H, maximum=4 * H, linger=[1, 2])]))
    # cancelled, running or unknown
    out.append(dict(name="cancelled", tasks=[
        task(5, now - H, cancelled=True), task(3, now - H, status="unknown", cancelled=True), task(4, now - H)],
        successes=[], groups={}, checks=[check(now, 1000 * H, cancel=[3, 5])]))
    return out


if __name__ == "__main__":
    doc = {"_source": "test/cook/test/scheduler/scheduler.clj test-get-lingering-tasks and test-kill-lingering-tasks, "
                      "and test/cook/test/group.clj test-find-stragglers, of the reference scheduler, transcribed at a "
                      "fixed now; the scenarios after them are hand-computed edges of the same rules",
           "scenarios": scenarios()}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sweeps_golden.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
