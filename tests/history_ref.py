"""Plain-Python restatement of a handle's finished-instance history and of cook_state_history_stats.

`History` is the table: rows {task_id, user, start, end, cpus, mem, reason (code, -1: none), success} in arrival order,
a horizon `since` and an on flag.  `seed` replaces it, `finish` appends the finished running rows whose start is at or
after the horizon (the reason given, or else the running row's reason fact), `advance` raises the horizon and drops
the rows that start before it, `reset` empties it and turns it off.

The stats reuse instance_stats_ref: the reference side through generate_all_stats, the device side through `answer`,
both with run time = end - start.  Each row is handed to them with its start moved to -(end - start) and one now of 0,
so that (now - start) is exactly end - start; the selection (status, id bounds, start window) is made here on the true
start.  A task id one handle holds twice stays two rows in table order, which is the call's last sort key.
"""
import instance_stats_ref as I

SUCCESS, FAILED = "success", "failed"


class History:
    def __init__(self):
        self.on, self.since, self.rows = False, 0, []

    def seed(self, since, rows):
        self.on, self.since, self.rows = True, since, [dict(r) for r in rows]

    def finish(self, running, task_ids, end, success, reason=None):
        """running {task id: row with user, start_time, cpus, mem, reason}: the finished rows, in batch order."""
        for i, t in enumerate(task_ids):
            r = running[t]
            if end[i] < r["start_time"]:
                raise ValueError("a row that ends before its start")
            if self.on and r["start_time"] >= self.since:
                self.rows.append(dict(task_id=t, user=r["user"], start=r["start_time"], end=end[i], cpus=r["cpus"],
                                      mem=r["mem"], reason=r.get("reason", -1) if reason is None else reason[i],
                                      success=bool(success[i])))

    def advance(self, since):
        if not self.on or since < self.since:
            raise ValueError("history off, or since below the horizon")
        self.since = since
        self.rows = [r for r in self.rows if r["start"] >= since]

    def reset(self):
        self.on, self.since, self.rows = False, 0, []


def _selected(r, status, start_ms, end_ms, lo, hi):
    return r["success"] == (status == SUCCESS) and lo <= r["task_id"] < hi and start_ms <= r["start"] < end_ms


def _moved(r):
    """The row as instance_stats_ref reads it at now = 0: (0 - start) / 1000.0 is (end - start) / 1000.0."""
    return {"user": r["user"], "start_time": -(r["end"] - r["start"]), "cpus": r["cpus"], "mem": r["mem"],
            "reason": r["reason"]}


class _Rows:
    """One handle's selected rows as (task id, row) pairs in table order; `answer` sorts them stably by (task id,
    handle), so a task id held twice keeps its table order."""

    def __init__(self, pairs):
        self.pairs = pairs

    def items(self):
        return self.pairs


def check_window(histories, start_ms):
    if any(not h.on or h.since > start_ms for h in histories):
        raise ValueError("a history that is off, or a window before its horizon")


def answer(histories, status, start_ms, end_ms, lo=-(1 << 63), hi=(1 << 63) - 1):
    """cook_state_history_stats over the histories: instance_stats_ref.answer's shape."""
    check_window(histories, start_ms)
    views = [_Rows([(r["task_id"], _moved(r)) for r in h.rows if _selected(r, status, start_ms, end_ms, lo, hi)])
             for h in histories]
    return I.answer(views, 0, "running", -(1 << 63), 1)


def engine_answer(histories, status, start_ms, end_ms, lo=-(1 << 63), hi=(1 << 63) - 1):
    """`answer` in engine.state_history_stats' shape, for cycle.instance_stats_response on the CPU."""
    import numpy as np
    segs, lc, lm = answer(histories, status, start_ms, end_ms, lo, hi)
    col = lambda i, dt: np.array([s[i] for s in segs], dt)
    return {"kind": col(0, np.int32), "user": col(1, np.int32), "reason": col(2, np.int32), "count": col(3, np.int64),
            "total": np.array([s[4] for s in segs], np.float64).reshape(-1, 3),
            "pct": np.array([s[5] for s in segs], np.float64).reshape(-1, 3, 5), "leaders_cpu": lc, "leaders_mem": lm}


def instances_of(histories, reason_of=None):
    """The finished instances get_stats reads, from the histories, with their status, and their start moved as in
    `_moved` (the reference's run time with the instance's own end)."""
    reason_of = reason_of or (lambda c: None if c == -1 else c)
    return [{"task_id": r["task_id"], "user": r["user"], "start": r["start"], "end": r["end"], "cpus": r["cpus"],
             "mem": r["mem"], "reason": reason_of(r["reason"]), "status": SUCCESS if r["success"] else FAILED}
            for h in histories for r in h.rows]


def get_stats(instances, status, start_ms, end_ms, lo, hi):
    """task-stats/get-stats for success or failed: get-tasks on the true start, then generate-all-stats with
    task-run-time over the instance's end (instance_stats_ref's with the start moved and now = 0)."""
    tasks = I.get_tasks(instances, status, start_ms, end_ms, lo, hi)
    return I.generate_all_stats([dict(t, start=-(t["end"] - t["start"])) for t in tasks], 0)


def d2h_bytes(n_handles_with_rows, segs, leaders, any_selected):
    """The call's downloads: 4 per handle holding a row, then instance_stats_ref's formula without its first 8."""
    if not n_handles_with_rows:
        return 0
    return 4 * n_handles_with_rows + I.d2h_bytes(segs, leaders, any_selected) - 8
