"""Writes list_jobs_golden.json: the reference's answers for listing waiting and running jobs, transcribed, and
hand-computed edges.

Each scenario holds handles (one per pool: its pool code, pending rows [user, job id, facts] and running rows
[user, job id, task id, facts], facts null or [submit ms, submit pool code, custom executor -1 / 0 / 1]; a running
row may say "unknown" (status unknown) or "parked" (its job launched with retry facts, so its pending slot is
parked)) and queries.  A query gives user, states (names, the caller's order), the window, the id window, the pool
code, include_custom_executor, limit and the host's completed / uncommitted parts, and what the reference answers:
  response   the job ids list-job-ents returns, newest first
  get_jobs   the job ids get-jobs-by-user-and-states returns (ascending submit time); `count` when only the count
             was asserted, `first` / `second` for the asserted positions of the response
  missing    the rows of the user in the id window without facts
Entity ids grow with submit time, as Datomic's do.
"""
import json
import os

T0 = 1_700_000_000_000
U1, U2, U3 = 0, 1, 2
FULL = dict(lo=-(1 << 63), hi=(1 << 63) - 1)
MAXI = (1 << 31) - 1


def q(user, states, start, end, include_custom_executor, limit=MAXI, pool=-1, **kw):
    d = dict(user=user, states=states, start=start, end=end, pool=pool, include_custom_executor=include_custom_executor,
             limit=limit, **FULL)
    d.update(kw)
    return d


def get_jobs_by_user_and_states(state):
    """test-get-jobs-by-user-and-states (test/cook/test/tools.clj:419), one state: job1 and job1.5 (custom executor,
    never returned) at start, job2 5 ms later, half-way, job3 of u2, job4, end; limit 10, 2 or 1; name filter any."""
    start, half, end = T0, T0 + 10, T0 + 20
    jobs = [(U1, 101, T0), (U1, 102, T0), (U1, 103, T0 + 5), (U2, 104, T0 + 10), (U1, 105, T0 + 15)]
    cex = {102: 1}
    rows = [[u, j, [t, -1, cex.get(j, 0)]] for u, j, t in jobs]
    h = {"pool": 0, "pending": rows, "running": []} if state == "waiting" else \
        {"pool": 0, "pending": [], "running": [[u, j, 1000 + j, f] for u, j, f in rows]}
    qs = [dict(q(U1, [state], start, half, False, 10), get_jobs=[101, 103]),
          dict(q(U1, [state], start, half, False, 1), get_jobs=[101]),
          dict(q(U1, [state], start, end, False, 10), count=3),
          dict(q(U1, [state], start, end, False, 2), get_jobs=[101, 103]),
          dict(q(U2, [state], start, end, False, 10), count=1),
          dict(q(U3, [state], start, end, False, 10), count=0),
          dict(q(U1, [state], 1_496_275_200_000, 1_496_361_600_000, False, 10, lo=0, hi=0), count=0)]
    return {"name": f"test-get-jobs-by-user-and-states {state}", "handles": [h], "queries": qs}


def list_jobs_by_time():
    """test-list-jobs-by-time (test/cook/test/rest/api.clj:2168): two submitted (waiting) jobs 10 ms apart, /list
    running+waiting+completed: start inclusive, end exclusive, newest first."""
    t1, t2 = T0 + 1000, T0 + 1010
    h = {"pool": 0, "pending": [[U1, 201, [t1, -1, 0]], [U1, 202, [t2, -1, 0]]], "running": []}
    st = ["running", "waiting", "completed"]
    return {"name": "test-list-jobs-by-time", "handles": [h], "queries": [
        dict(q(U1, st, t1 + 1, t2, False), response=[]),
        dict(q(U1, st, t1, t2, False), first=201, response=[201]),
        dict(q(U1, st, t1 + 1, t2 + 1, False), first=202, response=[202]),
        dict(q(U1, st, t1, t2 + 1, False), first=202, second=201, response=[202, 201])]}


def list_jobs_include_custom_executor():
    """test-list-jobs-include-custom-executor (:2192): /jobs running waiting completed; job 1 set to a custom executor
    after submission, both listed, job 2 first (submitted in the same ms: the reverse puts it first)."""
    t = T0 + 2000
    h = {"pool": 0, "pending": [[U1, 301, [t, -1, 1]], [U1, 302, [t, -1, 0]]], "running": []}
    return {"name": "test-list-jobs-include-custom-executor", "handles": [h], "queries": [
        dict(q(U1, ["running", "waiting", "completed"], T0, t + 1, True), count=2, first=302, second=301,
             response=[302, 301])]}


def list_jobs_with_pool():
    """test-list-jobs-with-pool (:2216): alice's running jobs in pools foo (0) and bar (1), then jobs in foo-1 (2) and
    foo-2 (3) submitted to foo; /jobs ["running"] per pool."""
    def h(pool, j, spool):
        return {"pool": pool, "pending": [], "running": [[U1, j, 10 * j, [T0 + j, spool, 0]]]}
    st = ["running"]
    return {"name": "test-list-jobs-with-pool", "handles": [h(0, 401, -1), h(1, 402, -1), h(2, 403, 0), h(3, 404, 0)],
            "queries": [dict(q(U1, st, T0, T0 + 1000, True, pool=2), count=1, response=[403]),
                        dict(q(U1, st, T0, T0 + 1000, True, pool=3), count=1, response=[404]),
                        dict(q(U1, st, T0, T0 + 1000, True, pool=1), count=1, response=[402]),
                        dict(q(U1, st, T0, T0 + 1000, True, pool=0), count=3, response=[404, 403, 401])]}


def edges():
    """Hand-computed: a nil custom executor (dropped by /list, kept by /jobs); a job whose smaller id has the later
    submit time (the per-state cut is by id, not by submit time); equal submit times across states (the reverse of the
    concatenation order); a job in the time window but outside the id window; two live instances of one job, one of
    them unknown, listed once; a parked copy that is not waiting; rows without facts counted as missing; an
    uncommitted waiting job /list merges in and a completed job from the Datomic path, where the cut after the
    ascending sort keeps the oldest entries."""
    S = T0 + 5000
    pend = [[U1, 501, [S + 100, -1, 0]], [U1, 502, [S + 50, -1, 0]], [U1, 503, [S + 200, -1, 0]],
            [U1, 506, [S + 300, -1, -1]], [U1, 507, None], [U1, 600, [S + 10, -1, 0]], [U2, 508, [S, -1, 0]]]
    run = [[U1, 504, 9001, [S + 200, -1, 0]], [U1, 505, 9002, [S + 150, -1, 0]],
           {"row": [U1, 505, 9003, [S + 150, -1, 0]], "unknown": True}, {"row": [U1, 509, 9004, [S + 20, -1, 0]],
                                                                        "parked": True},
           [U1, 510, 9005, None]]
    h = {"pool": 0, "pending": pend, "running": run}
    W, R = ["waiting"], ["running"]
    win = dict(lo=0, hi=600)
    return {"name": "edges", "handles": [h], "queries": [
        dict(q(U1, W, S, S + 1000, False, **win), response=[503, 501, 502], missing=1),
        dict(q(U1, W, S, S + 1000, True, **win), response=[506, 503, 501, 502], missing=1),
        dict(q(U1, W, S, S + 1000, True), response=[506, 503, 501, 502, 600], missing=1),
        dict(q(U1, W, S, S + 1000, False, limit=1, **win), response=[501]),
        dict(q(U1, ["waiting", "running"], S + 200, S + 201, True, **win), response=[504, 503]),
        dict(q(U1, ["running", "waiting"], S + 200, S + 201, True, **win), response=[503, 504]),
        dict(q(U1, R, S, S + 1000, True, **win), response=[504, 505, 509], missing=1),
        dict(q(U1, ["running", "waiting", "completed"], S, S + 1000, False, limit=3, **win,
               uncommitted=[[500, S + 10]], completed={"completed": [[498, S + 5]]}), response=[509, 500, 498]),
        dict(q(U2, W + R, S, S + 1000, False, **win), response=[508], missing=0)]}


def main():
    out = {"scenarios": [get_jobs_by_user_and_states("waiting"), get_jobs_by_user_and_states("running"),
                         list_jobs_by_time(), list_jobs_include_custom_executor(), list_jobs_with_pool(), edges()]}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "list_jobs_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
