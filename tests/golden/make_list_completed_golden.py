"""Writes list_completed_golden.json: the reference's answers for listing completed, success and failed jobs,
transcribed, and hand-computed edges.

Each scenario holds handles (one per pool: its pool code, its log's horizon `since`, its pending rows [user, job id,
facts] as in list_jobs_golden.json, the records it is seeded with and the record batches sent after, in order; a
record is [job id, stamp, user, submit ms, submit pool code, custom executor -1 / 0 / 1, kind 1 success / 2 failed /
3 reopened]) and queries.  A query gives user, states (names, the caller's order), the window, the id window, the pool
code, include_custom_executor and limit, and what the reference answers:
  response   the job ids list-job-ents returns, newest first
  get_jobs   the job ids get-jobs-by-user-and-states returns (ascending submit time); `count` when only the count
             was asserted, `first` / `second` for the asserted positions of the response
  refused    true when the window starts before a handle's horizon, so the completed states keep the Datomic path
Entity ids grow with submit time, as Datomic's do.
"""
import json
import os

T0 = 1_700_000_000_000
U1, U2, U3 = 0, 1, 2
FULL = dict(lo=-(1 << 63), hi=(1 << 63) - 1)
MAXI = (1 << 31) - 1
S, F, R = 1, 2, 3


def q(user, states, start, end, include_custom_executor, limit=MAXI, pool=-1, **kw):
    d = dict(user=user, states=states, start=start, end=end, pool=pool, include_custom_executor=include_custom_executor,
             limit=limit, **FULL)
    d.update(kw)
    return d


def handle(pool, since, seed=(), record=(), pending=()):
    return {"pool": pool, "since": since, "pending": [list(p) for p in pending], "seed": [list(r) for r in seed],
            "record": [[list(r) for r in b] for b in record]}


def get_jobs_by_user_and_states():
    """test-get-jobs-by-user-and-states (test/cook/test/tools.clj:419), the :job.state/completed pass: job1 and job1.5
    (custom executor, never returned) at start, job2 5 ms later, half-way, job3 of u2, job4, end; limit 10, 2 or 1.  The
    jobs have no instance, so each is failed (job-ent->state)."""
    start, half, end = T0, T0 + 10, T0 + 20
    jobs = [(U1, 101, T0, 0), (U1, 102, T0, 1), (U1, 103, T0 + 5, 0), (U2, 104, T0 + 10, 0), (U1, 105, T0 + 15, 0)]
    recs = [[j, 7, u, t, -1, cex, F] for u, j, t, cex in jobs]
    st = ["completed"]
    qs = [dict(q(U1, st, start, half, False, 10), count=2),
          dict(q(U1, st, start, half, False, 1), get_jobs=[101]),
          dict(q(U1, st, start, end, False, 10), count=3),
          dict(q(U1, st, start, end, False, 2), get_jobs=[101, 103]),
          dict(q(U2, st, start, end, False, 10), count=1),
          dict(q(U3, st, start, end, False, 10), count=0),
          dict(q(U1, st, 1_496_275_200_000, 1_496_361_600_000, False, 10, lo=0, hi=0), count=0),
          # the same jobs by instance state: failed, never success
          dict(q(U1, ["failed"], start, end, False, 10), get_jobs=[101, 103, 105]),
          dict(q(U1, ["success"], start, end, False, 10), count=0)]
    return {"name": "test-get-jobs-by-user-and-states completed", "handles": [handle(0, 1_400_000_000_000, recs)],
            "queries": qs}


def descriptive_state():
    """descriptive-state (test/cook/test/rest/api.clj:212-249): a waiting, a running, a completed job with successful
    instances (success) and a completed job without one (failed: the second instance is the success job's)."""
    t = T0 + 100
    pend = [[U1, 601, [t, -1, 0]]]
    recs = [[603, 11, U1, t + 2, -1, 0, S], [604, 12, U1, t + 3, -1, 0, F]]
    w = (T0, T0 + 1000)
    return {"name": "descriptive-state", "handles": [handle(0, T0, recs, pending=pend)], "queries": [
        dict(q(U1, ["success"], *w, True), response=[603]),
        dict(q(U1, ["failed"], *w, True), response=[604]),
        dict(q(U1, ["completed"], *w, True), response=[604, 603]),
        dict(q(U1, ["waiting", "completed"], *w, True), response=[604, 603, 601])]}


def edges():
    """Hand-computed, over two handles (pools 0 and 1) with horizon H:
      701 failed, reopened, completed again with a success: success
      702 a success, then reopened and waiting again: in no completed state, listed as waiting
      703 failed, then a late successful instance: success, not failed
      704 the same record sent twice: listed once
      705 failed and reopened in pool 0, then a success in pool 1: once, from pool 1
      706 a nil custom executor: dropped by /list (0), kept by /jobs (1)
      707 / 708 the smaller id submitted later: the cut is by id
      709 in the time window but outside the id window
      710 submitted at the horizon: kept; 711 submitted before it: not kept
      712 waiting and 713 completed, submitted in the same ms: the response reverses the order of `states`"""
    H = T0 + 10_000
    s = H + 100
    h0 = handle(0, H, seed=[[701, 10, U1, s + 1, -1, 0, F], [702, 10, U1, s + 2, -1, 0, S],
                            [703, 10, U1, s + 3, -1, 0, F], [705, 10, U1, s + 5, -1, 0, F]],
                record=[[[701, 20, U1, s + 1, -1, 0, R], [702, 20, U1, s + 2, -1, 0, R], [705, 20, U1, s + 5, -1, 0, R],
                         [704, 21, U1, s + 4, -1, 0, S]],
                        [[701, 30, U1, s + 1, -1, 0, S], [703, 40, U1, s + 3, -1, 0, S], [704, 21, U1, s + 4, -1, 0, S],
                         [706, 41, U1, s + 6, -1, -1, F], [707, 42, U1, s + 90, -1, 0, S], [708, 43, U1, s + 10, -1, 0, S],
                         [709, 44, U1, s + 9, -1, 0, S], [710, 45, U1, H, -1, 0, S], [711, 45, U1, H - 1, -1, 0, S],
                         [713, 46, U1, s + 500, -1, 0, F], [714, 47, U2, s + 7, -1, 0, S]]],
                pending=[[U1, 702, [s + 2, -1, 0]], [U1, 712, [s + 500, -1, 0]]])
    h1 = handle(1, H, record=[[[705, 30, U1, s + 5, -1, 0, S]]])
    end = s + 1000
    C, SU, FA = ["completed"], ["success"], ["failed"]
    return {"name": "edges", "handles": [h0, h1], "queries": [
        dict(q(U1, SU, s, s + 9, True), response=[705, 704, 703, 701]),
        dict(q(U1, FA, s, s + 9, True), response=[706]),
        dict(q(U1, FA, s, s + 9, False), response=[]),
        dict(q(U1, C, s, s + 9, False), response=[705, 704, 703, 701]),
        dict(q(U1, C, s, end, True, limit=8, lo=0, hi=709), response=[707, 708, 706, 705, 704, 703, 701]),
        dict(q(U1, C, s, end, True, limit=6, lo=0, hi=709), response=[707, 706, 705, 704, 703, 701]),
        dict(q(U1, C, s, end, True, limit=5, lo=0, hi=709), response=[706, 705, 704, 703, 701]),
        dict(q(U1, C, s + 9, s + 91, True, lo=0, hi=709), response=[707, 708]),
        dict(q(U1, C, s + 9, s + 91, True, limit=1, lo=0, hi=709), response=[707]),
        dict(q(U1, C, s + 9, s + 91, True), response=[707, 708, 709]),
        dict(q(U1, SU, s, end, True, pool=0), response=[707, 708, 709, 704, 703, 701]),
        dict(q(U1, SU, s, end, True, pool=1), response=[705]),
        dict(q(U1, ["waiting"] + C, H, s + 3, True), response=[702, 701, 710]),
        dict(q(U1, C, H, H + 1, True), response=[710]),
        dict(q(U1, C, H - 1, H + 1, True), refused=True),
        dict(q(U1, ["waiting", "completed"], s + 500, s + 501, True), response=[713, 712]),
        dict(q(U1, ["completed", "waiting"], s + 500, s + 501, True), response=[712, 713]),
        dict(q(U2, SU, s, end, True), response=[714])]}


def main():
    out = {"scenarios": [get_jobs_by_user_and_states(), descriptive_state(), edges()]}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "list_completed_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
