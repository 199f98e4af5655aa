"""The job listing's device half restated over row lists in plain Python: get-active-jobs-by-user-and-state
(tools.clj:445-466) for the waiting and running states as cook_state_list_jobs answers it.

A handle is {"pending": [(user, job id, facts)], "running": [(user, job id, task id, facts)]}, facts None (not
written) or (submit ms, submit pool code, custom executor -1 / 0 / 1).  Waiting entries are the pending rows; running
entries are the distinct (handle, job id) of the running rows, each represented by its row with the greatest task id.
"""
WAITING, RUNNING = 1, 2
INT32_MAX = (1 << 31) - 1


def selected(facts, job_id, k, q):
    """job-submitted-in-range?, the id window, check-pool-for-listing (pool.clj:22-42) and the executor filter."""
    if facts is None:
        return False
    submit, spool, cex = facts
    return (q["start"] <= submit < q["end"] and q["lo"] <= job_id < q["hi"] and
            (q["pool"] == -1 or q["handle_pool"][k] == q["pool"] or spool == q["pool"]) and
            (q["include_custom_executor"] or cex == 0))


def query(user, states, start, end, lo=-(1 << 63), hi=(1 << 63) - 1, pool=-1, handle_pool=None,
          include_custom_executor=True, limit=INT32_MAX):
    return dict(user=user, states=states, start=start, end=end, lo=lo, hi=hi, pool=pool, handle_pool=handle_pool,
                include_custom_executor=include_custom_executor, limit=limit)


def list_jobs(handles, q):
    """cook_state_list_jobs: ([(state, job id, submit ms, handle index)], rows without facts).  Each state in ascending
    (job id, handle index), cut to q["limit"]; waiting first."""
    out, missing = [], 0
    for state in (WAITING, RUNNING):
        if not q["states"] & state:
            continue
        cand = []
        for k, h in enumerate(handles):
            if state == WAITING:
                rows = [(j, -1, f) for u, j, f in h["pending"] if u == q["user"]]
            else:
                rows = [(j, t, f) for u, j, t, f in h["running"] if u == q["user"]]
            missing += sum(1 for j, _, f in rows if f is None and q["lo"] <= j < q["hi"])
            rep = {}
            for j, t, f in rows:
                if j not in rep or t > rep[j][0]:
                    rep[j] = (t, f)
            cand += [(j, k, f) for j, (_, f) in rep.items()]
        picked = sorted((j, k, f[0]) for j, k, f in cand if selected(f, j, k, q))[:q["limit"]]
        out += [(state, j, s, k) for j, k, s in picked]
    return out, missing
