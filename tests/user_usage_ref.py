"""Plain-Python restatement of GET /usage (get-user-usage, api.clj:2946-2969) and of cook_state_user_usage.

The reference's functions over plain job values {job_id, user, pool (None: no pool), cpus, mem[, gpus], group (None:
ungrouped)}: total-resources-of-jobs (tools.clj:294-306, a left fold of merge-with + from {cpus 0.0 mem 0.0 gpus 0.0
jobs (count jobs)}), user-usage, no-usage-map, usage and get-user-usage, in the JSON response's key names.  The jobs'
order is the fold order and the order of every job list; groups come in ascending code.

`answer` is what cook_state_user_usage returns over a host mirror of its handles' running rows, one {task id: row} per
handle: one representative per (handle, job id), the row with the greatest task id; its group the first entry of its
group list; segments (user, scope, group) in ascending order, each a left fold from +0.0 in ascending (task id,
handle) with its job ids in that order.
"""
TOTAL, UNGROUPED = -2, -1
SEG_BYTES = 44   # user, scope, group, jobs, cpus, mem, gpus; + 4 (list offset) with by_group


# ---- the reference ------------------------------------------------------------------------------------------------
def total_resources_of_jobs(jobs):
    acc = {"cpus": 0.0, "mem": 0.0, "gpus": 0.0, "jobs": len(jobs)}
    for j in jobs:
        for k in ("cpus", "mem", "gpus"):
            if j.get(k) is not None:
                acc[k] = acc[k] + j[k]
    return acc


def user_usage(with_group_breakdown, jobs, groups=None):
    """groups: {group code: (uuid, name)} (default: the code and None)."""
    out = {"total_usage": total_resources_of_jobs(jobs)}
    if with_group_breakdown:
        by = {}
        for j in jobs:
            by.setdefault(j.get("group"), []).append(j)
        info = lambda g: (groups or {}).get(g, (g, None))
        out["grouped"] = [{"group": {"uuid": info(g)[0], "name": info(g)[1], "running_jobs": [j["job_id"] for j in js]},
                           "usage": total_resources_of_jobs(js)}
                          for g, js in sorted((g, js) for g, js in by.items() if g is not None)]
        un = by.get(None, [])
        out["ungrouped"] = {"running_jobs": [j["job_id"] for j in un], "usage": total_resources_of_jobs(un)}
    return out


def no_usage_map(with_group_breakdown):
    out = {"total_usage": total_resources_of_jobs([])}
    if with_group_breakdown:
        out["grouped"] = []
        out["ungrouped"] = {"running_jobs": [], "usage": total_resources_of_jobs([])}
    return out


def pool_of(job, default_pool):
    return job["pool"] if job.get("pool") is not None else default_pool


def usage(pool, with_group_breakdown, jobs, pools=(), default_pool=None, groups=None):
    if pool is not None or not pools:
        return user_usage(with_group_breakdown, jobs, groups)
    by = {}
    for j in jobs:
        by.setdefault(pool_of(j, default_pool), []).append(j)
    out = user_usage(with_group_breakdown, jobs, groups)
    out["pools"] = {p: no_usage_map(with_group_breakdown) for p in pools}
    out["pools"].update({p: user_usage(with_group_breakdown, js, groups) for p, js in by.items()})
    return out


def get_user_usage(jobs, user=None, pool=None, group_breakdown=False, pools=(), default_pool=None, groups=None):
    """jobs: every running job in the fold order.  user None: {"users": {user: usage}} over the users that run a job."""
    sel = [j for j in jobs if pool is None or pool_of(j, default_pool) == pool]
    if user is not None:
        return usage(pool, group_breakdown, [j for j in sel if j["user"] == user], pools, default_pool, groups)
    by = {}
    for j in sel:
        by.setdefault(j["user"], []).append(j)
    return {"users": {u: usage(pool, group_breakdown, js, pools, default_pool, groups) for u, js in sorted(by.items())}}


# ---- cook_state_user_usage over a host mirror ---------------------------------------------------------------------
def representatives(handles):
    """[(task id, handle index, row)] of each (handle, job id)'s row with the greatest task id, in ascending (task id,
    handle)."""
    rep = {}
    for p, run in enumerate(handles):
        for t, r in run.items():
            k = (p, r["job_id"])
            if k not in rep or t > rep[k][0]:
                rep[k] = (t, p, r)
    return sorted(rep.values(), key=lambda x: (x[0], x[1]))


def first_group(r):
    g = r.get("groups") or []
    return g[0] if g else UNGROUPED


def answer(handles, users=None, per_pool=False, by_group=False):
    """[(user, scope, group, jobs, cpus, mem, gpus, job ids or None)] in the call's segment order."""
    segs = {}
    for t, p, r in representatives(handles):
        if users is not None and r["user"] not in users:
            continue
        scopes = [-1] + ([p] if per_pool else [])
        grps = [TOTAL] + ([first_group(r)] if by_group else [])
        for s in scopes:
            for g in grps:
                segs.setdefault((r["user"], s, g), []).append(r)
    out = []
    for (u, s, g), rs in sorted(segs.items()):
        c = m = x = 0.0
        for r in rs:   # the left fold, ascending (task id, handle)
            c, m, x = c + r["cpus"], m + r["mem"], x + r.get("gpus", 0.0)
        out.append((u, s, g, len(rs), c, m, x, [r["job_id"] for r in rs] if by_group and g != TOTAL else None))
    return out


def rows_queried(handles, users=None):
    """R_q: the live running rows of the queried users over the handles (the call's capacity bound)."""
    return sum(1 for run in handles for r in run.values() if users is None or r["user"] in users)


def d2h_bytes(segs, by_group):
    return 8 + (SEG_BYTES + 4 * bool(by_group)) * len(segs) + 8 * sum(len(s[7]) for s in segs if s[7] is not None)


def jobs_of(handles, names):
    """The running jobs the reference reads, as `get_user_usage` takes them, in the call's fold order: one per
    representative, its pool the handle's name, its group the first of its list (None: ungrouped)."""
    out = []
    for t, p, r in representatives(handles):
        g = first_group(r)
        j = {"job_id": r["job_id"], "user": r["user"], "pool": names[p], "cpus": r["cpus"], "mem": r["mem"],
             "group": None if g == UNGROUPED else g}
        if "gpus" in r:
            j["gpus"] = r["gpus"]
        out.append(j)
    return out


def engine_answer(handles, users=None, per_pool=False, by_group=False):
    """`answer` in engine.state_user_usage's shape (numpy columns), for cycle.usage_response on the CPU."""
    import numpy as np
    a = answer(handles, users, per_pool, by_group)
    col = lambda i, dt: np.array([s[i] for s in a], dt)
    out = {"user": col(0, np.int32), "scope": col(1, np.int32), "group": col(2, np.int32), "jobs": col(3, np.int64),
           "cpus": col(4, np.float64), "mem": col(5, np.float64), "gpus": col(6, np.float64),
           "lists": [s[7] for s in a]}
    if by_group:
        off, jid = [], []
        for s in a:
            off.append(-1 if s[7] is None else len(jid))
            jid += s[7] or []
        out["list_off"], out["job_id"] = np.array(off, np.int32), np.array(jid, np.int64)
    return out
