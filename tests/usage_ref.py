"""Plain restatement of cook_state_usage over host tables.  Test infrastructure only: every sum is a Python
loop of float additions in the order DESIGN.md §2 fixes for running usage, ascending task id.

  running_usage(rows, n_users, hostname_id)
    rows         running tasks as dicts with user, task_id, cpus, mem, gpus (absent: 0.0) and host (a hostname
                 code, -1: unknown)
    returns      {"user": {count, cpus, mem, gpus: [n_users]}, "pool": [count, cpus, mem, gpus],
                  "run_cpus", "run_mem": [H] float64, "run_count": [H] int32} for the H codes of hostname_id

generate-user-usage-map (scheduler.clj:711-727) per user, task-ents->usage (:2118-2123) over the pool, and
Fenzo's tracker state (:877-881) per host of the list.  A row whose host is -1 or not listed counts for its
user and the pool only.
"""
import numpy as np

KEYS = ("count", "cpus", "mem", "gpus")


def running_usage(rows, n_users, hostname_id=()):
    idx = {int(c): h for h, c in enumerate(hostname_id)}
    H = len(idx)
    user = {k: [0.0] * n_users for k in KEYS}
    pool = [0.0] * 4
    hc, hm, hn = [0.0] * H, [0.0] * H, [0] * H
    for r in sorted(rows, key=lambda r: int(r["task_id"])):
        u = int(r["user"])
        x = (1.0, float(r["cpus"]), float(r["mem"]), float(r.get("gpus", 0.0)))
        for k, v in zip(KEYS, x):
            user[k][u] = user[k][u] + v
        for k in range(4):
            pool[k] = pool[k] + x[k]
        h = idx.get(int(r.get("host", -1)))
        if h is not None:
            hc[h] = hc[h] + x[1]
            hm[h] = hm[h] + x[2]
            hn[h] += 1
    return {"user": {k: np.array(v, np.float64) for k, v in user.items()}, "pool": np.array(pool, np.float64),
            "run_cpus": np.array(hc, np.float64), "run_mem": np.array(hm, np.float64),
            "run_count": np.array(hn, np.int32)}


def aggregate_quota_groups(quota_groups, pool_usage):
    """aggregate-quota-groups (scheduler.clj:2125-2132): the pools' usage summed per quota group, pools in the
    given order (merge-with + over group-by), pools without a group left out."""
    out = {}
    for pool, usage in pool_usage.items():
        g = quota_groups.get(pool)
        if g is None:
            continue
        acc = out.setdefault(g, [0.0] * 4)
        for k in range(4):
            acc[k] = acc[k] + float(usage[k])
    return {g: np.array(v, np.float64) for g, v in out.items()}
