"""Plain restatement of the monitor's user stats (cook/monitor.clj) and the queue lengths (cook/queue_limit.clj) over
row lists.  Test infrastructure only: each function follows its Clojure counterpart map operation by map operation,
every sum a Python float addition in the order DESIGN.md §2 fixes.

  rows            pending jobs or running jobs as dicts with id (job id / task id), user, pool, cpus and mem
  job_stats       get-job-stats (:40-57): {user: {"cpus", "mem", "jobs"}}, rows folded in ascending id
  starved_stats   get-starved-job-stats (:69-90) over shares(user) -> {"cpus", "mem"}
  wuq_stats       get-waiting-under-quota-job-stats (:92-116) over quota(user) -> the user's quota map ("count", "cpus",
                  "mem" and any other keys)
  add_aggregated  add-aggregated-stats (:59-67), users folded in the given order
  set_stats_counters  set-stats-counters! (:177-207): the counter values it sets, per state and user, and the user
                  counts; a user absent from a state reads 0, as after clear-old-counters!
  queue_lengths   jobs->queue-lengths (queue_limit.clj:64-90)
  user_stats      the same stats in cook_state_user_stats' layout over user codes: the CPU stand-in of
                  engine.state_user_stats
"""
import numpy as np

STATES = ("running", "waiting", "starved", "waiting-under-quota")
COUNTS = ("total", "starved", "waiting-under-quota", "hungry", "satisfied")
LONG_MAX = 2 ** 63 - 1


def merge_with(f, a, b):
    """(merge-with f a b) for two maps, b possibly nil."""
    out = dict(a)
    for k, v in (b or {}).items():
        out[k] = f(out[k], v) if k in out else v
    return out


def in_pool(pool_name, job_pool, grouping):
    """job-ent-in-pool (:35-38)."""
    return pool_name == job_pool or pool_name == grouping.get(job_pool)


def job_stats(rows, pool_name, grouping=None):
    out = {}
    for r in sorted(rows, key=lambda r: r["id"]):
        if in_pool(pool_name, r["pool"], grouping or {}):
            s = {"cpus": r["cpus"], "mem": r["mem"], "jobs": 1}
            out[r["user"]] = merge_with(lambda x, y: x + y, out[r["user"]], s) if r["user"] in out else s
    return out


def _under(used, promised):
    return all((used or {}).get(k, 0.0) < v for k, v in promised.items())


def starved_stats(running, waiting, shares):
    out = {}
    for user in waiting:
        share, used = shares(user), running.get(user)
        if _under(used, share):
            out[user] = merge_with(min, waiting[user], merge_with(lambda s, r: s - r, share, used))
    return out


def wuq_stats(running, waiting, quota):
    out = {}
    for user in waiting:
        promised = {("jobs" if k == "count" else k): v for k, v in quota(user).items()}
        used = running.get(user)
        if _under(used, promised):
            out[user] = merge_with(min, waiting[user], merge_with(lambda q, r: max(q - r, 0), promised, used))
    return out


def add_aggregated(stats, order):
    if not stats:
        return {"all": {"cpus": 0, "mem": 0, "jobs": 0}}
    total = None
    for u in order:
        if u in stats:
            total = dict(stats[u]) if total is None else merge_with(lambda x, y: x + y, total, stats[u])
    return dict(stats, all=total)


def counter(x):
    """set-counter!'s (long (min value Long/MAX_VALUE))."""
    if isinstance(x, (int, np.integer)):
        return min(int(x), LONG_MAX)
    return LONG_MAX if float(x) >= 2.0 ** 63 else int(float(x))


def set_stats_counters(pending, running, pool_name, shares, quota, order, grouping=None):
    """{state: {user: {key: counter value}}} including "all", and "users": {count name: n}.  order: every user in
    ascending user code."""
    run = job_stats(running, pool_name, grouping)
    wait = job_stats(pending, pool_name, grouping)
    st = {"running": run, "waiting": wait, "starved": starved_stats(run, wait, shares),
          "waiting-under-quota": wuq_stats(run, wait, quota)}
    out = {s: {u: {k: counter(v) for k, v in m.items()} for u, m in add_aggregated(st[s], order).items()}
           for s in STATES}
    ru, wu = set(run), set(wait)
    starved, wuq = set(st["starved"]), set(st["waiting-under-quota"])
    out["users"] = {"total": len(ru | wu), "starved": len(starved), "waiting-under-quota": len(wuq),
                    "hungry": len(wu - starved), "satisfied": len(ru - wu)}
    return out


def queue_lengths(pending):
    """{"pool->queue-length": {pool: n}, "pool->user->queue-length": {pool: {user: n}}}."""
    per = {}
    for r in pending:
        u = per.setdefault(r["pool"], {})
        u[r["user"]] = u.get(r["user"], 0) + 1
    return {"pool->queue-length": {p: sum(m.values()) for p, m in per.items()}, "pool->user->queue-length": per}


def user_stats(pending, running, n_users, div_cpus, div_mem, quota_count, quota_cpus, quota_mem, rest_ok=None):
    """engine.state_user_stats' result over rows whose user is a code and pool is ignored (every row counts).  The
    quota map of user u is count, cpus and mem plus one more key, > 0 exactly when rest_ok[u]."""
    pend = [dict(r, pool=0) for r in pending]
    run = [dict(r, pool=0) for r in running]
    shares = lambda u: {"cpus": float(div_cpus[u]), "mem": float(div_mem[u])}
    quota = lambda u: {"count": float(quota_count[u]), "cpus": float(quota_cpus[u]), "mem": float(quota_mem[u]),
                       "rest": 1.0 if rest_ok is None or rest_ok[u] else 0.0}
    r, w = job_stats(run, 0), job_stats(pend, 0)
    st = [r, w, starved_stats(r, w, shares), wuq_stats(r, w, quota)]
    U = n_users
    jobs, cpus, mem = np.zeros((4, U), np.int64), np.zeros((4, U)), np.zeros((4, U))
    member = np.zeros(U, np.uint8)
    tot = {}
    for s, m in enumerate(st):
        for u, v in m.items():
            jobs[s, u], cpus[s, u], mem[s, u] = int(v["jobs"]), v["cpus"], v["mem"]
            member[u] |= 1 << s
        a = add_aggregated({u: {k: v[k] for k in ("jobs", "cpus", "mem")} for u, v in m.items()}, range(U))["all"]
        tot[STATES[s]] = (int(a["jobs"]), float(a["cpus"]), float(a["mem"]))
    ru, wu, sv, wq = (set(m) for m in st)
    return {"jobs": jobs, "cpus": cpus, "mem": mem, "member": member, "all": tot,
            "users": {"total": len(ru | wu), "starved": len(sv), "waiting-under-quota": len(wq),
                      "hungry": len(wu - sv), "satisfied": len(ru - wu)}}
