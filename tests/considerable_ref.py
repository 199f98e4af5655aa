"""A plain-Python restatement of Cook's considerable-job selection over a ranked queue.

filter-pending-jobs-for-quota (tools.clj:961-973): per user, the running usage plus the user's queued jobs in queue
order, left folded; a job stays while the fold up to and including it is within the user's quota
(filter-based-on-user-quota :903-915); with the launch-rate limit enforced, only the first `tokens` survivors of each
user stay (:940-959); then the pool quota over the survivors in queue order, starting from the sum of every user's
usage (users 0 .. U-1, a left fold; :917-933, :969).  pending-jobs->considerable-jobs (scheduler.clj:729-762) adds
job-allowed-to-start? and the launch plugin, then takes num_considerable.

Every sum is an IEEE f64 left fold, so the result is bit for bit what the reference computes.
"""
KEYS = ("count", "cpus", "mem", "gpus")


def considerable(queue, user, cpus, mem, gpus, quota, usage, num_considerable, tokens=None, enforce_rate_limit=False,
                 pool_quota=None, allowed=None, plugin_accept=None):
    """queue: job indices in rank order; user / cpus / mem / gpus: per-job columns; quota / usage: {key: per-user
    sequence}; tokens: per-user launch-rate tokens (None: unlimited); pool_quota: {key: value} or None; allowed /
    plugin_accept: per-job flags or None (all allowed).  Returns the considerable job indices in take order."""
    n_users = len(quota["count"])
    acc = {u: [float(usage[k][u]) for k in KEYS] for u in range(n_users)}
    kept_of = [0] * n_users
    survivors = []
    for j in queue:
        u = int(user[j])
        a = acc[u]
        x = (1.0, float(cpus[j]), float(mem[j]), float(gpus[j]))
        for i in range(4):
            a[i] = a[i] + x[i]
        if not all(a[i] <= float(quota[k][u]) for i, k in enumerate(KEYS)):
            continue
        kept_of[u] += 1
        if enforce_rate_limit and tokens is not None and kept_of[u] > int(tokens[u]):
            continue
        survivors.append(j)
    if pool_quota is not None:
        pool = [0.0, 0.0, 0.0, 0.0]
        for u in range(n_users):
            for i, k in enumerate(KEYS):
                pool[i] = pool[i] + float(usage[k][u])
        kept = []
        for j in survivors:
            x = (1.0, float(cpus[j]), float(mem[j]), float(gpus[j]))
            for i in range(4):
                pool[i] = pool[i] + x[i]
            if all(pool[i] <= float(pool_quota[k]) for i, k in enumerate(KEYS)):
                kept.append(j)
        survivors = kept
    out = []
    for j in survivors:
        if len(out) >= num_considerable:
            break
        if allowed is not None and not allowed[j]:
            continue
        if plugin_accept is not None and not plugin_accept[j]:
            continue
        out.append(j)
    return out


def offensive(order, cpus, mem, max_mem_mb, max_cpus):
    """filter-offensive-jobs (scheduler.clj:2198-2229) over a ranked queue: the jobs whose mem or cpus exceed the
    caps, in queue order."""
    return [j for j in order if float(mem[j]) > max_mem_mb or float(cpus[j]) > max_cpus]
