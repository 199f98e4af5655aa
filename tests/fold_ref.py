"""Plain references for the f64 running sums of cook_b200/csrc/fold.cuh, and the traces that reach
their path switches through the C ABI.  Test infrastructure only: no numpy reduction is trusted for a
sum here, every fold is a Python loop of float additions (IEEE f64, round to nearest) in a stated order.

The grid rule (common.cuh): every addend is a multiple of 2^-10 in [0, 2^40] and
(n + 1) * max(m, 1) + start < 2^43, with start itself on the grid.  Then every partial sum of every
subset is exact, so any association gives the left fold's bits and a parallel scan is legal.
"""
import math
import struct

import numpy as np

from cook_b200 import abi

GRID = 2.0 ** -10
VMAX = 2.0 ** 40
LIMIT = 2.0 ** 43

OS_TILE = 2048     # fold.cuh: order_scan tile
CP_BLOCK = 1024    # fold.cuh: compaction block
QF_CH = 1024       # rank.cu: quota filter chunk


# ---- folds ---------------------------------------------------------------------------------------
def left_fold(xs, start=0.0):
    """Inclusive running sums ((start + x0) + x1) + ..., one float addition per item."""
    out = []
    acc = float(start)
    for x in xs:
        acc = acc + float(x)
        out.append(acc)
    return out


def left_total(xs, start=0.0):
    acc = float(start)
    for x in xs:
        acc = acc + float(x)
    return acc


def exact_sum(xs, start=0.0):
    """The correctly rounded sum of start and xs."""
    return math.fsum([float(start)] + [float(x) for x in xs])


def pairwise_sum(xs):
    """Pairwise tree sum (the association of a parallel reduction)."""
    xs = [float(x) for x in xs]
    if not xs:
        return 0.0
    while len(xs) > 1:
        nxt = [xs[i] + xs[i + 1] for i in range(0, len(xs) - 1, 2)]
        if len(xs) % 2:
            nxt.append(xs[-1])
        xs = nxt
    return xs[0]


def reversed_sum(xs, start=0.0):
    return left_total(list(xs)[::-1], start)


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def same_bits(a, b):
    """Bit equality of two f64 arrays (NaN equals NaN of the same payload; -0.0 differs from 0.0)."""
    a = np.ascontiguousarray(a, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


# ---- the grid rule, restated -------------------------------------------------------------------
def grid_value_ok(x):
    x = float(x)
    if not (x >= 0.0 and x <= VMAX):      # NaN, inf and negatives fail here
        return False
    y = x * 1024.0
    return y == math.floor(y)


def grid_flag(*cols):
    """(bad, max_bits) as grid_check_kernel leaves them over the given columns (None = a zero column)."""
    cols = [np.asarray(c, np.float64) for c in cols if c is not None]
    n = max((len(c) for c in cols), default=0)
    bad, mb = 0, 0
    for i in range(n):
        vals = [float(c[i]) for c in cols]
        if not all(grid_value_ok(v) for v in vals):
            bad = 1
        m = 0.0
        for v in vals:
            m = max(m, v) if not math.isnan(v) else m   # fmax ignores NaN
        if m > 0.0:
            mb = max(mb, bits(m))
    return bad, mb


def grid_exact(flag, n, start=0.0):
    bad, mb = flag
    if bad:
        return False
    m = struct.unpack("<d", struct.pack("<Q", mb))[0]
    return grid_value_ok(start) and (float(n + 1) * max(m, 1.0) + float(start)) < LIMIT


# ---- association sensitivity -------------------------------------------------------------------
def association_sensitive(xs, start=0.0):
    """True when some prefix of the left fold differs from the reversed or the pairwise sum of the same
    prefix: a kernel that summed in another order would give other bits there."""
    xs = [float(x) for x in xs]
    fold = left_fold(xs, start)
    n = len(xs)
    ks = range(n) if n <= 256 else sorted(set(range(256)) | set(range(255, n, 61)) | {n - 1})
    for k in ks:
        pre = xs[:k + 1]
        if fold[k] != reversed_sum(pre, start) or fold[k] != float(start) + pairwise_sum(pre):
            return True
    return False


def segments_sensitive(amount, user, start=None):
    """association_sensitive over the per-user segments of an amount column (items in index order)."""
    for u in np.unique(user):
        xs = list(np.asarray(amount)[user == u])
        s = 0.0 if start is None else float(start[u])
        if association_sensitive(xs, s):
            return True
    return False


# ---- trace builders ----------------------------------------------------------------------------
# per-user task counts at the chunk edges of user_fold_kernel / cons_user_kernel (32 slots, 4 chunks
# prefetched), a user starting exactly at an order_scan tile edge, and one user longer than two tiles
EDGE_COUNTS = [1, 31, 32, 33, 127, 128, 129]
LONG_USER = 2 * OS_TILE + 405


def edge_counts():
    """Counts whose cumulative sums put a user's first task at position 0 and at OS_TILE exactly."""
    c = list(EDGE_COUNTS)
    c.append(OS_TILE - sum(c))          # pad: the next user starts at position OS_TILE
    c += [129, 1, LONG_USER, 33, 1, 128, 2, 31]
    return c


MIXED_BIG = 2.0 ** 32    # on the grid; (len + 1) * 2^32 < 2^43 holds for users below 2047 tasks only
REB_BIG = 2.0 ** 36      # the rebalancer traces: users of 127 tasks or more take the chain


def amounts(rng, regime, n, long_mask=None, big=None):
    """(cpus, mem) of n tasks.  grid: halves and 512 MiB steps.  off: sevenths and tenths, every partial
    sum rounds.  mixed: on the grid, but the tasks of long_mask carry mem near 2^32 with 2^-10 parts, so
    the order-wide total passes 2^43 (no order-wide scan) and a long user's running sum rounds."""
    if regime == "grid":
        cpus = rng.choice(np.array([0.5, 1.0, 2.0, 4.0]), n)
        mem = 512.0 * rng.integers(1, 65, n)
    elif regime == "off":
        cpus = rng.choice(np.array([0.1, 0.3, 0.7, 1.1, 2.9]), n)
        mem = rng.integers(1, 40000, n) / 7.0
    elif regime == "mixed":
        cpus = rng.choice(np.array([0.5, 1.0, 2.0, 4.0]), n)
        mem = 512.0 * rng.integers(1, 65, n)
        if long_mask is not None and long_mask.any():
            k = int(long_mask.sum())
            mem[long_mask] = (big or MIXED_BIG) - GRID * rng.integers(1, 2 ** 20, k)
    else:
        raise ValueError(regime)
    return cpus.astype(np.float64), mem.astype(np.float64)


def _task_cols(user, cpus, mem, running, id_base, rng):
    n = len(user)
    prio = rng.choice(np.array([10, 50, 90], np.int32), size=n, p=(0.1, 0.8, 0.1)).astype(np.int32)
    job_id = (id_base + np.arange(n)).astype(np.int64) * 2
    if running:
        start = (1_600_000_000_000 + rng.integers(0, 86_400_000, size=n)).astype(np.int64)
        task_id = job_id + 1
    else:
        start = np.full(n, abi.INT64_MAX, np.int64)
        task_id = np.full(n, -1, np.int64)
    return dict(user=np.asarray(user, np.int32), priority=prio, start_time=start, task_id=task_id, job_id=job_id,
                cpus=cpus, mem=mem, gpus=np.zeros(n))


def fold_pool(regime, seed, counts=None, run_frac=0.3, n_offers=160, mem_scale=1.0):
    """Rank + match inputs with EXACT per-user task counts (running + pending), users in name order so
    segment k starts at sum(counts[:k]).  Returns the plain columns too, so a caller can rebuild the
    structs with other amounts (build_pool: mem scaling, user quotas, usage)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    counts = edge_counts() if counts is None else list(counts)
    U = len(counts)
    owner = np.repeat(np.arange(U, dtype=np.int32), counts)
    N = len(owner)
    is_run = rng.random(N) < run_frac
    long_mask = np.repeat(np.asarray(counts) >= OS_TILE, counts)
    cpus, mem = amounts(rng, regime, N, long_mask)
    cols = dict(
        run=_task_cols(owner[is_run], cpus[is_run], mem[is_run], True, 1, rng),
        pend=_task_cols(owner[~is_run], cpus[~is_run], mem[~is_run], False, 1_000_000, rng),
        div_cpus=np.full(U, 100.0 if regime != "off" else 100.0 / 7.0),
        div_mem=np.full(U, 400000.0 if regime != "off" else 400000.0 / 3.0),
        offer_cpus=np.array([16.0, 32.0, 64.0])[rng.integers(0, 3, n_offers)],
        offer_mem=np.array([65536.0, 131072.0, 262144.0])[rng.integers(0, 3, n_offers)],
        run_frac=rng.integers(0, 4, n_offers) / 8.0,
        host_rank=rng.permutation(n_offers).astype(np.int32),
        n_users=U, counts=counts)
    if regime == "off":
        cols["offer_mem"] = cols["offer_mem"] / 3.0
    return build_pool(cols, mem_scale)


def build_pool(cols, mem_scale=1.0, user_quota=None, user_usage=None, tokens=None):
    """The ABI structs of fold_pool's columns, every mem quantity multiplied by mem_scale (a power of
    two, so every product is exact)."""
    s = float(mem_scale)
    run, pend, U = cols["run"], cols["pend"], cols["n_users"]
    rt = dict(run, mem=run["mem"] * s)
    pt = dict(pend, mem=pend["mem"] * s)
    running = abi.make_tasks(**rt)
    pending = abi.make_tasks(**pt)
    if user_usage is None:
        user_usage = {k: np.zeros(U) for k in ("count", "cpus", "mem", "gpus")}
        np.add.at(user_usage["count"], run["user"], 1.0)
        for i in range(len(run["user"])):      # left fold in task order
            u = run["user"][i]
            user_usage["cpus"][u] = user_usage["cpus"][u] + run["cpus"][i]
            user_usage["mem"][u] = user_usage["mem"][u] + run["mem"][i]
    usage = dict(user_usage, mem=np.asarray(user_usage["mem"]) * s)
    quota = None
    if user_quota is not None:
        quota = dict(user_quota, mem=np.asarray(user_quota["mem"]) * s)
    users = abi.make_users(U, name_rank=np.arange(U, dtype=np.int32), div_mem=cols["div_mem"] * s,
                           div_cpus=cols["div_cpus"], div_gpus=np.ones(U), quota=quota, usage=usage,
                           tokens=tokens)
    n_off = len(cols["offer_cpus"])
    run_cpus = np.floor(cols["offer_cpus"] * cols["run_frac"] * 2.0) / 2.0
    run_mem = np.floor(cols["offer_mem"] * cols["run_frac"])
    jobs = abi.JobsSoA(n=len(pend["user"]), user=pend["user"], cpus=pend["cpus"], mem=pt["mem"], gpus=pend["gpus"],
                       ports=np.zeros(len(pend["user"]), np.int32), allowed=np.ones(len(pend["user"]), np.uint8),
                       plugin_accept=np.ones(len(pend["user"]), np.uint8))
    offers = abi.OffersSoA(n=n_off, hostname_id=np.arange(n_off, dtype=np.int32), name_rank=cols["host_rank"],
                           cpus=cols["offer_cpus"] - run_cpus, mem=(cols["offer_mem"] - run_mem) * s,
                           run_cpus=run_cpus, run_mem=run_mem * s,
                           run_count=np.where(run_cpus > 0, 3, 0).astype(np.int32), n_attr_cols=0)
    return dict(cols=cols, running=running, pending=pending, users=users, jobs=jobs, offers=offers,
                n_users=U, mem_scale=s, usage=user_usage)


def fold_rebalance(regime, seed, counts=None, n_hosts=60, n_pending=24, mem_scale=1.0, lead_mem_offset=0.0):
    """Rebalancer inputs with exact per-user running-task counts; the pending jobs belong to the last
    users (under-served), one of them with no running task at all.  lead_mem_offset is added to the mem
    of the lead pending jobs (1/3: an off-grid request on top of on-grid running tasks)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    counts = [40, 1, 31, 32, 33, 127, 128, 129, 700, 126, 5, 0] if counts is None else list(counts)
    U = len(counts)
    owner = np.repeat(np.arange(U, dtype=np.int32), counts)
    R = len(owner)
    long_mask = np.repeat(np.asarray(counts) >= 500, counts)
    cpus, mem = amounts(rng, regime, R, long_mask, big=REB_BIG)
    run = _task_cols(owner, cpus, mem, True, 1, rng)
    s = float(mem_scale)
    host = rng.integers(0, n_hosts, R).astype(np.int32)
    running = abi.RunningSoA(t=abi.make_tasks(**dict(run, mem=run["mem"] * s)), host=host)
    # the lead pending jobs: a user without running tasks, users of 129 and 127 tasks, the long user,
    # the user of 126 tasks (whose segment leaves the grid rule when a task joins it, REB_BIG) and the
    # user of 128 tasks
    lead = [U - 1, 7, 5, 8, 9, 6]
    pu = np.concatenate([lead, rng.integers(U - 4, U, n_pending - len(lead))]).astype(np.int32)
    pc, pm = amounts(rng, "grid" if regime == "mixed" else regime, n_pending)
    pend = _task_cols(pu, pc * 2.0, pm * 2.0, False, 10_000_000, rng)
    pend["mem"][:len(lead)] += lead_mem_offset
    share_c = 8.0 if regime != "off" else 8.0 / 7.0
    share_m = 4096.0 if regime != "off" else 4096.0 / 3.0
    div_mem, div_cpus = np.full(U, share_m * s), np.full(U, share_c)
    users = abi.make_users(U, name_rank=np.arange(U, dtype=np.int32), div_mem=div_mem, div_cpus=div_cpus,
                           div_gpus=np.ones(U))
    has_spare = (rng.random(n_hosts) < 0.1).astype(np.uint8)
    hosts = abi.HostTable(n=n_hosts, hostname_id=np.arange(n_hosts, dtype=np.int32),
                          name_rank=rng.permutation(n_hosts).astype(np.int32), has_spare=has_spare,
                          spare_cpus=np.where(has_spare, rng.integers(0, 9, n_hosts), 0).astype(float),
                          spare_mem=np.where(has_spare, 1024.0 * rng.integers(0, 17, n_hosts), 0.0) * s,
                          spare_gpus=np.zeros(n_hosts), n_attr_cols=0)
    jobs = abi.JobsSoA(n=n_pending, user=pu, cpus=pend["cpus"], mem=pend["mem"] * s, gpus=np.zeros(n_pending))
    return dict(running=running, pending=jobs, pending_job_id=pend["job_id"], pending_priority=pend["priority"],
                hosts=hosts, users=users, run=run, host=host, counts=counts, mem_scale=s, pend=pend, lead=lead,
                div_mem=div_mem, div_cpus=div_cpus, params=abi.RebalanceParams(16, 0.5, 1.0, 0))


def user_task_order(r, u):
    """The running tasks of user u in the rebalancer's per-user order (priority desc, start, task, job)."""
    run = r["run"]
    mine = np.flatnonzero(run["user"] == u)
    return sorted(mine, key=lambda i: (-run["priority"][i], run["start_time"][i], run["task_id"][i],
                                       run["job_id"][i]))


def below_quota_mem(r, p):
    """The addends of job-below-quota's mem fold for pending job p: its own mem first, then the mem of
    its user's running tasks in order (all scaled as the ABI sees them)."""
    s = r["mem_scale"]
    u = int(r["pend"]["user"][p])
    return [r["pend"]["mem"][p] * s] + [r["run"]["mem"][i] * s for i in user_task_order(r, u)]


def quota_at_fold(r, below):
    """Users whose mem quota sits exactly on the left fold of job-below-quota for each lead pending job
    (below=True: the job is below quota) or one ulp under it (below=False: it is not).  Any other
    association that rounds the other way flips the answer.  Other quotas stay unlimited."""
    U = len(r["counts"])
    qm = np.full(U, np.finfo(np.float64).max)
    for p, u in enumerate(r["lead"]):
        f = left_total(below_quota_mem(r, p))
        qm[u] = f if below else np.nextafter(f, -np.inf)
    return abi.make_users(U, name_rank=np.arange(U, dtype=np.int32), div_mem=r["div_mem"], div_cpus=r["div_cpus"],
                          div_gpus=np.ones(U), quota={"mem": qm})
