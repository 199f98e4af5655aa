"""Cases that put the rank's pool quota on the last bit of its running fold (tests/test_state_rank_quota.py).

The pool quota filter (filter-based-on-quota, scheduler.clj:2134-2157) starts from the pool's running usage, a left
fold over the running tasks, and advances it over the queue in order.  Off the binary grid that fold's last bit
depends on the order of the running rows; the project fixes it as ascending task id (DESIGN §2).  A case here holds
running rows of several users and a queue of more than QF_CH + 1 jobs, and for each quota column and boundary k the
quota q* that lies exactly on the fold of the first k queued jobs continued from the task-id fold of the running
column.  At q* the queue keeps k jobs, at nextafter(q*, -inf) k - 1; a running total one ulp off moves the cut.

Two amount regimes:
  off    cpus in tenths, mem in sevenths, gpus in {0, 0.1, 1}: every partial sum rounds.
  mixed  on the 2^-10 grid, but user 0's running rows (256 or more) carry cpus and mem just under 2^35, so the
         running totals pass 2^43: the rank's call-wide grid flag fails and the folds take the serial chain with
         every value on the grid.  The gpus are small integers, so their fold is exact in every order.
Half the pending jobs ask for no gpus; a gpus boundary sits where two queued jobs in a row ask for some (`cut`).

Layouts: the order in which one delta on a fresh handle lists the running rows, as indices into the rows sorted by
task id.  asc is the control; desc the reversal; above / below a seeded permutation whose left fold lies above /
below the task-id fold in every column whose fold depends on the order (seeds found by `find_seed`).
"""
import numpy as np

import fold_ref as F
import resident_model as M
from cook_b200 import abi

REGIMES = ("off", "mixed")
LAYOUTS = ("asc", "desc", "above", "below")
COLS = ("cpus", "mem", "gpus")
KS = (1, 37, F.QF_CH, F.QF_CH + 1)
N_RUN, N_PEND, N_USERS = 1200, 1800, 8
# np.random.default_rng(seed).permutation(N_RUN) of each regime's case: the first seed from 0 whose fold lies
# above (below) the task-id fold in every order-sensitive column (find_seed)
SEEDS = {("off", "above"): 20, ("off", "below"): 71, ("mixed", "above"): 36, ("mixed", "below"): 2}
CASE_SEED = {"off": 101, "mixed": 202}


def build(regime):
    """The case of a regime: running rows sorted by task id, pending rows [(job id, row)] in job id order, the
    user table."""
    rng = np.random.default_rng(CASE_SEED[regime])
    ru = M.zipf_users(rng, N_RUN, N_USERS)
    big = ru == 0
    rc, rm, rg = M.amounts(rng, regime, N_RUN, big)
    if regime == "off":
        rg = rng.choice(np.array([0.0, 0.1, 1.0]), N_RUN)
    else:
        rc[big] = M.BIG - F.GRID * rng.integers(1, 2 ** 20, int(big.sum()))
    tid = np.sort(rng.choice(10 ** 8, N_RUN, replace=False)).astype(np.int64) * 2 + 1
    prio = rng.choice(np.array([10, 50, 90]), N_RUN, p=(0.1, 0.8, 0.1))
    start = M.START + rng.integers(0, 86_400_000, N_RUN)
    run = [dict(user=int(ru[i]), priority=int(prio[i]), start_time=int(start[i]), task_id=int(tid[i]),
                job_id=int(tid[i]) + 1, cpus=float(rc[i]), mem=float(rm[i]), gpus=float(rg[i])) for i in range(N_RUN)]
    pu = M.zipf_users(rng, N_PEND, N_USERS)
    pc, pm, pg = M.amounts(rng, regime, N_PEND)
    pp = rng.choice(np.array([10, 50, 90]), N_PEND, p=(0.1, 0.8, 0.1))
    pend = [(10 ** 9 + 2 * i, dict(user=int(pu[i]), priority=int(pp[i]), cpus=float(pc[i]), mem=float(pm[i]),
                                   gpus=float(pg[i]), novel=[], attr=[], groups=[])) for i in range(N_PEND)]
    s = 1.0 if regime == "mixed" else 1.0 / 7.0
    users = abi.make_users(N_USERS, name_rank=rng.permutation(N_USERS).astype(np.int32),
                           div_mem=np.full(N_USERS, 4.0e5 * s), div_cpus=np.full(N_USERS, 100.0 * s),
                           div_gpus=np.ones(N_USERS))
    return dict(regime=regime, run=run, pend=pend, users=users, big=int(big.sum()))


def running_table(c, order=None):
    """cook_rank's running table of the case's rows in `order` (indices into the task-id order; None: that order)."""
    rows = c["run"] if order is None else [c["run"][i] for i in order]
    return M.tasks_soa(rows)


def pending_table(c):
    jobs, prio, jid = M.jobs_soa(c["pend"])
    return abi.make_tasks(user=jobs.col("user"), priority=prio, start_time=np.full(jobs.n, abi.INT64_MAX),
                          task_id=np.full(jobs.n, -1, np.int64), job_id=jid, cpus=jobs.col("cpus"),
                          mem=jobs.col("mem"), gpus=jobs.col("gpus")), jid


def run_col(c, col, order=None):
    rows = c["run"] if order is None else [c["run"][i] for i in order]
    return [r[col] for r in rows]


def running_total(c, col, order=None):
    """The pool's running usage of one column: the left fold of the rows in `order` (None: ascending task id)."""
    return F.left_total(run_col(c, col, order))


def sensitive(c, col):
    """Whether some order of the running column folds to other bits than ascending task id (reversal or pairwise
    already does)."""
    xs = run_col(c, col)
    t = F.left_total(xs)
    return F.reversed_sum(xs) != t or F.pairwise_sum(xs) != t


def sensitive_cols(c):
    return [col for col in COLS if sensitive(c, col)]


def layout(c, name):
    """The layout's order of the running rows, as indices into the task-id order."""
    R = len(c["run"])
    if name == "asc":
        return np.arange(R)
    if name == "desc":
        return np.arange(R)[::-1].copy()
    return np.random.default_rng(SEEDS[(c["regime"], name)]).permutation(R)


def side(c, order, cols):
    """+1 when the fold in `order` lies above the task-id fold in every column of `cols`, -1 below, else 0."""
    d = [np.sign(running_total(c, col, order) - running_total(c, col)) for col in cols]
    return int(d[0]) if d and all(x == d[0] for x in d) else 0


def find_seed(c, want, limit=1000):
    """The first seed whose permutation folds above (want = +1) or below (-1) in every order-sensitive column."""
    cols = sensitive_cols(c)
    for s in range(limit):
        if side(c, np.random.default_rng(s).permutation(len(c["run"])), cols) == want:
            return s
    return None


def cut(c, queue_idx, col, k):
    """The boundary position of column `col` nearest k from above: k itself for cpus and mem (every request is
    positive), for gpus the first k' >= k whose job and the next ask for gpus, so one ulp moves the cut by one job."""
    if col != "gpus":
        return k
    g = [c["pend"][j][1]["gpus"] for j in queue_idx]
    return next(i for i in range(k, len(g)) if g[i - 1] > 0 and g[i] > 0)


def quota_at(c, queue_idx, col, k, start=None):
    """q*: the left fold of the first k queued requests of `col` (queue_idx: pending indices in rank order)
    continued from `start` (None: the task-id fold of the running column)."""
    s = running_total(c, col) if start is None else float(start)
    return F.left_total([c["pend"][j][1][col] for j in queue_idx[:k]], s)


def pool_quota(col, q):
    """A pool quota that cuts on `col` at q; the other columns unlimited."""
    return abi.make_pool_quota(dict({k: 1e18 for k in ("count", "cpus", "mem", "gpus")}, **{col: q}))


def group_usage(c):
    """The quota group's usage a shim builds from the pool totals: [count, cpus, mem, gpus] in task-id order."""
    return np.array([float(len(c["run"]))] + [running_total(c, col) for col in COLS])


def offers(n=60, seed=5):
    """A small offer table that places part of the queue."""
    rng = np.random.default_rng(seed)
    return abi.OffersSoA(n=n, hostname_id=np.arange(n, dtype=np.int32), name_rank=rng.permutation(n).astype(np.int32),
                         cpus=rng.choice(np.array([8.0, 16.0, 32.0]), n),
                         mem=rng.choice(np.array([16384.0, 32768.0, 65536.0]), n),
                         run_cpus=np.zeros(n), run_mem=np.zeros(n),
                         run_count=np.zeros(n, np.int32), n_attr_cols=0)
