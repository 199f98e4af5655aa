"""The resident-pool model the state tests share: the row vocabulary, one delta builder, and one handle-plus-model.

A pending row is a dict of JOB_COLS plus user, priority and the lists novel (hostname codes), attr ([(column,
value)]) and groups, keyed by job id.  A running row is a dict of RUN_KEYS plus host (a hostname code) and groups,
keyed by task id.  `delta` turns rows into a cook_state_delta; its options say which of the input's columns are
NULL.  `Pool` keeps a handle and the rows it should hold, and projects them onto the host tables cook_rank,
cook_match and cook_rebalance take.
"""
import numpy as np

import fold_ref as F
from cook_b200 import abi, traces
from cook_b200.engine import GpuEngine
from cotask_ref import cotasks
from usage_ref import KEYS, running_usage

START = 1_700_000_000_000
OPTIONAL = ("gpus", "ports", "allowed", "plugin_accept", "gpu_model", "disk_request", "disk_type", "est_end_ms",
            "ckpt_location", "reserved_host")
JOB_COLS = ("cpus", "mem") + OPTIONAL
DEFAULTS = dict(gpus=0.0, ports=0, allowed=1, plugin_accept=1, gpu_model=-1, disk_request=-1.0, disk_type=-1,
                est_end_ms=-1, ckpt_location=-1, reserved_host=-1)
DT = dict(cpus=np.float64, mem=np.float64, gpus=np.float64, ports=np.int32, allowed=np.uint8, plugin_accept=np.uint8,
          gpu_model=np.int32, disk_request=np.float64, disk_type=np.int32, est_end_ms=np.int64, ckpt_location=np.int32,
          reserved_host=np.int32)
RUN_KEYS = ("user", "priority", "start_time", "task_id", "job_id", "cpus", "mem", "gpus")
RUN_DEFAULTS = dict(priority=50, start_time=START, gpus=0.0, host=-1, groups=[])


# ---- rows of traces ------------------------------------------------------------------------------------------
def _lists(soa, off, *vals):
    o = soa.col(off)
    if o is None:
        return [[] for _ in range(soa.n)]
    cols = [soa.col(v) for v in vals]
    return [list(zip(*[c[o[i]:o[i + 1]].tolist() for c in cols])) if len(cols) > 1 else cols[0][o[i]:o[i + 1]].tolist()
            for i in range(soa.n)]


def _pending_lists(jobs):
    return (_lists(jobs, "novel_off", "novel_host"), _lists(jobs, "attr_off", "attr_col", "attr_val"),
            _lists(jobs, "group_off", "group_idx"))


def pool_rows(t):
    """The trace's pending jobs as dict rows keyed by job id, and its running tasks keyed by task id."""
    jobs, pc = t["jobs"], t["cols"]["pending"]
    nov, att, grp = _pending_lists(jobs)
    pend = {}
    for i in range(jobs.n):
        r = {"user": int(pc["user"][i]), "priority": int(pc["priority"][i])}
        for c in JOB_COLS:
            col = jobs.col(c)
            r[c] = col[i].item() if col is not None else DEFAULTS[c]
        r["novel"], r["attr"], r["groups"] = nov[i], att[i], grp[i]
        pend[int(pc["job_id"][i])] = r
    rc = t["cols"]["running"]
    run = {int(rc["task_id"][i]): {k: rc[k][i].item() for k in rc} for i in range(len(rc["task_id"]))}
    return pend, run


def remap_hosts(r, seed):
    """The gen_rebalance dict `r` with hostname codes 3 * perm + 7: the host table, novel-host lists and
    cotask hosts carry codes; running tasks keep their table index.  Returns the code of each index."""
    H = r["hosts"].n
    codes = (3 * np.random.default_rng(seed).permutation(H) + 7).astype(np.int32)
    r["hosts"] = with_fields(r["hosts"], hostname_id=codes)
    j = r["pending"]
    if j.col("novel_off") is not None and j.col("novel_off")[-1] > 0:
        r["pending"] = with_fields(j, novel_host=codes[j.col("novel_host")])
    g = r["groups"]
    if g is not None and g.col("cot_off")[-1]:
        r["groups"] = with_fields(g, cot_hostname_id=codes[g.col("cot_hostname_id")])
    return codes


def rows_of(r, codes):
    """The rebalance pool's pending jobs {job_id: row} and running tasks {task_id: row (with its hostname code)}."""
    j = r["pending"]
    nov, att, grp = _pending_lists(j)
    pend = {}
    for i in range(j.n):
        row = dict(DEFAULTS, user=int(j.col("user")[i]), priority=int(r["pending_priority"][i]),
                   cpus=float(j.col("cpus")[i]), mem=float(j.col("mem")[i]))
        if j.col("ckpt_location") is not None:
            row["ckpt_location"] = int(j.col("ckpt_location")[i])
        row["novel"], row["attr"], row["groups"] = nov[i], att[i], grp[i]
        pend[int(r["pending_job_id"][i])] = row
    t = r["running"].col("t")
    host = r["running"].col("host")
    run = {}
    for i in range(t.n):
        row = {k: t.col(k)[i].item() for k in RUN_KEYS}
        row["host"] = int(codes[host[i]])
        run[row["task_id"]] = row
    return pend, run


def c2(seed, cpus=(0.5, 1, 2, 4, 8)):
    return traces.gen_pool(seed, 3000, 200, 30, 600, cpus_choices=cpus)


def c3(seed):
    return traces.gen_c3_pool(seed, n_jobs=2500, n_offers=160, n_users=24, n_running=500)


def rebalance_trace(seed, constraints, n_running=3000, n_pending=300, n_hosts=200, n_users=40, mp=24):
    """A gen_rebalance pool with remapped hostname codes, and the codes."""
    r = traces.gen_rebalance(seed, n_running, n_pending, n_hosts, n_users, max_preemption=mp,
                             constraints=constraints)
    return r, remap_hosts(r, seed + 1)


def churn(p, rng, reserve, t_next, launched):
    """One realistic batch: launches of the last match, finishes, submissions, kills, priority changes."""
    up, rm, run_up, run_rm = [], [], [], []
    for j in launched:
        r = p.pend[j]
        rm.append(j)
        t_next[0] += 2
        run_up.append(dict(user=r["user"], priority=r["priority"], start_time=START + t_next[0],
                           task_id=t_next[0] + 1, job_id=j, cpus=r["cpus"], mem=r["mem"], gpus=r["gpus"]))
    fin = [t for t in p.run if rng.random() < 0.03]
    run_rm += fin
    for _ in range(min(len(fin) + 5, len(reserve))):
        up.append(reserve.pop())
    live = [j for j in p.pend if j not in set(rm)]
    rng.shuffle(live)
    rm += live[:4]                                   # kills
    for j in live[4:12]:                             # priority / allowed / reservation changes
        r = dict(p.pend[j])
        r["priority"] = int(rng.choice([10, 50, 90]))
        r["allowed"] = int(rng.random() < 0.9)
        up.append((j, r))
    return up, rm, run_up, run_rm


def task_of(row, job_id, task_id, start, host):
    """The running row a launch makes of pending row `row`."""
    return dict(user=row["user"], priority=row.get("priority", RUN_DEFAULTS["priority"]), start_time=int(start),
                task_id=int(task_id), job_id=int(job_id), cpus=row["cpus"], mem=row["mem"],
                gpus=row.get("gpus", DEFAULTS["gpus"]), host=int(host), groups=list(row.get("groups", [])))


def stored(up, run_up, drop=(), hosts=True, lists=True, gpus=True):
    """The rows a delta leaves on the handle: a NULL column or list stores its default."""
    if drop:
        up = [(j, dict(r, **{c: [] if c in ("novel", "attr", "groups") else DEFAULTS[c] for c in drop})) for j, r in up]
    over = {k: v for k, v, sent in (("host", -1, hosts), ("groups", [], lists)) if not sent}
    if not gpus:
        over["gpus"] = 0.0
    if over:
        run_up = [dict(r, **{k: v for k, v in over.items() if k in r or k == "gpus"}) for r in run_up]
    return up, run_up


BIG = 2.0 ** 35   # mixed: on the grid, but a user of 256 rows or more passes 2^43


# ---- running and pending rows of the usage and derived tests ----------------------------------------------
def amounts(rng, regime, n, big=None):
    """cpus, mem, gpus of n rows.  grid: halves and 512 MiB steps; off: tenths and sevenths; mixed: grid, the
    rows of `big` carry mem just under 2^35 with 2^-10 parts."""
    if regime == "off":
        cpus = rng.choice(np.array([0.1, 0.3, 0.7, 1.1]), n)
        mem = rng.integers(1, 40000, n) / 7.0
        gpus = rng.choice(np.array([0.0, 0.0, 0.1, 1.0]), n)
    else:
        cpus = rng.choice(np.array([0.5, 1.0, 2.0, 4.0]), n)
        mem = 512.0 * rng.integers(1, 65, n)
        gpus = rng.choice(np.array([0.0, 0.0, 1.0, 2.0]), n)
        if regime == "mixed" and big is not None and big.any():
            mem[big] = BIG - F.GRID * rng.integers(1, 2 ** 20, int(big.sum()))
    return cpus.astype(np.float64), mem.astype(np.float64), gpus.astype(np.float64)


def zipf_users(rng, n, U):
    """A third of the rows belong to user 0, the rest spread over the others."""
    u = rng.integers(1, U, n).astype(np.int32)
    u[rng.random(n) < 1.0 / 3.0] = 0
    return u


def random_rows(rng, regime, n, U, tid0, hosts):
    user = zipf_users(rng, n, U)
    cpus, mem, gpus = amounts(rng, regime, n, user == 0)
    tid = tid0 + 2 * rng.permutation(n).astype(np.int64)
    return [dict(user=int(user[i]), task_id=int(tid[i]), job_id=int(tid[i]) + 1, cpus=float(cpus[i]), mem=float(mem[i]),
                 gpus=float(gpus[i]), host=int(rng.choice(hosts))) for i in range(n)]


def pending_rows(rng, regime, n, U, jid0, codes):
    user = zipf_users(rng, n, U)
    cpus, mem, gpus = amounts(rng, regime, n, user == 0)
    return [dict(job_id=jid0 + 2 * i, user=int(user[i]), cpus=float(cpus[i]), mem=float(mem[i]), gpus=float(gpus[i]),
                 novel=[int(x) for x in rng.choice(codes, int(rng.integers(1, 4)), replace=False)]) for i in range(n)]


def keyed(rows):
    """[(job id, row)] of pending rows that carry their job_id."""
    return [(r["job_id"], r) for r in rows]


# ---- rows -> deltas and host tables ---------------------------------------------------------------------------
def pending_kw(rows, drop=()):
    """make_delta's pending arguments of [(job id, row)]; the columns and lists in `drop` are passed as NULL.  A
    column a row lacks takes DEFAULTS, a priority 50."""
    kw = {c: np.array([r.get(c, DEFAULTS.get(c)) for _, r in rows], DT[c]) for c in JOB_COLS if c not in drop}
    kw["user"] = np.array([r["user"] for _, r in rows], np.int32)
    if "novel" not in drop:
        kw["novel_off"], kw["novel_host"] = abi.csr([r["novel"] for _, r in rows])
    if "attr" not in drop:
        kw["attr_off"], kw["attr_col"] = abi.csr([[c for c, _ in r["attr"]] for _, r in rows])
        kw["attr_val"] = abi.csr([[v for _, v in r["attr"]] for _, r in rows])[1]
    if "groups" not in drop:
        kw["group_off"], kw["group_idx"] = abi.csr([r["groups"] for _, r in rows])
    return dict(pending=abi.JobsSoA(n=len(rows), **kw),
                pending_priority=np.array([r.get("priority", RUN_DEFAULTS["priority"]) for _, r in rows], np.int32),
                pending_job_id=np.array([j for j, _ in rows], np.int64))


def running_kw(rows, hosts=True, lists=True, gpus=True):
    """make_delta's running arguments of [row]: hostname codes unless not `hosts`, group lists unless not `lists`,
    the gpus column unless not `gpus` (NULL otherwise).  A key a row lacks takes RUN_DEFAULTS."""
    get = lambda r, k: r[k] if k in r else RUN_DEFAULTS[k]
    t = {k: np.array([get(r, k) for r in rows], np.int64 if k in ("start_time", "task_id", "job_id") else
                     np.int32 if k in ("user", "priority") else np.float64)
         for k in RUN_KEYS if k != "gpus" or gpus}
    kw = dict(running=abi.TasksSoA(n=len(rows), **t))
    if hosts:
        kw["running_hostname_id"] = np.array([get(r, "host") for r in rows], np.int32)
    if lists:
        kw["running_group_off"], kw["running_group_idx"] = abi.csr([get(r, "groups") for r in rows])
    return kw


def drop_all_but(*keep):
    """The `drop` of pending rows that carry user, cpus, mem and only the optional columns and lists in `keep`."""
    return tuple(c for c in OPTIONAL + ("novel", "attr", "groups") if c not in keep)


def delta(reset=False, up=(), rm=(), run_up=(), run_rm=(), drop=(), hosts=False, lists=False, gpus=True):
    """The cook_state_delta of pending upserts [(job id, row)], removals, running upserts [row] and removals."""
    up, run_up = list(up), list(run_up)
    kw = dict(pending_kw(up, drop)) if up else {}
    if run_up:
        kw.update(running_kw(run_up, hosts, lists, gpus))
    return abi.make_delta(reset=reset, pending_rm=list(rm), running_rm=list(run_rm), **kw)


def jobs_soa(rows):
    """JobsSoA, priority and job id of [(job_id, row)], every column present."""
    kw = pending_kw(rows)
    return kw["pending"], kw["pending_priority"], kw["pending_job_id"]


def tasks_soa(rows):
    return running_kw(rows, hosts=False, lists=False)["running"]


def with_fields(s, **over):
    """A copy of the SoA struct `s` with fields replaced (None: NULL)."""
    kw = {n: s.col(n) if t in abi._NP else getattr(s, n) for n, t in s._fields_}
    kw.update(over)
    return type(s)(**kw)


def nb(*arrays):
    return sum(a.nbytes for a in arrays if isinstance(a, np.ndarray))


def decisions_eq(got, want):
    keys = ("job_id", "pending_idx", "host", "victims", "dru", "mem", "cpus", "gpus")
    assert [tuple(d[k] for k in keys) for d in got] == [tuple(d[k] for k in keys) for d in want]


# ---- the handle and its model ---------------------------------------------------------------------------------
class Pool:
    """A resident handle (`gpu`), a host-table handle (`ref`) and the model of the rows the handle holds: pending
    {job id: row}, running {task id: row}, the last rank's `queue` and the jobs removed or replaced since (`gone`).

    The tables the checks read are attributes a test sets: users, offers, groups, params and max_ports for rank and
    match; hosts (a HostTable), codes (each host index's hostname code) and rparams for the rebalance.  What the
    upserts carry by default: `drop`, the pending columns and lists passed as NULL; `send_hosts` and `send_lists`,
    whether the running upserts carry hostname codes and group lists (else NULL)."""

    def __init__(self, name="state", dru_mode=0, drop=(), send_hosts=False, send_lists=False, ref=None, **tables):
        self.gpu, self._ref = GpuEngine(pool_name=name, dru_mode=dru_mode), ref
        self.drop, self.send_hosts, self.send_lists = drop, send_hosts, send_lists
        self.users = self.offers = self.groups = self.params = self.hosts = self.codes = self.rparams = None
        self.max_ports = 0
        self.__dict__.update(tables)
        self.pend, self.run = {}, {}
        self.queue, self.gone = [], set()

    @classmethod
    def of_trace(cls, t, groups=None, name="state", **kw):
        """A pool over a gen_pool / gen_c3_pool trace: its users and offers, a match of up to 1000 jobs."""
        kw.setdefault("users", t["users"])
        ports = t["jobs"].col("ports")
        return cls(name, offers=t["offers"], groups=groups, max_ports=int(ports.max()) if ports is not None else 0,
                   params=traces.match_params(min(1000, t["jobs"].n), host_lifetime_mins=t.get("host_lifetime_mins", 0)),
                   **kw)

    @classmethod
    def of_rebalance(cls, r, codes, dru_mode=0, name="state"):
        """A pool over a rebalance_trace: its users, host table, groups and rebalance parameters."""
        return cls(name, dru_mode, send_hosts=True, users=r["users"], hosts=r["hosts"],
                   groups=r["groups"], rparams=r["params"], codes=codes)

    @property
    def ref(self):
        """The host-table handle (another pool's when given), opened on first use."""
        if self._ref is None:
            self._ref = GpuEngine(pool_name="host")
        return self._ref

    def close(self):
        self.gpu.close()
        if self._ref is not None:
            self._ref.close()

    # -- changes, on the handle and the model --------------------------------------------------------------------
    def mirror(self, up=(), rm=(), run_up=(), run_rm=(), reset=False):
        """The model side of a delta."""
        if reset:
            self.pend, self.run = {}, {}
            self.gone |= set(self.queue)
        for j in rm:
            del self.pend[j]
        for t in run_rm:
            del self.run[t]
        for j, r in up:
            self.pend[j] = r
        for r in run_up:
            self.run[r["task_id"]] = r
        self.gone |= set(rm) | {j for j, _ in up}

    def apply(self, up=(), rm=(), run_up=(), run_rm=(), reset=False, drop=None, hosts=None, lists=None, gpus=True):
        up, run_up = list(up), list(run_up)
        drop = self.drop if drop is None else drop
        hosts = self.send_hosts if hosts is None else hosts
        lists = self.send_lists if lists is None else lists
        self.gpu.state_apply(delta(reset, up, rm, run_up, run_rm, drop, hosts, lists, gpus))
        up, run_up = stored(up, run_up, drop, hosts, lists, gpus)
        self.mirror(up, rm, run_up, run_rm, reset)

    def launch(self, jobs, tids, starts, hosts=None):
        """cook_state_launch: the jobs become running tasks (hosts None: host unknown)."""
        self.gpu.state_launch(jobs, tids, starts, hosts)
        self.mirror(rm=jobs, run_up=[task_of(self.pend[j], j, tids[k], starts[k], -1 if hosts is None else hosts[k])
                                     for k, j in enumerate(jobs)])

    def patch(self, jobs, clear=False, **cols):
        """cook_state_patch; the jobs keep their place in the queue."""
        if clear:
            self.pend = {j: dict(r, reserved_host=-1) if r.get("reserved_host", -1) != -1 else r
                         for j, r in self.pend.items()}
        for k, j in enumerate(jobs):
            self.pend[j] = dict(self.pend[j], **{c: int(v[k]) for c, v in cols.items() if v is not None})
        self.gpu.state_patch(jobs, clear_reservations=clear, **cols)

    def rank(self, **kw):
        q = self.gpu.state_rank(self.users, **kw)
        self.queue, self.gone = q.tolist(), set()
        return q

    def live_queue(self):
        return [j for j in self.queue if j not in self.gone]

    # -- host tables of the model ------------------------------------------------------------------------------------
    def tables(self):
        """cook_rank's running and pending tables, cook_match's jobs and the job ids, in job id order.  A column (or
        list) whose every value is absent is passed as NULL, as a host shim passes an absent constraint; the resident
        state makes the same choice from its counts.  (cook_match picks its cpu+mem kernel by which columns are
        present, and the two kernels may report a different fail reason.)"""
        ids = sorted(self.pend)
        jobs, prio, jid = jobs_soa([(j, self.pend[j]) for j in ids])
        kw = {n: jobs.col(n) for n, _ in jobs._fields_ if isinstance(jobs.col(n), np.ndarray)}
        for c in JOB_COLS[2:]:
            absent = np.all(kw[c] < 0) if c == "disk_request" else np.all(kw[c] == DEFAULTS[c])
            if absent and c != "disk_type":
                del kw[c]
        if "disk_request" not in kw:   # the disk type only counts with a request
            del kw["disk_type"]
        for off, vals in (("novel_off", ("novel_host",)), ("attr_off", ("attr_col", "attr_val")),
                          ("group_off", ("group_idx",))):
            if kw[off][-1] == 0:
                for n in (off,) + vals:
                    del kw[n]
        jobs = abi.JobsSoA(n=len(ids), **kw)
        pending = abi.make_tasks(user=jobs.col("user"), priority=prio, start_time=np.full(len(ids), abi.INT64_MAX),
                                 task_id=np.full(len(ids), -1, np.int64), job_id=jid, cpus=jobs.col("cpus"),
                                 mem=jobs.col("mem"), gpus=jobs.col("gpus"))
        running = tasks_soa([self.run[t] for t in sorted(self.run)])
        return running, pending, jobs, jid

    def ranked(self, queue):
        """The jobs table, the job ids and the positions of the queue's jobs in it."""
        _, _, jobs, jid = self.tables()
        pos = {j: i for i, j in enumerate(jid.tolist())}
        return jobs, jid, np.array([pos[j] for j in queue], np.int32)

    def taken(self):
        """The jobs cook_state_rebalance walks: the first max_preemption allowed jobs of the live queue."""
        return [j for j in self.live_queue() if self.pend[j]["allowed"]][:self.rparams.max_preemption]

    def rebalance_tables(self):
        """cook_rebalance's host tables of the same rows, and the task id of each running index."""
        idx = {int(c): i for i, c in enumerate(self.codes)}
        rows = [self.run[t] for t in sorted(self.run)]
        running = abi.RunningSoA(t=tasks_soa(rows), host=np.array([idx[r["host"]] for r in rows], np.int32))
        jobs, prio, jid = jobs_soa([(j, self.pend[j]) for j in self.taken()])
        return running, jobs, jid, prio, np.array([r["task_id"] for r in rows], np.int64)

    # -- the resident calls against the host-table calls --------------------------------------------------------------
    def check_rank(self, oracle=None, **kw):
        """state_rank, equal to cook_rank on the model's tables (and the oracle's rank).  kw: pool_quota,
        group_quota, group_usage and params, passed to all three."""
        q = self.rank(**kw)
        running, pending, _, jid = self.tables()
        host = self.ref.rank(running if running.n else None, pending, self.users, **kw)
        assert np.array_equal(q, jid[host["ranked"]]), "resident rank != cook_rank on the same rows"
        if oracle is not None and pending.n:
            o = oracle.rank(running if running.n else None, pending, self.users, **kw)
            assert np.array_equal(q, jid[o["ranked"]]), "resident rank != oracle"
        return q

    def quota_at(self, queue, key, k):
        """The pool quota on the last bit of the rank's fold: the `key` requests of the first k jobs of `queue` (job
        ids) folded on from the model's running usage, itself a left fold in ascending task id."""
        start = F.left_total([self.run[t][key] for t in sorted(self.run)])
        return F.left_total([self.pend[j][key] for j in queue[:k]], start)

    def check_match(self, offers=None):
        """state_match, equal to cook_match on the model's tables over the live queue, failure counts and the usage
        exchange included."""
        e = self.gpu
        offers = offers if offers is not None else self.offers
        got = e.state_match(offers, self.users, self.params, groups=self.groups, max_ports=self.max_ports)
        jobs, jid, ranked = self.ranked(self.live_queue())
        if len(ranked) == 0:
            assert len(got["considerable"]) == 0
            return got
        want = self.ref.match(ranked, jobs, offers, self.users, self.params, groups=self.groups,
                              max_ports=self.max_ports)
        assert np.array_equal(got["considerable"], jid[want["considerable"]]), "considerable"
        for k in ("assign", "ports", "fail"):
            assert np.array_equal(got[k], want[k]), k
        n = len(got["considerable"])
        if n:
            k = np.unique(np.linspace(0, n - 1, min(n, 16)).astype(np.int32))
            assert e.match_failures(k) == self.ref.match_failures(k)
        nu = self.users.n_users
        assert np.array_equal(e.exchange_usage(nu), self.ref.exchange_usage(nu))
        return got

    def want_rebalance(self, engine_):
        """cook_rebalance on the model's tables by engine_, as state_rebalance reports it."""
        running, jobs, jid, prio, tids = self.rebalance_tables()
        if jobs.n == 0:
            return []
        out = engine_.rebalance(running, jobs, jid, prio, self.hosts, self.users, self.rparams, groups=self.groups)
        R = len(tids)
        for d in out:
            d["job_id"] = int(jid[d["pending_idx"]])
            d["victims"] = [int(tids[v]) if v < R else -1 - (v - R) for v in d["victims"]]
        return out

    def check_rebalance(self, oracle=None):
        """state_rebalance, equal to cook_rebalance on the model's tables (and the oracle)."""
        got = self.gpu.state_rebalance(self.hosts, self.users, self.rparams, groups=self.groups)
        decisions_eq(got, self.want_rebalance(self.ref))
        if oracle is not None:
            decisions_eq(got, self.want_rebalance(oracle))
        return got


# ---- the running-side inputs of a match, from a model's running rows ---------------------------------------------
USAGE_FIELDS = ("usage_count", "usage_cpus", "usage_mem", "usage_gpus")
RUN_FIELDS = ("run_cpus", "run_mem", "run_count")
COT_FIELDS = ("cot_off", "cot_hostname_id", "cot_attr_val")


def fed_tables(offers, users, groups, usage, cot):
    """The tables of a sequenced call: usage (state_usage's dict) and cot (state_cotasks' triple) filled in."""
    users = with_fields(users, **{f: usage["user"][k] for f, k in zip(USAGE_FIELDS, KEYS)})
    offers = with_fields(offers, run_cpus=usage["run_cpus"], run_mem=usage["run_mem"], run_count=usage["run_count"])
    if groups is not None and cot is not None:
        groups = with_fields(groups, cot_off=np.asarray(cot[0], np.int32),
                             cot_hostname_id=np.asarray(cot[1] if len(cot[1]) else [0], np.int32),
                             cot_attr_val=np.asarray(cot[2] if len(cot[2]) else [0], np.int32))
    return offers, users, groups


def host_inputs(run_rows, offers, users, groups):
    """The same tables from a model's running rows (usage_ref / cotask_ref restatements)."""
    hn = offers.col("hostname_id") if offers.n else np.zeros(0, np.int32)
    usage = running_usage(run_rows, users.n_users, hn)
    cot = None
    if groups is not None and groups.n_groups:
        at = offers.col("attr")
        cot = cotasks(run_rows, groups.n_groups, groups.col("attr_col"), hn,
                      at.reshape(offers.n_attr_cols, offers.n) if at is not None and offers.n else None)
    return fed_tables(offers, users, groups, usage, cot)


# ---- pools whose rows matter by their groups and hosts ----------------------------------------------------------
def group_pool(name):
    """A resident handle and its model: pending upserts carry user, cpus, mem and group lists only, running upserts
    hostname codes and group lists."""
    return Pool(name, drop=drop_all_but("groups"), send_hosts=True, send_lists=True)


def group_row(**kw):
    """A row of one cpu and 64 MiB."""
    return dict(cpus=1.0, mem=64.0, **kw)


class K13:
    """One pool through the resident cycle: jobs submitted as pending rows, ranked, matched with cotasks derived
    from the running rows an earlier launch created, and the placed jobs launched on the hosts the match chose."""

    def __init__(self, oracle, groups):
        self.o, self.e = oracle, group_pool("k13")
        self.kind = np.array([g["kind"] for g in groups], np.int32)
        self.col = np.array([g.get("col", -1) for g in groups], np.int32)
        self.minimum = np.array([g.get("minimum", 0) for g in groups], np.int32)
        self.users, self.code, self.jid, self.tid = abi.make_users(1), {}, 1000, 50

    def close(self):
        self.e.close()

    def offers(self, spec, n_attr_cols=1):
        for o in spec:
            self.code.setdefault(o["host"], len(self.code))
        O = len(spec)
        attr = np.zeros((n_attr_cols, O), np.int32)
        for i, o in enumerate(spec):
            for c, v in o.get("attrs", {}).items():
                attr[c, i] = v
        order = sorted(range(O), key=lambda i: spec[i]["host"])
        rank = np.zeros(O, np.int32)
        rank[order] = np.arange(O, dtype=np.int32)
        return abi.OffersSoA(n=O, hostname_id=np.array([self.code[o["host"]] for o in spec], np.int32), name_rank=rank,
                             cpus=np.array([o["cpus"] for o in spec]), mem=np.array([o.get("mem", 100000.0) for o in spec]),
                             run_cpus=np.zeros(O), run_mem=np.zeros(O), run_count=np.zeros(O, np.int32),
                             n_attr_cols=n_attr_cols, attr=attr.reshape(-1))

    def submit(self, n, group=0):
        rows = [(self.jid + 2 * i, group_row(user=0, groups=[group])) for i in range(n)]
        self.jid += 2 * n
        self.e.apply(up=rows)

    def jobs(self):
        """The live job ids in order and the host table of their rows."""
        ids = sorted(self.e.pend)
        return ids, pending_kw([(j, self.e.pend[j]) for j in ids], self.e.drop)["pending"]

    def launch_placed(self, m, offers):
        """Launch the jobs match m placed on the hosts it chose."""
        placed = m["assign"] >= 0
        jl = m["considerable"][placed].tolist()
        tids = [self.tid + 3 * i for i in range(len(jl))]
        self.tid += 3 * len(jl) + 3
        self.e.launch(jl, tids, np.full(len(jl), START, np.int64), offers.col("hostname_id")[m["assign"][placed]])

    def groups(self, cot):
        vals = [np.asarray(x if len(x) else [0], np.int32) for x in cot[1:]]   # empty: a valid pointer all the same
        return abi.Groups(n_groups=len(self.kind), kind=self.kind, attr_col=self.col, minimum=self.minimum,
                          cot_off=np.asarray(cot[0], np.int32), cot_hostname_id=vals[0], cot_attr_val=vals[1])
