"""-m gpu: the resident pool state (cook_state_apply / cook_state_rank / cook_state_match).

A Python model keeps the same rows as the handle; after every batch the resident rank and match must
equal cook_rank / cook_match run on host tables built from the model (and rank the oracle), whatever the
slot layout, across capacity doublings and arena compactions.  Plus the upload accounting and the
all-or-nothing errors.
"""
import numpy as np
import pytest

from cook_b200 import abi, traces
from cook_b200.engine import CookError, GpuEngine

pytestmark = pytest.mark.gpu

JOB_COLS = ("cpus", "mem", "gpus", "ports", "allowed", "plugin_accept", "gpu_model", "disk_request", "disk_type",
            "est_end_ms", "ckpt_location", "reserved_host")
DEFAULTS = dict(gpus=0.0, ports=0, allowed=1, plugin_accept=1, gpu_model=-1, disk_request=-1.0, disk_type=-1,
                est_end_ms=-1, ckpt_location=-1, reserved_host=-1)
DT = dict(cpus=np.float64, mem=np.float64, gpus=np.float64, ports=np.int32, allowed=np.uint8,
          plugin_accept=np.uint8, gpu_model=np.int32, disk_request=np.float64, disk_type=np.int32,
          est_end_ms=np.int64, ckpt_location=np.int32, reserved_host=np.int32)


def _lists(soa, off, *vals):
    o = soa.col(off)
    if o is None:
        return [[] for _ in range(soa.n)]
    cols = [soa.col(v) for v in vals]
    return [list(zip(*[c[o[i]:o[i + 1]].tolist() for c in cols])) if len(cols) > 1 else cols[0][o[i]:o[i + 1]].tolist()
            for i in range(soa.n)]


def pool_rows(t):
    """The trace's pending jobs as dict rows keyed by job id, and its running tasks keyed by task id."""
    jobs, pc = t["jobs"], t["cols"]["pending"]
    nov, att, grp = _lists(jobs, "novel_off", "novel_host"), _lists(jobs, "attr_off", "attr_col", "attr_val"), \
        _lists(jobs, "group_off", "group_idx")
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


def jobs_soa(rows):
    """JobsSoA (+ priority, job id) of [(job_id, row)]."""
    n = len(rows)
    kw = {c: np.array([r[c] for _, r in rows], DT[c]) for c in JOB_COLS}
    kw["user"] = np.array([r["user"] for _, r in rows], np.int32)
    kw["novel_off"], kw["novel_host"] = abi.csr([r["novel"] for _, r in rows])
    kw["attr_off"], kw["attr_col"] = abi.csr([[c for c, _ in r["attr"]] for _, r in rows])
    _, kw["attr_val"] = abi.csr([[v for _, v in r["attr"]] for _, r in rows])
    kw["group_off"], kw["group_idx"] = abi.csr([r["groups"] for _, r in rows])
    return (abi.JobsSoA(n=n, **kw), np.array([r["priority"] for _, r in rows], np.int32),
            np.array([j for j, _ in rows], np.int64))


def tasks_soa(rows):
    return abi.make_tasks(**{k: np.array([r[k] for r in rows], np.int64 if k in ("start_time", "task_id", "job_id")
                                         else np.int32 if k in ("user", "priority") else np.float64)
                             for k in ("user", "priority", "start_time", "task_id", "job_id", "cpus", "mem", "gpus")})


def delta(reset=False, up=(), rm=(), run_up=(), run_rm=()):
    """up: [(job_id, row)], run_up: [row]."""
    pend, prio, jid = jobs_soa(list(up)) if up else (None, None, None)
    return abi.make_delta(reset=reset, pending=pend, pending_priority=prio, pending_job_id=jid, pending_rm=list(rm),
                          running=tasks_soa(list(run_up)) if run_up else None, running_rm=list(run_rm))


class Model:
    """What the handle should hold, and the host tables cook_rank / cook_match take."""

    def __init__(self):
        self.pend, self.run = {}, {}

    def apply(self, d_up=(), d_rm=(), r_up=(), r_rm=(), reset=False):
        if reset:
            self.pend, self.run = {}, {}
        for j in d_rm:
            del self.pend[j]
        for t in r_rm:
            del self.run[t]
        for j, r in d_up:
            self.pend[j] = r
        for r in r_up:
            self.run[r["task_id"]] = r

    def tables(self):
        """A column (or list) whose every value is absent is passed as NULL, as a host shim passes an absent
        constraint; the resident state makes the same choice from its counts.  (cook_match picks its cpu+mem
        kernel by which columns are present, and the two kernels may report a different fail reason.)"""
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


class Pool:
    """A trace as a pool: the handle under test, the host-table handle, and the model."""

    def __init__(self, t, groups=None):
        self.t, self.users, self.offers, self.groups = t, t["users"], t["offers"], groups
        self.params = traces.match_params(min(1000, t["jobs"].n), host_lifetime_mins=t.get("host_lifetime_mins", 0))
        self.max_ports = int(t["jobs"].col("ports").max()) if t["jobs"].col("ports") is not None else 0
        self.gpu, self.ref, self.m = GpuEngine(pool_name="state"), GpuEngine(pool_name="host"), Model()
        self.queue, self.gone = [], set()   # the last rank's queue, the jobs removed or replaced since

    def close(self):
        self.gpu.close()
        self.ref.close()

    def apply(self, up=(), rm=(), run_up=(), run_rm=(), reset=False):
        self.gpu.state_apply(delta(reset, up, rm, run_up, run_rm))
        self.m.apply(up, rm, run_up, run_rm, reset)
        self.gone |= set(rm) | {j for j, _ in up}
        if reset:
            self.gone |= set(self.queue)

    def rank(self, oracle=None):
        q = self.gpu.state_rank(self.users)
        running, pending, _, jid = self.m.tables()
        host = self.ref.rank(running if running.n else None, pending, self.users)
        assert np.array_equal(q, jid[host["ranked"]]), "resident rank != cook_rank on the same rows"
        if oracle is not None and pending.n:
            o = oracle.rank(running if running.n else None, pending, self.users)
            assert np.array_equal(q, jid[o["ranked"]]), "resident rank != oracle"
        self.queue, self.gone = q.tolist(), set()
        return q

    def match(self):
        got = self.gpu.state_match(self.offers, self.users, self.params, groups=self.groups, max_ports=self.max_ports)
        _, _, jobs, jid = self.m.tables()
        pos = {j: i for i, j in enumerate(jid.tolist())}
        ranked = np.array([pos[j] for j in self.queue if j not in self.gone], np.int32)
        if len(ranked) == 0:
            assert len(got["considerable"]) == 0
            return got
        want = self.ref.match(ranked, jobs, self.offers, self.users, self.params, groups=self.groups,
                              max_ports=self.max_ports)
        assert np.array_equal(got["considerable"], jid[want["considerable"]])
        for k in ("assign", "ports", "fail"):
            assert np.array_equal(got[k], want[k]), k
        n = len(got["considerable"])
        if n:
            k = np.unique(np.linspace(0, n - 1, min(n, 16)).astype(np.int32))
            assert self.gpu.match_failures(k) == self.ref.match_failures(k)
        nu = self.users.n_users
        assert np.array_equal(self.gpu.exchange_usage(nu), self.ref.exchange_usage(nu))
        return got


def _c2(seed, cpus=(0.5, 1, 2, 4, 8)):
    return traces.gen_pool(seed, 3000, 200, 30, 600, cpus_choices=cpus)


def _c3(seed):
    return traces.gen_c3_pool(seed, n_jobs=2500, n_offers=160, n_users=24, n_running=500)


def _churn(p, rng, reserve, t_next, launched):
    """One realistic batch: launches of the last match, finishes, submissions, kills, priority changes."""
    up, rm, run_up, run_rm = [], [], [], []
    for j in launched:
        r = p.m.pend[j]
        rm.append(j)
        t_next[0] += 2
        run_up.append(dict(user=r["user"], priority=r["priority"], start_time=1_700_000_000_000 + t_next[0],
                           task_id=t_next[0] + 1, job_id=j, cpus=r["cpus"], mem=r["mem"], gpus=r["gpus"]))
    fin = [t for t in p.m.run if rng.random() < 0.03]
    run_rm += fin
    for _ in range(min(len(fin) + 5, len(reserve))):
        up.append(reserve.pop())
    live = [j for j in p.m.pend if j not in set(rm)]
    rng.shuffle(live)
    rm += live[:4]                                   # kills
    for j in live[4:12]:                             # priority / allowed / reservation changes
        r = dict(p.m.pend[j])
        r["priority"] = int(rng.choice([10, 50, 90]))
        r["allowed"] = int(rng.random() < 0.9)
        up.append((j, r))
    return up, rm, run_up, run_rm


@pytest.mark.parametrize("kind", ["c2", "c3"])
def test_equivalence_random_deltas(kind, oracle):
    t = _c2(11) if kind == "c2" else _c3(13)
    p = Pool(t, t.get("groups"))
    try:
        pend, run = pool_rows(t)
        items = sorted(pend.items())
        rng = np.random.default_rng(5)
        cut = int(len(items) * 0.85)
        reserve = items[cut:]
        p.apply(up=items[:cut], run_up=list(run.values()), reset=True)
        t_next = [10 ** 9]
        for cycle in range(5):
            p.rank(oracle if cycle % 2 == 0 else None)
            launched = []
            for rnd in range(2):                     # two match rounds per rank, a kill between rank and match
                live_q = [j for j in p.queue if j not in p.gone]
                if live_q:
                    p.apply(rm=[live_q[int(rng.integers(len(live_q)))]])
                got = p.match()
                launched = [int(j) for j, a in zip(got["considerable"], got["assign"]) if a >= 0][:40]
                up, rm, run_up, run_rm = _churn(p, rng, reserve, t_next, launched)
                p.apply(up, rm, run_up, run_rm)
            if cycle == 3:                            # new leadership
                pend_now = sorted(p.m.pend.items())
                run_now = list(p.m.run.values())
                p.apply(up=pend_now, run_up=run_now, reset=True)
                with pytest.raises(CookError):       # nothing survives a reset: old ids are unknown to removals
                    p.gpu.state_apply(delta(rm=[10 ** 12]))
        p.rank(oracle)
        p.match()
    finally:
        p.close()


def test_layout_independence():
    t = _c2(21, cpus=(0.1, 0.5, 1.0, 2.0))           # off the binary grid: the serial folds run
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    a, b = Pool(t), Pool(t)
    try:
        a.apply(up=items, run_up=list(run.values()))
        rng = np.random.default_rng(3)
        perm = rng.permutation(len(items))
        junk = [(10 ** 11 + i, items[i][1]) for i in range(500)]
        b.apply(up=junk)                              # churn that frees slots the real rows then reuse
        b.apply(rm=[j for j, _ in junk])
        b.apply(up=[items[i] for i in perm[: len(perm) // 2]])
        rr = list(run.values())
        b.apply(up=[items[i] for i in perm[len(perm) // 2:]], run_up=[rr[i] for i in rng.permutation(len(rr))])
        qa, qb = a.rank(), b.rank()
        assert np.array_equal(qa, qb)
        ma, mb = a.match(), b.match()
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
    finally:
        a.close()
        b.close()


def test_growth_and_compaction():
    t = _c3(31)
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    p = Pool(t, t.get("groups"))
    try:
        hosts = t["offers"].col("hostname_id")
        for i in range(0, len(items), 300):           # from empty past several capacity doublings
            p.apply(up=items[i:i + 300])
            if i % 900 == 0:
                p.rank()
                p.match()
        p.apply(run_up=list(run.values()))
        p.rank()
        p.match()
        long_rows = []
        for k, (j, r) in enumerate(items[:400]):      # long novel-host lists, upserted then removed
            r = dict(r)
            r["novel"] = hosts[(np.arange(60) * 7 + k) % len(hosts)].tolist()
            long_rows.append((j, r))
        p.apply(up=long_rows)
        p.rank()
        p.match()
        p.apply(rm=[j for j, _ in long_rows[:300]])   # dead entries now outnumber the live ones
        p.apply(up=[items[k] for k in range(300, 400)])
        p.rank()
        p.match()
    finally:
        p.close()


def _nb(*arrays):
    return sum(a.nbytes for a in arrays if isinstance(a, np.ndarray))


@pytest.mark.parametrize("scale", [1, 2])
def test_accounting(scale):
    t = traces.gen_pool(41, 2000 * scale, 150, 20, 400 * scale)
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    p = Pool(t)
    try:
        d = delta(up=items, run_up=list(run.values()))
        p.gpu.state_apply(d)
        p.m.apply(items, (), list(run.values()))
        pj, rt = d.col("pending"), d.col("running")
        lists = {"novel_host": "novel_off", "attr_col": "attr_off", "attr_val": "attr_off", "group_idx": "group_off"}
        want = sum(4 * int(pj.col(lists[n])[-1]) if n in lists else pj.col(n).nbytes
                   for n, _ in pj._fields_ if isinstance(pj.col(n), np.ndarray))   # a list uploads its entries
        want += _nb(d.col("pending_priority"), d.col("pending_job_id"), *[rt.col(n) for n, _ in rt._fields_])
        want += 4 * (pj.n + rt.n)                      # one slot per row
        st = p.gpu.last_stats(abi.PHASE_STATE)
        assert st["h2d_bytes"] == want and st["n_launches"] >= 2
        p.rank()
        u = t["users"]
        rk = p.gpu.last_stats(abi.PHASE_RANK)
        assert rk["h2d_bytes"] == _nb(*[u.col(n) for n in ("name_rank", "div_mem", "div_cpus", "div_gpus",
                                                            "quota_count", "quota_cpus", "quota_mem", "quota_gpus")])
        assert rk["n_launches"] > 0
        got = p.match()
        o = t["offers"]
        # name_rank stays on the host; the offer order it gives (O int32) is uploaded instead
        want = _nb(*[o.col(n) for n, _ in o._fields_]) + _nb(*[u.col(n) for n in (
            "quota_count", "quota_cpus", "quota_mem", "quota_gpus", "usage_count", "usage_cpus", "usage_mem",
            "usage_gpus", "tokens")])
        assert got["stats"]["h2d_bytes"] == want      # the same at scale 1 and 2: nothing per resident job
        assert got["stats"]["n_launches"] > 0
        # a launch batch uploads its own rows only
        j = int(got["considerable"][0])
        r = p.m.pend[j]
        task = dict(user=r["user"], priority=r["priority"], start_time=1, task_id=7, job_id=j, cpus=r["cpus"],
                    mem=r["mem"], gpus=r["gpus"])
        d = delta(rm=[j], run_up=[task])
        p.gpu.state_apply(d)
        assert p.gpu.last_stats(abi.PHASE_STATE)["h2d_bytes"] == _nb(*[d.col("running").col(n) for n, _ in
                                                                         abi.TasksSoA._fields_]) + 4 + 4
    finally:
        p.close()


def test_errors():
    t = _c3(51)
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    p = Pool(t, t["groups"])
    try:
        with pytest.raises(CookError) as e:           # match before any rank
            p.gpu.state_match(p.offers, p.users, p.params, groups=p.groups)
        assert e.value.code == abi.COOK_E_BADARG
        p.apply(up=items, run_up=list(run.values()))
        q0 = p.rank()

        def fails(fn, code=abi.COOK_E_BADARG):
            with pytest.raises(CookError) as e:
                fn()
            assert e.value.code == code
            assert np.array_equal(p.gpu.state_rank(p.users), q0)

        fails(lambda: p.gpu.state_apply(delta(rm=[items[0][0], 10 ** 12])))          # unknown id
        fails(lambda: p.gpu.state_apply(delta(up=[items[1]], rm=[items[1][0]])))      # an id twice
        fails(lambda: p.gpu.state_apply(delta(up=[items[2], items[2]])))
        bad = delta(up=items[3:5])
        bad.col("pending").col("novel_off")[1] = -1                                   # malformed CSR
        fails(lambda: p.gpu.state_apply(bad))
        nu = p.users.n_users
        r = dict(items[5][1]); r["user"] = nu
        p.apply(up=[(10 ** 12, r)])                    # a user code the user table does not cover
        with pytest.raises(CookError) as e:
            p.gpu.state_rank(p.users)
        assert e.value.code == abi.COOK_E_BADARG
        p.apply(rm=[10 ** 12])
        assert np.array_equal(p.gpu.state_rank(p.users), q0)
        G = p.groups.n_groups
        r = dict(items[6][1]); r["groups"] = [G]       # a group code the groups table does not cover
        p.apply(up=[(10 ** 12 + 1, r)])
        with pytest.raises(CookError) as e:
            p.gpu.state_match(p.offers, p.users, p.params, groups=p.groups)
        assert e.value.code == abi.COOK_E_BADARG
        p.apply(rm=[10 ** 12 + 1])
        prm = traces.match_params(100, reuse_resident=1)
        fails(lambda: p.gpu.state_match(p.offers, p.users, prm, groups=p.groups))
        p.rank()
        p.match()
    finally:
        p.close()
