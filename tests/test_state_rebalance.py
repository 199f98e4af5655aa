"""cook_state_rebalance: the rebalancer over the resident pool state.

A Python model keeps the same rows as the handle; the resident rebalance must equal cook_rebalance run on host
tables built from the model (running tasks by task id, each on the table index of its hostname code; pending
jobs the first max_preemption allowed jobs of the last rank's queue that are still live), and the oracle, over a
stream of deltas, whatever the slot layout.  Plus: the state is left as it was, the upload accounting, the
errors.  Host codes are a permuted, non-contiguous set, so a host's index differs from its code.
"""
import ctypes as C
import os

import numpy as np
import pytest

from cook_b200 import abi, engine, traces
from cook_b200.engine import CookError, GpuEngine
from test_state_resident import DEFAULTS, _lists, jobs_soa, pool_rows, tasks_soa

RUN_KEYS = ("user", "priority", "start_time", "task_id", "job_id", "cpus", "mem", "gpus")


def test_state_rebalance_symbol_exported():
    if not os.path.exists(engine.LIB_PATH):
        pytest.skip("libcookgpu.so not built")
    assert hasattr(engine.load_library(), "cook_state_rebalance")


def remap_hosts(r, seed):
    """The gen_rebalance dict `r` with hostname codes 3 * perm + 7: the host table, novel-host lists and
    cotask hosts carry codes; running tasks keep their table index.  Returns the code of each index."""
    H = r["hosts"].n
    codes = (3 * np.random.default_rng(seed).permutation(H) + 7).astype(np.int32)
    h = r["hosts"]
    kw = {n: h.col(n) for n, _ in h._fields_ if h.col(n) is not None}
    kw.update(n=H, n_attr_cols=h.n_attr_cols, hostname_id=codes)
    r["hosts"] = abi.HostTable(**kw)
    j = r["pending"]
    if j.col("novel_off") is not None and j.col("novel_off")[-1] > 0:
        kw = {n: j.col(n) for n, _ in j._fields_ if j.col(n) is not None}
        kw.update(n=j.n, novel_host=codes[j.col("novel_host")])
        r["pending"] = abi.JobsSoA(**kw)
    g = r["groups"]
    if g is not None:
        kw = {n: g.col(n) for n, _ in g._fields_ if g.col(n) is not None}
        kw.update(n_groups=g.n_groups, cot_hostname_id=codes[g.col("cot_hostname_id")] if g.col("cot_off")[-1] else
                  g.col("cot_hostname_id"))
        r["groups"] = abi.Groups(**kw)
    return codes


def rows_of(r, codes):
    """The pool's pending jobs {job_id: row} and running tasks {task_id: row (with its hostname code)}."""
    j = r["pending"]
    nov, att, grp = _lists(j, "novel_off", "novel_host"), _lists(j, "attr_off", "attr_col", "attr_val"), \
        _lists(j, "group_off", "group_idx")
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


def rdelta(reset=False, up=(), rm=(), run_up=(), run_rm=(), with_hosts=True):
    up, run_up = list(up), list(run_up)
    pend, prio, jid = jobs_soa(up) if up else (None, None, None)
    hn = np.array([r["host"] for r in run_up], np.int32) if run_up and with_hosts else None
    return abi.make_delta(reset=reset, pending=pend, pending_priority=prio, pending_job_id=jid, pending_rm=list(rm),
                          running=tasks_soa(run_up) if run_up else None, running_rm=list(run_rm),
                          running_hostname_id=hn)


def decisions_eq(got, want):
    keys = ("job_id", "pending_idx", "host", "victims", "dru", "mem", "cpus", "gpus")
    assert [tuple(d[k] for k in keys) for d in got] == [tuple(d[k] for k in keys) for d in want]


class RPool:
    """A rebalance pool: the handle under test, a host-table handle, and the model."""

    def __init__(self, r, codes, dru_mode=0):
        self.r, self.codes = r, codes
        self.idx = {int(c): i for i, c in enumerate(codes)}
        self.users, self.hosts, self.groups, self.params = r["users"], r["hosts"], r["groups"], r["params"]
        self.gpu, self.ref = GpuEngine(pool_name="state", dru_mode=dru_mode), GpuEngine(pool_name="host")
        self.pend, self.run = {}, {}
        self.queue, self.gone = [], set()

    def close(self):
        self.gpu.close()
        self.ref.close()

    def apply(self, up=(), rm=(), run_up=(), run_rm=(), reset=False):
        up, run_up = list(up), list(run_up)
        self.gpu.state_apply(rdelta(reset, up, rm, run_up, run_rm))
        if reset:
            self.pend, self.run = {}, {}
            self.gone |= set(self.queue)
        for j in rm:
            del self.pend[j]
        for t in run_rm:
            del self.run[t]
        for j, row in up:
            self.pend[j] = row
        for row in run_up:
            self.run[row["task_id"]] = row
        self.gone |= set(rm) | {j for j, _ in up}

    def rank(self):
        self.queue, self.gone = self.gpu.state_rank(self.users).tolist(), set()
        return self.queue

    def taken(self):
        return [j for j in self.queue if j not in self.gone and self.pend[j]["allowed"]][:self.params.max_preemption]

    def tables(self):
        """cook_rebalance's host tables of the same rows, and the task id of each running index."""
        rows = [self.run[t] for t in sorted(self.run)]
        running = abi.RunningSoA(t=tasks_soa(rows), host=np.array([self.idx[r["host"]] for r in rows], np.int32))
        take = self.taken()
        jobs, prio, jid = jobs_soa([(j, self.pend[j]) for j in take])
        return running, jobs, jid, prio, np.array([r["task_id"] for r in rows], np.int64)

    def want(self, engine_):
        running, jobs, jid, prio, tids = self.tables()
        if jobs.n == 0:
            return []
        out = engine_.rebalance(running, jobs, jid, prio, self.hosts, self.users, self.params, groups=self.groups)
        R = len(tids)
        for d in out:
            d["job_id"] = int(jid[d["pending_idx"]])
            d["victims"] = [int(tids[v]) if v < R else -1 - (v - R) for v in d["victims"]]
        return out

    def check(self, oracle=None):
        got = self.gpu.state_rebalance(self.hosts, self.users, self.params, groups=self.groups)
        decisions_eq(got, self.want(self.ref))
        if oracle is not None:
            decisions_eq(got, self.want(oracle))
        return got


def _pool(seed, constraints, n_running=3000, n_pending=300, n_hosts=200, n_users=40, mp=24):
    r = traces.gen_rebalance(seed, n_running, n_pending, n_hosts, n_users, max_preemption=mp,
                             constraints=constraints)
    codes = remap_hosts(r, seed + 1)
    return r, codes


@pytest.mark.gpu
@pytest.mark.parametrize("constraints", [False, True])
def test_equivalence_over_deltas(constraints, oracle):
    r, codes = _pool(71 if constraints else 73, constraints)
    pend, run = rows_of(r, codes)
    p = RPool(r, codes)
    rng = np.random.default_rng(9)
    try:
        items = sorted(pend.items())
        reserve = items[-60:]
        p.apply(up=items[:-60], run_up=list(run.values()), reset=True)
        t_next = [10 ** 9]
        many_victims = removed_ahead = 0
        for cycle in range(5):
            p.rank()
            # after the rank: the first job the walk would take is killed, one more allowed flag flips (the
            # upsert replaces the job: it leaves the queue), one priority changes
            live = [j for j in p.queue if p.pend[j]["allowed"]]
            kill = [live[0]] + [int(j) for j in rng.choice(live[1:], 2, replace=False)]
            flip = [j for j in p.queue if j not in kill][5]
            prio = [j for j in p.queue if j not in kill and j != flip][7]
            ups = [(flip, dict(p.pend[flip], allowed=1 - p.pend[flip]["allowed"])),
                   (prio, dict(p.pend[prio], priority=int(rng.choice([10, 50, 90]))))]
            p.apply(up=ups, rm=kill)
            got = p.check(oracle if cycle % 2 == 0 else None)
            many_victims = max([many_victims] + [len(d["victims"]) for d in got])
            removed_ahead += len(got) > 0
            # churn: the victims die, some tasks finish, some jobs start on random hosts, new jobs arrive,
            # some jobs are disallowed or change priority before the next rank
            dead = {v for d in got for v in d["victims"] if v >= 0 and v in p.run}
            fin = [t for t in p.run if t not in dead and rng.random() < 0.03]
            starts = [j for j in p.pend if rng.random() < 0.05]
            run_up = []
            for j in starts:
                t_next[0] += 1
                row = p.pend[j]
                run_up.append(dict(user=row["user"], priority=row["priority"], start_time=1_700_000_000_000 + t_next[0],
                                   task_id=t_next[0], job_id=j, cpus=row["cpus"], mem=row["mem"], gpus=0.0,
                                   host=int(codes[rng.integers(len(codes))])))
            up = [reserve.pop() for _ in range(min(10, len(reserve)))]
            for j in [j for j in p.pend if j not in starts][:: 17]:
                up.append((j, dict(p.pend[j], allowed=int(rng.random() < 0.7), priority=int(rng.choice([10, 50, 90])))))
            p.apply(up=up, rm=starts, run_up=run_up, run_rm=sorted(dead) + fin)
            if cycle == 2:                           # new leadership
                p.apply(up=sorted(p.pend.items()), run_up=list(p.run.values()), reset=True)
        assert many_victims >= 2, "no decision with several victims"
        assert removed_ahead >= 1, "no cycle decided after the queue's first allowed job was removed"
    finally:
        p.close()


@pytest.mark.gpu
def test_layout_independence():
    r, codes = _pool(81, True)
    pend, run = rows_of(r, codes)
    for k, t in enumerate(sorted(run)):              # off the binary grid: the serial folds run
        if k % 3 == 0:
            run[t]["cpus"] += 0.1
    for k, j in enumerate(sorted(pend)):
        if k % 4 == 0:
            pend[j]["cpus"] += 0.1
    items = sorted(pend.items())
    a, b = RPool(r, codes), RPool(r, codes)
    rng = np.random.default_rng(4)
    try:
        a.apply(up=items, run_up=[run[t] for t in sorted(run)])
        junk = [(10 ** 11 + i, items[i][1]) for i in range(200)]
        jrun = [dict(row, task_id=10 ** 12 + i) for i, row in enumerate(list(run.values())[:500])]
        b.apply(up=junk, run_up=jrun)                # slots the real rows then reuse
        b.apply(rm=[j for j, _ in junk], run_rm=[row["task_id"] for row in jrun])
        perm = rng.permutation(len(items))
        rr = list(run.values())
        b.apply(up=[items[i] for i in perm[: len(perm) // 2]], run_up=[rr[i] for i in rng.permutation(len(rr))])
        b.apply(up=[items[i] for i in perm[len(perm) // 2:]])
        assert a.rank() == b.rank()
        ga, gb = a.check(), b.check()
        assert len(ga) > 0
        decisions_eq(ga, gb)
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_stated_size_c4_pool3():
    r = traces.gen_config_pool("c4", 3)["rebalance"]
    assert (r["running"].col("t").n, r["params"].max_preemption) == (40_000, 128)
    codes = remap_hosts(r, 5)
    pend, run = rows_of(r, codes)
    p = RPool(r, codes)
    try:
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.rank()
        got = p.check()
        assert len(got) > 0
    finally:
        p.close()


def _c3_with_hosts(seed):
    """A config-#3-like pool with offers, its running tasks on the offers' hosts, and the host table."""
    t = traces.gen_c3_pool(seed, n_jobs=2500, n_offers=160, n_users=24, n_running=500)
    o = t["offers"]
    hn = o.col("hostname_id")
    hosts = abi.HostTable(n=o.n, hostname_id=hn, name_rank=o.col("name_rank"), has_spare=np.zeros(o.n, np.uint8),
                          spare_cpus=np.zeros(o.n), spare_mem=np.zeros(o.n), spare_gpus=np.zeros(o.n),
                          n_attr_cols=o.n_attr_cols, attr=o.col("attr"))
    pend, run = pool_rows(t)
    rng = np.random.default_rng(seed)
    for row in run.values():
        row["host"] = int(hn[rng.integers(o.n)])
    return t, hosts, pend, run


@pytest.mark.gpu
def test_state_untouched():
    t, hosts, pend, run = _c3_with_hosts(91)
    prm = abi.RebalanceParams(32, 0.0, 0.0, 0)
    params = traces.match_params(1000)
    mp = int(t["jobs"].col("ports").max()) if t["jobs"].col("ports") is not None else 0
    a, b = GpuEngine(pool_name="a"), GpuEngine(pool_name="b")
    try:
        d = rdelta(up=sorted(pend.items()), run_up=list(run.values()))
        for e in (a, b):
            e.state_apply(d)
        qa, qb = a.state_rank(t["users"]), b.state_rank(t["users"])
        assert np.array_equal(qa, qb)
        a.state_rebalance(hosts, t["users"], prm, groups=t["groups"])
        ma = a.state_match(t["offers"], t["users"], params, groups=t["groups"], max_ports=mp)
        mb = b.state_match(t["offers"], t["users"], params, groups=t["groups"], max_ports=mp)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
        assert np.array_equal(a.state_rank(t["users"]), qa)
    finally:
        a.close()
        b.close()


def _nb(*arrays):
    return sum(a.nbytes for a in arrays if isinstance(a, np.ndarray))


@pytest.mark.gpu
def test_accounting():
    r, codes = _pool(101, True, n_running=2000, n_pending=200, n_hosts=150, n_users=30, mp=16)
    pend, run = rows_of(r, codes)
    h, u, g = r["hosts"], r["users"], r["groups"]
    want = _nb(*[h.col(n) for n, _ in h._fields_])
    want += _nb(*[u.col(n) for n in ("name_rank", "div_mem", "div_cpus", "quota_count", "quota_cpus", "quota_mem",
                                      "quota_gpus")])
    want += _nb(*[g.col(n) for n, _ in g._fields_])
    got = []
    for scale in (1, 2):                             # the same rows, and as many again under new ids
        p = RPool(r, codes)
        try:
            up = sorted(pend.items())
            rr = list(run.values())
            if scale == 2:
                up += [(j + 10 ** 10, row) for j, row in up]
                rr += [dict(row, task_id=row["task_id"] + 10 ** 10) for row in rr]
            p.apply(up=up, run_up=rr)
            p.rank()
            p.check()
            st = p.gpu.last_stats(abi.PHASE_REBALANCE)
            assert st["n_launches"] > 0
            got.append(st["h2d_bytes"])
        finally:
            p.close()
    assert got == [want, want]


@pytest.mark.gpu
def test_errors():
    r, codes = _pool(111, True, mp=16)
    pend, run = rows_of(r, codes)
    items = sorted(pend.items())
    p = RPool(r, codes)
    try:
        p.apply(up=items, run_up=list(run.values()))

        def code_of(fn):
            with pytest.raises(CookError) as e:
                fn()
            return e.value.code

        reb = lambda hosts=p.hosts, groups=p.groups: p.gpu.state_rebalance(hosts, p.users, p.params, groups=groups)
        assert code_of(reb) == abi.COOK_E_BADARG                 # no rank yet
        q0 = p.rank()
        r0 = reb()
        assert len(r0) > 0

        def fails(fn, code=abi.COOK_E_BADARG, undo=None):
            assert code_of(fn) == code
            if undo:
                undo()
            assert reb() == r0
            assert p.rank() == q0
            assert reb() == r0

        R, MP = len(p.run), p.params.max_preemption

        def raw(cap, dec=True):
            out = (abi.Decision * MP)()
            jid, vict, n = np.zeros(MP, np.int64), np.zeros(max(cap, 1), np.int64), C.c_int32(0)
            rc = p.gpu.lib.cook_state_rebalance(p.gpu.pool, C.byref(p.hosts), C.byref(p.groups), C.byref(p.users),
                                                C.byref(p.params), out if dec else None, abi.ptr(jid, abi.P_I64),
                                                abi.ptr(vict, abi.P_I64), int(cap), C.byref(n))
            if rc != 0:
                p.gpu._err(rc)

        fails(lambda: raw(R + MP, dec=False))                      # a null required argument
        fails(lambda: raw(R + MP - 1))                             # victim_cap below the bound
        raw(R + MP)
        task = dict(next(iter(p.run.values())), task_id=10 ** 13)
        p.gpu.state_apply(rdelta(run_up=[task], with_hosts=False))  # host unknown (-1)
        fails(reb, undo=lambda: p.gpu.state_apply(rdelta(run_rm=[10 ** 13])))
        p.gpu.state_apply(rdelta(run_up=[dict(task, host=int(codes.max()) + 1)]))   # a code not in the table
        fails(reb, undo=lambda: p.gpu.state_apply(rdelta(run_rm=[10 ** 13])))
        hn = p.hosts.col("hostname_id").copy()
        hn[1] = hn[0]
        kw = {n: p.hosts.col(n) for n, _ in p.hosts._fields_ if p.hosts.col(n) is not None}
        kw.update(n=p.hosts.n, n_attr_cols=p.hosts.n_attr_cols, hostname_id=hn)
        fails(lambda: reb(hosts=abi.HostTable(**kw)))             # a hostname code twice
        bad_rows = [dict(items[0][1], user=p.users.n_users),       # user, group, attribute column out of range
                    dict(items[0][1], groups=[p.groups.n_groups]),
                    dict(items[0][1], attr=[(p.hosts.n_attr_cols, 1)])]
        for row in bad_rows:
            p.gpu.state_apply(rdelta(up=[(10 ** 13, row)]))
            fails(reb, undo=lambda: p.gpu.state_apply(rdelta(rm=[10 ** 13])))
        g = GpuEngine(pool_name="gpu-dru", dru_mode=1)              # GPU DRU mode
        try:
            with pytest.raises(CookError) as e:
                g.state_rebalance(p.hosts, p.users, p.params)
            assert e.value.code == abi.COOK_E_UNSUPPORTED_CONSTRAINT
        finally:
            g.close()
    finally:
        p.close()
