"""cook_state_launch and cook_state_patch: launches and match-time column changes by job id on the resident state.

Handle A launches through cook_state_launch and patches through cook_state_patch.  Its twin B receives the same
changes as cook_state_apply deltas.  A model keeps the rows; rank and match must equal cook_rank / cook_match on host
tables built from it (and rank the oracle).  A launch must leave exactly the state the equivalent delta leaves; a
patch must keep the job in the ranked queue where an upsert drops it.  Plus the match's column-presence switch, slot
layout, the rebalancer's view of launched tasks, upload accounting and the all-or-nothing errors.
"""
import ctypes as C
import os

import numpy as np
import pytest

from cook_b200 import abi, engine, traces
from cook_b200.engine import CookError, GpuEngine
from test_state_rebalance import RPool, _pool, decisions_eq, rdelta, rows_of
from test_state_resident import Model, _c2, _c3, _churn, pool_rows

START = 1_700_000_000_000


def test_launch_patch_symbols_exported():
    if not os.path.exists(engine.LIB_PATH):
        pytest.skip("libcookgpu.so not built")
    lib = engine.load_library()
    for name in ("cook_state_launch", "cook_state_patch"):
        assert hasattr(lib, name), name
    assert callable(GpuEngine.state_launch) and callable(GpuEngine.state_patch)


def hosts_of(offers):
    """A host table over the offers' hosts (no spare resources): the rebalancer's view of the same cluster."""
    o = offers
    return abi.HostTable(n=o.n, hostname_id=o.col("hostname_id"), name_rank=o.col("name_rank"),
                         has_spare=np.zeros(o.n, np.uint8), spare_cpus=np.zeros(o.n), spare_mem=np.zeros(o.n),
                         spare_gpus=np.zeros(o.n), n_attr_cols=o.n_attr_cols, attr=o.col("attr"))


def with_reserved(offers, idx):
    """The offers with `reserved` set on the offer indices idx."""
    kw = {n: offers.col(n) for n, _ in offers._fields_ if offers.col(n) is not None}
    res = np.zeros(offers.n, np.uint8)
    res[list(idx)] = 1
    kw.update(n=offers.n, n_attr_cols=offers.n_attr_cols, reserved=res)
    return abi.OffersSoA(**kw)


def task_of(row, job_id, task_id, start, host):
    return dict(user=row["user"], priority=row["priority"], start_time=int(start), task_id=int(task_id),
                job_id=int(job_id), cpus=row["cpus"], mem=row["mem"], gpus=row["gpus"], host=int(host))


class Twin:
    """A (launches and patches by id), B (the same as deltas), the host-table handle and the model."""

    def __init__(self, t, groups=None):
        self.t, self.users, self.offers, self.groups = t, t["users"], t["offers"], groups
        self.hosts = hosts_of(t["offers"])
        self.params = traces.match_params(min(1000, t["jobs"].n), host_lifetime_mins=t.get("host_lifetime_mins", 0))
        self.rparams = abi.RebalanceParams(32, 0.0, 0.0, 0)
        self.max_ports = int(t["jobs"].col("ports").max()) if t["jobs"].col("ports") is not None else 0
        self.a, self.b, self.ref = GpuEngine(pool_name="launch"), GpuEngine(pool_name="delta"), GpuEngine(pool_name="host")
        self.m = Model()
        self.queue, self.gone = [], {"a": set(), "b": set()}

    def close(self):
        for e in (self.a, self.b, self.ref):
            e.close()

    def apply(self, up=(), rm=(), run_up=(), run_rm=(), reset=False):
        up, run_up = list(up), list(run_up)
        for e in (self.a, self.b):
            e.state_apply(rdelta(reset, up, rm, run_up, run_rm))
        self.m.apply(up, rm, run_up, run_rm, reset)
        for g in self.gone.values():
            g |= set(rm) | {j for j, _ in up} | (set(self.queue) if reset else set())

    def launch(self, jobs, tids, starts, hosts=None):
        """A: cook_state_launch; B: the batch pending_rm = jobs plus the running upserts built from the rows."""
        tasks = [task_of(self.m.pend[j], j, t, s, -1 if hosts is None else h)
                 for j, t, s, h in zip(jobs, tids, starts, hosts if hosts is not None else [None] * len(jobs))]
        self.a.state_launch(jobs, tids, starts, hosts)
        self.b.state_apply(rdelta(rm=jobs, run_up=tasks, with_hosts=hosts is not None))
        self.m.apply(d_rm=jobs, r_up=tasks)
        for g in self.gone.values():
            g |= set(jobs)
        return tasks

    def patch(self, jobs, allowed=None, plugin_accept=None, reserved_host=None, clear=False, upsert_b=True):
        """A: cook_state_patch.  B (upsert_b): the same columns as pending upserts, which drop the jobs from the
        queue; else B is patched too."""
        if clear:
            for r in self.m.pend.values():
                r["reserved_host"] = -1
        cols = {"allowed": allowed, "plugin_accept": plugin_accept, "reserved_host": reserved_host}
        for k, j in enumerate(jobs):
            self.m.pend[j] = dict(self.m.pend[j], **{c: int(v[k]) for c, v in cols.items() if v is not None})
        self.a.state_patch(jobs, allowed, plugin_accept, reserved_host, clear)
        if upsert_b:
            if clear:
                self.b.state_patch([], clear_reservations=True)
            self.b.state_apply(rdelta(up=[(j, self.m.pend[j]) for j in jobs]))
            self.gone["b"] |= set(jobs)
        else:
            self.b.state_patch(jobs, allowed, plugin_accept, reserved_host, clear)

    def rank(self, oracle=None):
        qa, qb = self.a.state_rank(self.users), self.b.state_rank(self.users)
        assert np.array_equal(qa, qb), "launch handle and delta twin rank differently"
        running, pending, _, jid = self.m.tables()
        host = self.ref.rank(running if running.n else None, pending, self.users)
        assert np.array_equal(qa, jid[host["ranked"]]), "resident rank != cook_rank on the same rows"
        if oracle is not None and pending.n:
            o = oracle.rank(running if running.n else None, pending, self.users)
            assert np.array_equal(qa, jid[o["ranked"]]), "resident rank != oracle"
        self.queue, self.gone = qa.tolist(), {"a": set(), "b": set()}
        return qa

    def _match_one(self, e, gone, offers):
        got = e.state_match(offers, self.users, self.params, groups=self.groups, max_ports=self.max_ports)
        _, _, jobs, jid = self.m.tables()
        pos = {j: i for i, j in enumerate(jid.tolist())}
        ranked = np.array([pos[j] for j in self.queue if j not in gone], np.int32)
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

    def match(self, offers=None, same=True):
        """Both handles against the host-table path on the model; `same`: A and B must also agree."""
        offers = offers if offers is not None else self.offers
        ga = self._match_one(self.a, self.gone["a"], offers)
        gb = self._match_one(self.b, self.gone["b"], offers)
        if same:
            for k in ("considerable", "assign", "ports", "fail"):
                assert np.array_equal(ga[k], gb[k]), k
        return ga, gb

    def rebalance(self):
        ra = self.a.state_rebalance(self.hosts, self.users, self.rparams, groups=self.groups)
        rb = self.b.state_rebalance(self.hosts, self.users, self.rparams, groups=self.groups)
        decisions_eq(ra, rb)
        return ra


def _load(t, frac=0.85, seed=1):
    """The trace's rows, each running task on a random host of the offers; loads `frac` of the jobs."""
    pend, run = pool_rows(t)
    hn = t["offers"].col("hostname_id")
    rng = np.random.default_rng(seed)
    for r in run.values():
        r["host"] = int(hn[rng.integers(len(hn))])
    items = sorted(pend.items())
    cut = int(len(items) * frac)
    return items[:cut], items[cut:], list(run.values())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["c2", "c3"])
def test_launch_equivalence(kind, oracle):
    t = _c2(11) if kind == "c2" else _c3(13)
    p = Twin(t, t.get("groups"))
    try:
        first, reserve, run = _load(t)
        p.apply(up=first, run_up=run, reset=True)
        rng = np.random.default_rng(5)
        hn = t["offers"].col("hostname_id")
        t_next = [10 ** 9]
        n_launched = 0
        for cycle in range(6):
            p.rank(oracle if cycle % 2 == 0 else None)
            p.rebalance()
            for rnd in range(2):                     # two match rounds per rank
                ga, _ = p.match()
                placed = [(int(j), int(a)) for j, a in zip(ga["considerable"], ga["assign"]) if a >= 0][:60]
                launched = [j for j, _ in placed]
                up, rm, run_up, run_rm = _churn(p, rng, reserve, t_next, launched)
                # _churn's launches: the first len(launched) removals and every running upsert
                assert rm[:len(launched)] == launched and len(run_up) == len(launched)
                p.launch(launched, [r["task_id"] for r in run_up], [r["start_time"] for r in run_up],
                         [int(hn[a]) for _, a in placed])
                n_launched += len(launched)
                p.apply(up, rm[len(launched):], (), run_rm)
                p.rebalance()
            if cycle == 3:                            # new leadership
                p.apply(up=sorted(p.m.pend.items()), run_up=list(p.m.run.values()), reset=True)
        p.rank(oracle)
        p.match()
        p.rebalance()
        assert n_launched > 100
    finally:
        p.close()


@pytest.mark.gpu
def test_patch_keeps_queue():
    t = _c3(17)
    p = Twin(t, t["groups"])
    try:
        first, _, run = _load(t, frac=1.0)
        p.apply(up=first, run_up=run)
        q = p.rank().tolist()
        hn = t["offers"].col("hostname_id")
        rng = np.random.default_rng(2)
        no_allow, no_plugin, resv, all3 = q[3:13], q[20:30], q[40:50], q[60:66]
        p.patch(no_allow, allowed=np.zeros(len(no_allow), np.uint8))
        p.patch(no_plugin, plugin_accept=np.zeros(len(no_plugin), np.uint8))
        p.patch(resv, reserved_host=hn[rng.integers(len(hn), size=len(resv))])
        p.patch(all3, allowed=np.array([1, 0, 1, 0, 1, 1], np.uint8), plugin_accept=np.array([0, 1, 1, 0, 1, 1], np.uint8),
                reserved_host=np.array([-1, int(hn[0]), -1, int(hn[1]), int(hn[2]), -1], np.int32))
        # A keeps every patched job in its queue; B (upserts) drops them: both equal the host-table path
        ga, gb = p.match(same=False)
        kept = set(resv) | {all3[0], all3[2], all3[4], all3[5]}
        assert kept & set(ga["considerable"].tolist()), "no patched job was considered"
        assert not (set(no_allow + no_plugin + resv + all3) & set(gb["considerable"].tolist()))
        # a reservation made between rank and match on the host the job fits best: reserve the host of the
        # first placement of an unreserved match for its job and mark that offer reserved
        p.rank()
        ga, _ = p.match()
        k = int(np.flatnonzero(ga["assign"] >= 0)[0])
        j, o = int(ga["considerable"][k]), int(ga["assign"][k])
        others = [int(x) for x, a in zip(ga["considerable"], ga["assign"]) if a == o and int(x) != j]
        p.patch([j], reserved_host=np.array([hn[o]], np.int32), upsert_b=False)
        ga, _ = p.match(offers=with_reserved(t["offers"], [o]))
        assign = dict(zip(ga["considerable"].tolist(), ga["assign"].tolist()))
        assert assign[j] == o, "the reserved job lost its host"
        assert [x for x, a in assign.items() if a == o] == [j], "another job was placed on a reserved host"
        assert others, "the host held other jobs before the reservation: pick a pool where it does"
    finally:
        p.close()


@pytest.mark.gpu
def test_reservation_map_replacement():
    t = _c3(19)
    p = Twin(t, t["groups"])
    try:
        first, _, run = _load(t, frac=1.0)
        p.apply(up=first, run_up=run)
        q = p.rank().tolist()
        hn = t["offers"].col("hostname_id")
        set1, set2 = q[0:40:2], q[1:41:2]
        h1, h2 = hn[np.arange(20)], hn[np.arange(20, 40)]
        p.patch(set1, reserved_host=h1, clear=True, upsert_b=False)
        n1 = sum(r["reserved_host"] != -1 for r in p.m.pend.values())
        p.patch(set2, reserved_host=h2, clear=True, upsert_b=False)
        st = p.a.last_stats(abi.PHASE_STATE)
        assert st["h2d_bytes"] == 4 * n1 + len(set2) * (4 + 4)
        assert all(p.m.pend[j]["reserved_host"] == -1 for j in set1)
        # every host of both sets is reserved: set 1's hosts now take no job at all, set 2's only their own
        ga, _ = p.match(offers=with_reserved(t["offers"], range(40)))
        for j, a in zip(ga["considerable"].tolist(), ga["assign"].tolist()):
            assert a < 0 or a >= 40 or (20 <= a < 40 and p.m.pend[j]["reserved_host"] == hn[a]), (j, a)
        # the second set's jobs without reservation again: a clear with an empty batch
        p.patch([], clear=True, upsert_b=False)
        assert p.a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 4 * len(set2)
        p.match()
    finally:
        p.close()


@pytest.mark.gpu
def test_presence_switch():
    t = _c2(23)                                       # no job holds a reservation, a disallow or a plugin veto
    p = Twin(t)
    try:
        first, _, run = _load(t, frac=1.0)
        p.apply(up=first, run_up=run)
        q = p.rank().tolist()
        ga, _ = p.match()
        k = int(np.flatnonzero(ga["assign"] >= 0)[0])  # the first placement: its host is the job's best fit
        j, o = int(ga["considerable"][k]), int(ga["assign"][k])
        offers = with_reserved(t["offers"], [o])
        hn = int(t["offers"].col("hostname_id")[o])
        # reserved_host: the first reservation switches the constraint path on, clearing the last one off
        p.match(offers=offers)
        p.patch([j], reserved_host=np.array([hn], np.int32), upsert_b=False)
        ga, _ = p.match(offers=offers)
        assert dict(zip(ga["considerable"].tolist(), ga["assign"].tolist()))[j] == o
        p.patch([j], reserved_host=np.array([-1], np.int32), upsert_b=False)
        p.match(offers=offers)
        p.patch([j], reserved_host=np.array([hn], np.int32), upsert_b=False)
        p.patch([], clear=True, upsert_b=False)       # and by a clear
        p.match(offers=offers)
        # allowed and plugin_accept likewise
        for col in ("allowed", "plugin_accept"):
            p.patch(q[:3], **{col: np.zeros(3, np.uint8)}, upsert_b=False)
            ga, _ = p.match()
            assert not (set(q[:3]) & set(ga["considerable"][ga["assign"] >= 0].tolist()))
            p.patch(q[:3], **{col: np.ones(3, np.uint8)}, upsert_b=False)
            p.match()
    finally:
        p.close()


@pytest.mark.gpu
def test_launch_layout():
    t = _c3(29)
    p = Twin(t, t["groups"])
    try:
        first, reserve, run = _load(t, frac=0.6)
        hn = t["offers"].col("hostname_id")
        run = run + [dict(r, task_id=3 * 10 ** 10 + k) for k, r in enumerate(run)]
        run = run[:1000]                              # the running table holds 1000 of 1024 slots
        p.apply(up=first, run_up=run)
        p.rank()
        p.match()
        # 400 new jobs with long novel-host lists: the list arena is mostly theirs
        long_rows = [(10 ** 11 + k, dict(r, novel=hn[(np.arange(60) * 7 + k) % len(hn)].tolist()))
                     for k, (_, r) in enumerate(reserve[:400])]
        p.apply(up=long_rows)
        p.rank()
        p.match()
        # launching 300 of them frees most of the arena (a compaction) and grows the running table past 1024
        jobs = [j for j, _ in long_rows[:300]]
        tids = [5 * 10 ** 9 + 3 * k for k in range(300)]
        p.launch(jobs, tids, [START + k for k in range(300)], [int(hn[k % len(hn)]) for k in range(300)])
        st = p.a.last_stats(abi.PHASE_STATE)
        assert st["n_launches"] > 2, "the launch compacted no list arena"
        p.match()
        p.rank()
        p.match()
        p.rebalance()
        # submissions reuse the pending slots the launches freed
        p.apply(up=reserve[400:700])
        small = [j for j, _ in first[:50]]
        p.launch(small, [6 * 10 ** 9 + k for k in range(50)], [START] * 50)
        p.apply(up=[(10 ** 11 + 1000 + k, r) for k, (_, r) in enumerate(first[:50])])
        p.rank()
        p.match()
    finally:
        p.close()


class LRPool(RPool):
    """RPool plus launches by job id."""

    def launch(self, jobs, tids, starts, hosts=None):
        self.gpu.state_launch(jobs, tids, starts, hosts)
        for k, j in enumerate(jobs):
            row = self.pend.pop(j)
            self.run[tids[k]] = task_of(row, j, tids[k], starts[k], -1 if hosts is None else hosts[k])
        self.gone |= set(jobs)


@pytest.mark.gpu
def test_rebalance_after_launch(oracle):
    r, codes = _pool(121, True)
    pend, run = rows_of(r, codes)
    p = LRPool(r, codes)
    try:
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.rank()
        before = p.check()
        # new jobs of the victims' user start on the hosts the walk preempts on, later than all its tasks: the
        # walk should now take some of them
        u = min(p.run[v]["user"] for d in before for v in d["victims"] if v >= 0)
        jobs = [8 * 10 ** 9 + k for k in range(20)]
        p.apply(up=[(j, dict(next(iter(pend.values())), user=u)) for j in jobs])
        tids = [9 * 10 ** 9 + k for k in range(len(jobs))]
        hosts = [int(codes[before[k % len(before)]["host"]]) for k in range(len(jobs))]
        p.launch(jobs, tids, [START + 10 ** 6 + k for k in range(len(jobs))], hosts)
        p.rank()
        got = p.check(oracle)
        victims = {v for d in got for v in d["victims"]}
        assert victims & set(tids), "no launched task was chosen as a victim"
        # a launch with no host leaves a running row the rebalancer cannot place
        j = next(j for j in p.queue if j in p.pend)
        p.launch([j], [9 * 10 ** 9 + 999], [START])
        p.rank()
        with pytest.raises(CookError) as e:
            p.gpu.state_rebalance(p.hosts, p.users, p.params, groups=p.groups)
        assert e.value.code == abi.COOK_E_BADARG
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [7, 300])
def test_accounting(n):
    t = _c2(31)
    p = Twin(t)
    try:
        first, reserve, run = _load(t, frac=0.7)
        p.apply(up=first, run_up=run)
        hn = t["offers"].col("hostname_id")
        jobs = [j for j, _ in first[:2 * n]]
        for k, (js, hosts) in enumerate(((jobs[:n], [int(hn[i % len(hn)]) for i in range(n)]), (jobs[n:], None))):
            tids = [7 * 10 ** 9 + 10 * k * n + i for i in range(n)]
            p.launch(js, tids, [START + i for i in range(n)], hosts)
            a, b = p.a.last_stats(abi.PHASE_STATE), p.b.last_stats(abi.PHASE_STATE)
            assert a["h2d_bytes"] == n * (4 + 4 + 8 + 8) + (4 * n if hosts else 0)
            # the delta: the task rows (8 columns, 56 B), a slot per removal and per upsert
            assert b["h2d_bytes"] == n * (56 + 4 + 4) + (4 * n if hosts else 0)
            assert a["h2d_bytes"] < b["h2d_bytes"]
        rest = [j for j, _ in first[2 * n:3 * n]]
        z8, z32 = np.zeros(n, np.uint8), np.full(n, -1, np.int32)
        codes = hn[np.arange(n) % len(hn)].astype(np.int32)
        for cols, size in (({"allowed": z8}, 5), ({"plugin_accept": z8, "reserved_host": z32}, 9),
                           ({"allowed": z8, "plugin_accept": z8, "reserved_host": codes}, 10), ({}, 0)):
            p.patch(rest, upsert_b=False, **cols)
            assert p.a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == n * size
        p.patch([], clear=True, upsert_b=False)        # n reservations from the third patch
        assert p.a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 4 * n
        p.rank()
        p.match()
    finally:
        p.close()


@pytest.mark.gpu
def test_errors():
    t = _c3(37)
    p = Twin(t, t["groups"])
    try:
        first, _, run = _load(t, frac=1.0)
        p.apply(up=first, run_up=run)
        p.rank()
        ids = [j for j, _ in first]
        live_tid = next(iter(p.m.run))
        gone = ids[0]
        p.launch([gone], [10 ** 10], [START], [int(t["offers"].col("hostname_id")[0])])   # no longer pending
        p.rank()
        p.match()

        def fails(fn):
            with pytest.raises(CookError) as e:
                fn()
            assert e.value.code == abi.COOK_E_BADARG
            p.rank()
            p.match()
            p.rebalance()

        def raw_launch(n, jid, tid, st, hn=None):
            arr = [np.ascontiguousarray(x, np.int64) if x is not None else None for x in (jid, tid, st)]
            h = np.ascontiguousarray(hn, np.int32) if hn is not None else None
            rc = p.a.lib.cook_state_launch(p.a.pool, int(n), *[abi.ptr(x, abi.P_I64) if x is not None else None for x in arr],
                                           abi.ptr(h, abi.P_I32) if h is not None else None)
            if rc != 0:
                p.a._err(rc)

        def raw_patch(n, jid, rh=None):
            j = np.ascontiguousarray(jid, np.int64) if jid is not None else None
            h = np.ascontiguousarray(rh, np.int32) if rh is not None else None
            rc = p.a.lib.cook_state_patch(p.a.pool, int(n), abi.ptr(j, abi.P_I64) if j is not None else None, None,
                                          None, abi.ptr(h, abi.P_I32) if h is not None else None, 0)
            if rc != 0:
                p.a._err(rc)

        j1, j2 = ids[1], ids[2]
        fails(lambda: raw_launch(-1, [j1], [1], [1]))                                  # n < 0
        fails(lambda: raw_launch(1, None, [1], [1]))                                   # null required columns
        fails(lambda: raw_launch(1, [j1], None, [1]))
        fails(lambda: raw_launch(1, [j1], [1], None))
        fails(lambda: p.a.state_launch([j1, 10 ** 13], [1, 2], [1, 1]))               # unknown job id
        fails(lambda: p.a.state_launch([j1, gone], [1, 2], [1, 1]))                   # not live
        fails(lambda: p.a.state_launch([j1, j1], [1, 2], [1, 1]))                     # job id twice
        fails(lambda: p.a.state_launch([j1, j2], [3, 3], [1, 1]))                     # task id twice
        fails(lambda: p.a.state_launch([j1, j2], [3, live_tid], [1, 1]))              # task id already live
        fails(lambda: p.a.state_launch([j1, j2], [3, 4], [1, 1], [0, -2]))            # hostname code below -1
        fails(lambda: raw_patch(-1, [j1]))                                             # n < 0
        fails(lambda: raw_patch(1, None))                                              # null job_id
        fails(lambda: p.a.state_patch([j1, 10 ** 13], allowed=[0, 0]))               # unknown job id
        fails(lambda: p.a.state_patch([j1, gone], allowed=[0, 0]))                    # not live
        fails(lambda: p.a.state_patch([j1, j1], allowed=[0, 0]))                      # job id twice
        fails(lambda: raw_patch(2, [j1, j2], [3, -2]))                                 # reserved_host below -1
        fails(lambda: p.a.state_patch([j1, j2], reserved_host=[3, -2], clear_reservations=True))
    finally:
        p.close()
