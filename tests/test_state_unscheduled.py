"""-m gpu: cook_state_unscheduled against unscheduled_ref over a host mirror, bit for bit.

The golden scenarios (the reference's unscheduled tests and the hand-computed edges) replay on resident handles, and
cycle.unscheduled_reasons turns the device's answers into the reference's reasons.  A churn of launches, finishes,
extra instances, kills and priority upserts, with a Zipf user past one 2048-wide sort tile, on and off the grid, checks
every query of a sample after every batch.  A twin handle shows the call changes nothing a match reads; Investigations
records a placement failure through cook_state_match_offers; BADARGs leave the digest unchanged; each call's transfers
follow the header's formula.
"""
import json
import os
import struct

import numpy as np
import pytest

import resident_model as M
import unscheduled_ref as U
from cook_b200 import abi, cycle, engine, traces
from cook_b200.engine import CookError

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "unscheduled_golden.json")))
DROP = M.drop_all_but("gpus", "plugin_accept")


def bits(x):
    return struct.unpack("<q", struct.pack("<d", float(x)))[0]


class Mirror:
    """A resident handle and its rows: pending {job id: row}, running {task id: row}."""

    def __init__(self, name="unscheduled"):
        self.e = engine.GpuEngine(pool_name=name)
        self.pend, self.run = {}, {}

    def close(self):
        self.e.close()

    def apply(self, up=(), rm=(), run_up=(), run_rm=()):
        up, run_up = list(up), list(run_up)
        self.e.state_apply(M.delta(up=[(r["job_id"], r) for r in up], rm=rm, run_up=run_up, run_rm=run_rm, drop=DROP))
        for j in rm:
            del self.pend[j]
        for t in run_rm:
            del self.run[t]
        self.pend.update((r["job_id"], r) for r in up)
        self.run.update((r["task_id"], r) for r in run_up)

    def launch(self, jobs, tids, starts):
        self.e.state_launch(jobs, tids, starts)
        for j, t, s in zip(jobs, tids, starts):
            r = self.pend.pop(j)
            self.run[t] = dict(task_id=t, job_id=j, user=r["user"], priority=r["priority"], start_time=s,
                               cpus=r["cpus"], mem=r["mem"], gpus=r["gpus"])

    def check(self, queries):
        """The call against the restatement, bit for bit, and its transfer formula."""
        got = self.e.state_unscheduled(queries)
        want = U.answer(self.pend, self.run, queries)
        for i, (st, usage, pos, ahead, pl) in enumerate(want):
            assert int(got["status"][i]) == st, (i, queries[i])
            assert [bits(x) for x in got["usage"][i]] == [bits(x) for x in usage], (i, queries[i])
            assert int(got["position"][i]) == pos and got["ahead"][i] == ahead, (i, queries[i])
            assert int(got["plugin_deferred"][i]) == pl
            assert not got["ahead_raw"][i, len(ahead):].any()
        users = {self.user_of(q) for q in queries} - {None}
        s = got["stats"]
        if users:
            assert s["h2d_bytes"] == 4 * len(users) + 4 * len(queries)
            assert s["d2h_bytes"] == 121 * len(queries)
        else:
            assert s["h2d_bytes"] == s["d2h_bytes"] == s["n_launches"] == 0
        return got

    def user_of(self, j):
        if j in self.pend:
            return self.pend[j]["user"]
        rows = [r for r in self.run.values() if r["job_id"] == j]
        return max(rows, key=lambda r: r["task_id"])["user"] if rows else None


def digest(e):
    return {k: v for k, v in e.state_digest().items() if "buckets" not in k}


def pend_row(r):
    return dict(M.DEFAULTS, **r)


def loaded(sc, name):
    m = Mirror(name)
    m.apply(up=[pend_row(r) for r in sc["pending"]], run_up=sc["running"])
    return m


# ---- the golden scenarios on resident handles ---------------------------------------------------------------------
def test_golden_reasons():
    sc = GOLDEN["reasons"]
    m = loaded(sc, "golden-reasons")
    try:
        assert m.e.state_unscheduled([sc["uncommitted"]])["status"][0] == abi.UNSCHED_ABSENT
        for check in sc["checks"]:
            q = 1 if check.get("state") == "running" else sc["job"]
            a = m.check([q])
            kw = dict(sc["facts"], enforcing_rate_limit=check.get("enforcing_rate_limit", False),
                      num_rate_limited=check.get("num_rate_limited", 0))
            assert cycle.unscheduled_reasons(a, 0, **kw) == check["want"]
    finally:
        m.close()


def test_golden_queue_position():
    sc = GOLDEN["queue_position"]
    m = loaded(sc, "golden-queue")
    try:
        a = m.check([c["job"] for c in sc["cases"]])
        for i, c in enumerate(sc["cases"]):
            assert a["position"][i] == c["position"]
            assert a["ahead"][i][:len(c.get("jobs", [c.get("first")]))] == c.get("jobs", [c.get("first")])
        assert a["position"][2] == 549
    finally:
        m.close()


def test_golden_edges():
    sc = GOLDEN["edges"]
    m = loaded(sc, "golden-edges")
    try:
        a = m.check(sc["queries"])
        for i, j in enumerate(sc["queries"]):
            w = sc["want"][str(j)]
            assert (a["status"][i], a["position"][i], a["ahead"][i]) == (w["status"], w["position"], w["ahead"])
            if str(j) in sc["usage"]:
                assert [bits(x) for x in a["usage"][i]] == [bits(x) for x in sc["usage"][str(j)]]
        lim = sc["limits"]
        i = sc["queries"].index(lim["job"])
        assert cycle.exceeded(lim["equal"], a["usage"][i]) == {}
        assert cycle.exceeded(lim["below"], a["usage"][i]) == lim["want_below"]
    finally:
        m.close()


# ---- a churn past one sort tile ----------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["grid", "off"])
def test_churn(regime):
    rng = np.random.default_rng(7 if regime == "grid" else 8)
    m = Mirror(f"churn-{regime}")
    U_ = 12
    next_job, next_tid, now = [1], [10 ** 6], [M.START]

    def new_pending(n):
        rows = []
        user = M.zipf_users(rng, n, U_)
        cpus, mem, gpus = M.amounts(rng, regime, n)
        for i in range(n):
            rows.append(dict(job_id=next_job[0], user=int(user[i]), priority=int(rng.choice([10, 50, 50, 90])),
                             cpus=float(cpus[i]), mem=float(mem[i]), gpus=float(gpus[i]),
                             plugin_accept=int(rng.random() < 0.9)))
            next_job[0] += 1 + int(rng.integers(0, 3))
        return rows

    def tids(n):
        out = []
        for _ in range(n):
            next_tid[0] += 1 + int(rng.integers(0, 3))
            out.append(next_tid[0])
        return out

    try:
        m.apply(up=new_pending(7500))
        for batch in range(6):
            pend = sorted(m.pend)
            # launches, in a shuffled task-id order so slot order is not task order
            go = [int(j) for j in rng.choice(pend, 1500 if batch == 0 else 150, replace=False)]
            t = tids(len(go))
            rng.shuffle(t)
            now[0] += 1000
            m.launch(go, t, [now[0] + int(rng.integers(0, 50_000)) for _ in go])
            # extra instances of running jobs (unknown rows of the same job), finishes, kills, priority upserts
            run = list(m.run.values())
            extra = [dict(r, task_id=tid, start_time=r["start_time"] + int(rng.integers(-5, 5)))
                     for r, tid in zip([run[k] for k in rng.choice(len(run), 60, replace=False)], tids(60))]
            fin = [int(x) for x in rng.choice(sorted(m.run), 80, replace=False)]
            m.apply(run_up=extra, run_rm=fin)
            pend = sorted(m.pend)
            kill = [int(j) for j in rng.choice(pend, 40, replace=False)]
            keep = [j for j in pend if j not in set(kill)]
            prio = [dict(m.pend[int(j)], priority=int(rng.choice([10, 50, 90]))) for j in rng.choice(keep, 100, replace=False)]
            m.apply(up=prio + new_pending(200), rm=kill)
            heavy = [j for j, r in m.pend.items() if r["user"] == 0]
            assert len(heavy) + len({r["job_id"] for r in m.run.values() if r["user"] == 0}) > 2048
            jobs = sorted({r["job_id"] for r in m.run.values()})
            q = ([int(x) for x in rng.choice(sorted(m.pend), 300)] + [int(x) for x in rng.choice(jobs, 200)] +
                 fin[:20] + kill[:20] + [10 ** 12])
            rng.shuffle(q)
            m.check(q + q[:50])
            m.check(heavy)
    finally:
        m.close()


# ---- nothing resident changes ------------------------------------------------------------------------------------
def test_match_in_between():
    """Two handles with the same rows, ranked alike: one answers queries around its match.  Queue, digest, the usage
    the match read and the next match are those of the twin."""
    t = M.c2(5)
    pend, run = M.pool_rows(t)
    twins = [M.Pool.of_trace(t, name=f"twin-{k}") for k in range(2)]
    try:
        for p in twins:
            p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
            p.rank()
        a, b = twins
        q = [int(j) for j in list(pend)[:300]] + [int(r["job_id"]) for r in list(run.values())[:100]]
        a.gpu.state_unscheduled(q)
        ga = a.gpu.state_match(a.offers, a.users, a.params, max_ports=a.max_ports, derived=True)
        gb = b.gpu.state_match(b.offers, b.users, b.params, max_ports=b.max_ports, derived=True)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ga[k], gb[k]), k
        a.gpu.state_unscheduled(q)
        assert np.array_equal(a.gpu.state_queue(), b.gpu.state_queue())
        assert digest(a.gpu) == digest(b.gpu)
        nu = a.users.n_users
        assert np.array_equal(a.gpu.exchange_usage(nu), b.gpu.exchange_usage(nu))
        ca = a.gpu.state_considerable(a.users, abi.ConsiderableParams(num_considerable=100, quota_only=1,
                                                                       usage_source=abi.USAGE_LAST_MATCH))
        cb = b.gpu.state_considerable(b.users, abi.ConsiderableParams(num_considerable=100, quota_only=1,
                                                                       usage_source=abi.USAGE_LAST_MATCH))
        assert np.array_equal(ca, cb)
        ga = a.gpu.state_match(a.offers, a.users, a.params, max_ports=a.max_ports, derived=True)
        gb = b.gpu.state_match(b.offers, b.users, b.params, max_ports=b.max_ports, derived=True)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ga[k], gb[k]), k
    finally:
        for p in twins:
            p.close()


# ---- the reasons through a resident match ------------------------------------------------------------------------
def test_investigations_through_match_offers():
    """Job 1 fits no host (cpus): its summary is recorded and shown.  Job 2 fails on every VM only for ports, which
    cook_match_failures counts in n_ports alone: its summary is empty and it stays under investigation."""
    from offer_ref import offers_soa
    users = abi.make_users(1)
    p = M.Pool("investigate", users=users)
    try:
        rows = [(0, dict(M.DEFAULTS, user=0, priority=90, cpus=1.0, mem=1.0, novel=[], attr=[], groups=[])),
                (1, dict(M.DEFAULTS, user=0, priority=80, cpus=1000.0, mem=1.0, novel=[], attr=[], groups=[])),
                (2, dict(M.DEFAULTS, user=0, priority=70, cpus=1.0, mem=1.0, ports=1, novel=[], attr=[], groups=[]))]
        p.apply(up=rows)
        inv = cycle.Investigations()
        a = p.gpu.state_unscheduled([0, 1, 2])
        for i in range(3):
            assert cycle.unscheduled_reasons(a, i, investigations=inv)[-1][0].startswith("The job is now under")
        leases = [{"id": 100 + i, "code": i, "hostname": f"host-{i}", "cpus": 4.0, "mem": 1024.0} for i in range(3)]
        soa, ids, _, _, names = offers_soa(leases)
        p.gpu.state_offers_add(soa, ids, M.START, hostnames=names)
        p.rank()
        got = p.gpu.state_match_offers(M.START, 60_000, users, traces.match_params(10))
        assign = dict(zip(got["considerable"].tolist(), got["assign"].tolist()))
        assert assign[0] >= 0 and assign[1] < 0 and assign[2] < 0
        inv.record(p.gpu, got)
        assert set(inv.summary) == {1} and inv.summary[1] == {"resources": {"cpus": 3}}
        assert inv.marked == {0, 2}
        a = p.gpu.state_unscheduled([1, 2])
        assert cycle.unscheduled_reasons(a, 0, investigations=inv)[-1] == [
            "The job couldn't be placed on any available hosts.",
            {"reasons": [{"reason": "Not enough cpus available.", "host_count": 3}]}]
        assert cycle.unscheduled_reasons(a, 1, investigations=inv)[-1][0].startswith("The job is now under")
    finally:
        p.close()


# ---- errors ------------------------------------------------------------------------------------------------------
def test_badargs_leave_the_digest():
    sc = GOLDEN["edges"]
    m = loaded(sc, "badargs")
    try:
        before = digest(m.e)
        lib, h = m.e.lib, m.e.pool
        jid = np.array([1103, 2000], np.int64)
        st, pl = np.full(2, 7, np.uint8), np.full(2, 7, np.uint8)
        us = np.full(8, 7.0)
        pos, na = np.full(2, 7, np.int32), np.full(2, 7, np.int32)
        ah = np.full(20, 7, np.int64)
        outs = [abi.ptr(st, abi.P_U8), abi.ptr(us, abi.P_F64), abi.ptr(pos, abi.P_I32), abi.ptr(na, abi.P_I32),
                abi.ptr(ah, abi.P_I64), abi.ptr(pl, abi.P_U8)]
        assert lib.cook_state_unscheduled(h, -1, abi.ptr(jid, abi.P_I64), *outs, None) == abi.COOK_E_BADARG
        assert lib.cook_state_unscheduled(None, 2, abi.ptr(jid, abi.P_I64), *outs, None) == abi.COOK_E_BADARG
        assert lib.cook_state_unscheduled(h, 2, None, *outs, None) == abi.COOK_E_BADARG
        for k in range(len(outs)):
            o = list(outs)
            o[k] = None
            assert lib.cook_state_unscheduled(h, 2, abi.ptr(jid, abi.P_I64), *o, None) == abi.COOK_E_BADARG
        for x in (st, us, pos, na, ah, pl):
            assert (x == 7).all()
        assert lib.cook_state_unscheduled(h, 0, None, None, None, None, None, None, None, None) == abi.COOK_OK
        assert digest(m.e) == before
        m.check(sc["queries"])
        # every query absent: no device work
        m.check([10 ** 9, 10 ** 9 + 1])
    finally:
        m.close()
    e = engine.GpuEngine(pool_name="empty")
    try:
        a = e.state_unscheduled([5, 5])
        assert list(a["status"]) == [abi.UNSCHED_ABSENT] * 2 and list(a["position"]) == [-1, -1]
        assert a["stats"]["n_launches"] == 0
    finally:
        e.close()
