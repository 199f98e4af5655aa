"""-m gpu: cook_state_user_usage against user_usage_ref over a host mirror, bit for bit.

The golden scenarios (the reference's usage tests, the shim routing jobs without a pool to the default pool's handle,
and the hand-computed edges) replay on resident handles through cycle.usage_response.  A churn of launches, finishes,
extra instances and group changes over three handles, with a Zipf user past one 2048-wide sort tile, on and off the
grid, checks one user, several users and every user, with and without per_pool and by_group, after every batch.
Cross-checks against cook_state_usage and cook_state_unscheduled; a twin handle shows the call changes nothing a match
reads; BADARGs leave the digest unchanged; each call's transfers follow the header's formula.
"""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import resident_model as M
import user_usage_ref as U
from cook_b200 import abi, cycle, engine
from cook_b200.engine import CookError

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "user_usage_golden.json")))
DROP = M.drop_all_but("gpus", "groups")


def bits(x):
    return struct.unpack("<q", struct.pack("<d", float(x)))[0]


def plain(x):
    return json.loads(json.dumps(x))


class Pools:
    """Resident handles and their running rows, {task id: row} per handle, and pending rows {job id: row}."""

    def __init__(self, names):
        self.names = list(names)
        self.e = [engine.GpuEngine(pool_name=f"uu-{n}") for n in self.names]
        self.run = [{} for _ in self.names]
        self.pend = [{} for _ in self.names]

    def close(self):
        for e in self.e:
            e.close()

    def apply(self, p, up=(), rm=(), run_up=(), run_rm=(), gpus=True):
        up, run_up = list(up), list(run_up)
        self.e[p].state_apply(M.delta(up=[(r["job_id"], r) for r in up], rm=rm, run_up=run_up, run_rm=run_rm,
                                      drop=DROP, lists=True, gpus=gpus))
        for j in rm:
            del self.pend[p][j]
        for t in run_rm:
            del self.run[p][t]
        self.pend[p].update((r["job_id"], r) for r in up)
        self.run[p].update((r["task_id"], r if gpus else dict(r, gpus=0.0)) for r in run_up)

    def launch(self, p, jobs, tids, starts):
        self.e[p].state_launch(jobs, tids, starts)
        for j, t, s in zip(jobs, tids, starts):
            r = self.pend[p].pop(j)
            self.run[p][t] = dict(task_id=t, job_id=j, user=r["user"], priority=r["priority"], start_time=s,
                                  cpus=r["cpus"], mem=r["mem"], gpus=r["gpus"], groups=list(r["groups"]))

    def check(self, users=None, per_pool=False, by_group=False, idx=None):
        """The call over handles idx (default all) against the restatement, bit for bit, and its transfers."""
        idx = list(range(len(self.e))) if idx is None else idx
        hs = [self.run[k] for k in idx]
        got = engine.state_user_usage([self.e[k] for k in idx], users, per_pool, by_group)
        want = U.answer(hs, None if users is None else set(users), per_pool, by_group)
        assert len(got["user"]) == len(want)
        for d, w in enumerate(want):
            assert (int(got["user"][d]), int(got["scope"][d]), int(got["group"][d]), int(got["jobs"][d])) == w[:4], d
            assert [bits(got[k][d]) for k in ("cpus", "mem", "gpus")] == [bits(x) for x in w[4:7]], (d, w)
            assert got["lists"][d] == w[7], d
        s = got["stats"]
        if U.rows_queried(hs, None if users is None else set(users)):
            assert s["h2d_bytes"] == 4 * len(users or ())
            assert s["d2h_bytes"] == U.d2h_bytes(want, by_group)
        else:
            assert s["h2d_bytes"] == s["d2h_bytes"] == s["n_launches"] == 0
        return got


def run_row(t, j, user, cpus, mem, gpus=0.0, groups=(), start=M.START):
    return dict(task_id=t, job_id=j, user=user, priority=50, start_time=start, cpus=cpus, mem=mem, gpus=gpus,
                groups=list(groups))


def digest(e):
    return {k: v for k, v in e.state_digest().items() if "buckets" not in k}


# ---- the golden scenarios on resident handles ---------------------------------------------------------------------
@pytest.mark.parametrize("k", range(len(GOLDEN["api"])))
def test_golden_api(k):
    """One handle per pool (one without pools); the shim puts a job without a pool in the default pool's handle."""
    step = GOLDEN["api"][k]
    req = step["request"]
    names = step["pools"] or [step["default_pool"]]
    ps = Pools(names)
    try:
        for j in step["jobs"]:
            p = names.index(U.pool_of(j, step["default_pool"])) if step["pools"] else 0
            ps.apply(p, run_up=[run_row(j["task_id"], j["job_id"], j["user"], j["cpus"], j["mem"], j["gpus"])])
        idx = [names.index(req["pool"])] if req.get("pool") else None
        per_pool = not req.get("pool") and bool(step["pools"])
        ps.check([req["user"]], per_pool, idx=idx)
        sel = idx or list(range(len(names)))
        a = engine.state_user_usage([ps.e[i] for i in sel], [req["user"]], per_pool)
        got = cycle.usage_response([(a, [names[i] for i in sel])], user=req["user"], pool=req.get("pool"),
                                   pools=step["pools"])
        assert plain(got) == step["want"]
    finally:
        ps.close()


def edge_pools():
    h = GOLDEN["edges"]["handles"]
    ps = Pools(list(h))
    for p, n in enumerate(ps.names):
        rows = [dict(r, priority=50, start_time=M.START) for r in h[n]]
        with_gpus = all("gpus" in r for r in rows)
        ps.apply(p, run_up=[dict(r, gpus=r.get("gpus", 0.0)) for r in rows], gpus=with_gpus)
    return ps


def test_golden_edges():
    ps = edge_pools()
    groups = {int(g): tuple(v) for g, v in GOLDEN["edges"]["groups"].items()}
    try:
        for case in GOLDEN["edges"]["cases"]:
            req = case["request"]
            gb = req.get("group_breakdown", False)
            users = [req["user"]] if "user" in req else None
            idx = [ps.names.index(req["pool"])] if "pool" in req else list(range(3))
            per_pool = "pool" not in req
            ps.check(users, per_pool, gb, idx=idx)
            a = engine.state_user_usage([ps.e[i] for i in idx], users, per_pool, gb)
            got = cycle.usage_response([(a, [ps.names[i] for i in idx])], user=req.get("user"), pool=req.get("pool"),
                                       pools=ps.names, group_breakdown=gb, group_info=groups.get)
            assert plain(got) == case["want"]
        for users in ([0], [1], [2], [2, 0, 1], [5], None):
            for pp in (False, True):
                for bg in (False, True):
                    ps.check(users, pp, bg)
    finally:
        ps.close()


# ---- a churn past one sort tile -----------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["grid", "off"])
def test_churn(regime):
    rng = np.random.default_rng(11 if regime == "grid" else 12)
    ps = Pools(["a", "b", "c"])
    U_ = 12
    next_job, next_tid, now = [1], [10 ** 6], [M.START]

    def new_pending(n):
        user = M.zipf_users(rng, n, U_)
        cpus, mem, gpus = M.amounts(rng, regime, n)
        rows = []
        for i in range(n):
            g = [int(x) for x in rng.choice(6, int(rng.integers(0, 3)), replace=False)]
            rows.append(dict(job_id=next_job[0], user=int(user[i]), priority=50, cpus=float(cpus[i]),
                             mem=float(mem[i]), gpus=float(gpus[i]), groups=g))
            next_job[0] += 1 + int(rng.integers(0, 2))
        return rows

    def tids(n):
        out = []
        for _ in range(n):
            next_tid[0] += 1 + int(rng.integers(0, 3))
            out.append(next_tid[0])
        return out

    try:
        for p in range(3):
            ps.apply(p, up=new_pending(9000 if p == 0 else 800))
        for batch in range(4):
            for p in range(3):
                pend = sorted(ps.pend[p])
                go = [int(j) for j in rng.choice(pend, min(len(pend), 7000 if batch == 0 and p == 0 else 120),
                                                 replace=False)]
                t = tids(len(go))
                rng.shuffle(t)
                now[0] += 1000
                ps.launch(p, go, t, [now[0]] * len(go))
                run = list(ps.run[p].values())
                # extra instances of running jobs, group changes of running rows, finishes
                extra = [dict(r, task_id=tid) for r, tid in zip([run[k] for k in rng.choice(len(run), 40, replace=False)],
                                                                tids(40))]
                regroup = [dict(r, groups=[int(x) for x in rng.choice(6, int(rng.integers(0, 3)), replace=False)])
                           for r in [run[k] for k in rng.choice(len(run), 30, replace=False)]]
                regroup = [r for r in regroup if r["task_id"] not in {x["task_id"] for x in extra}]
                fin = [int(x) for x in rng.choice(sorted(ps.run[p]), 50, replace=False)]
                fin = [t_ for t_ in fin if t_ not in {r["task_id"] for r in regroup}]
                ps.apply(p, run_up=extra + regroup, run_rm=fin)
            # the same job id in a second handle
            r0 = next(iter(ps.run[0].values()))
            ps.apply(1, run_up=[dict(r0, task_id=tids(1)[0])])
            heavy = sum(1 for run in ps.run for r in run.values() if r["user"] == 0)
            assert heavy > 2048
            for users in ([0], [3, 5, 7], None):
                for pp in (False, True):
                    for bg in (False, True):
                        ps.check(users, pp, bg)
            ps.check([1], True, True, idx=[2, 0])
    finally:
        ps.close()


# ---- cross-checks -------------------------------------------------------------------------------------------------
def test_cross_checks():
    rng = np.random.default_rng(5)
    ps = Pools(["x", "y", "z"])
    try:
        rows = M.random_rows(rng, "off", 3000, 6, 10 ** 6, [1, 2, 3])
        for p in range(3):
            ps.apply(p, run_up=[dict(r, priority=50, start_time=M.START, groups=[]) for r in rows[p::3]])
        # one handle, one row per job: the total is cook_state_usage's user row
        u = ps.e[0].state_usage(6)["user"]
        a = ps.check(None, False, False, idx=[0])
        for d in range(len(a["user"])):
            w = int(a["user"][d])
            assert [bits(a[k][d]) for k in ("cpus", "mem", "gpus")] == [bits(u[k][w]) for k in ("cpus", "mem", "gpus")]
            assert float(a["jobs"][d]) == u["count"][w]
        # no job has a group: every ungrouped segment equals its total
        g = ps.check(None, True, True)
        seg = {(int(g["user"][d]), int(g["scope"][d]), int(g["group"][d])): d for d in range(len(g["user"]))}
        for (w, s, grp), d in seg.items():
            assert grp in (abi.UU_TOTAL, abi.UU_UNGROUPED)
            t = seg[(w, s, abi.UU_TOTAL)]
            assert [bits(g[k][d]) for k in ("jobs", "cpus", "mem", "gpus")] == \
                [bits(g[k][t]) for k in ("jobs", "cpus", "mem", "gpus")]
        # a per-pool segment of the three-handle call is the one-handle call's total
        for p in range(3):
            one = ps.check(None, False, False, idx=[p])
            for d in range(len(one["user"])):
                e = seg[(int(one["user"][d]), p, abi.UU_TOTAL)]
                assert [bits(one[k][d]) for k in ("jobs", "cpus", "mem", "gpus")] == \
                    [bits(g[k][e]) for k in ("jobs", "cpus", "mem", "gpus")]
        # a waiting job: cook_state_unscheduled's usage is this call's total plus the job, in f64
        job = dict(job_id=9 * 10 ** 8, user=2, priority=50, cpus=0.3, mem=1000.0 / 7.0, gpus=0.1, groups=[])
        ps.apply(0, up=[job])
        un = ps.e[0].state_unscheduled([job["job_id"]])
        a = ps.check([2], False, False, idx=[0])
        assert len(a["user"]) == 1
        want = [float(a["jobs"][0]) + 1.0] + [a[k][0] + job[k] for k in ("cpus", "mem", "gpus")]
        assert [bits(x) for x in un["usage"][0]] == [bits(x) for x in want]
    finally:
        ps.close()


# ---- nothing resident changes -------------------------------------------------------------------------------------
def test_match_in_between():
    """Two handles with the same rows, ranked alike: one answers usage queries around its match.  Queue, digest, the
    usage the match read and the next match are those of the twin."""
    t = M.c2(5)
    pend, run = M.pool_rows(t)
    twins = [M.Pool.of_trace(t, name=f"uu-twin-{k}") for k in range(2)]
    try:
        for p in twins:
            p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
            p.rank()
        a, b = twins
        engine.state_user_usage([a.gpu], None, True, True)
        ga = a.gpu.state_match(a.offers, a.users, a.params, max_ports=a.max_ports, derived=True)
        gb = b.gpu.state_match(b.offers, b.users, b.params, max_ports=b.max_ports, derived=True)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ga[k], gb[k]), k
        engine.state_user_usage([a.gpu], [0, 1, 2], False, True)
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


# ---- errors -------------------------------------------------------------------------------------------------------
def test_badargs_leave_the_digest():
    ps = edge_pools()
    try:
        before = [digest(e) for e in ps.e]
        lib = ps.e[0].lib
        R_q = U.rows_queried(ps.run, {0})   # alice: 7 rows
        cap = 4 * R_q
        i32 = lambda: np.full(cap, 7, np.int32)
        outs = [i32(), i32(), i32(), np.full(cap, 7, np.int64), np.full(cap, 7.0), np.full(cap, 7.0), np.full(cap, 7.0),
                i32()]
        jid = np.full(cap, 7, np.int64)
        n = [C.c_int32(7), C.c_int32(7)]
        types = [abi.P_I32, abi.P_I32, abi.P_I32, abi.P_I64, abi.P_F64, abi.P_F64, abi.P_F64, abi.P_I32]
        op = [abi.ptr(o, t) for o, t in zip(outs, types)]

        def call(handles, users, n_users=None, pp=1, bg=1, seg_cap=cap, job_cap=2 * R_q, o=None, j="x", cnt=None):
            hs = (C.c_void_p * len(handles))(*handles)
            u = np.asarray(users, np.int32) if users is not None else None
            o = op if o is None else o
            return lib.cook_state_user_usage(hs, len(handles), abi.ptr(u, abi.P_I32) if u is not None else None,
                                             len(u) if n_users is None and u is not None else (n_users or 0), pp, bg,
                                             seg_cap, *o[:7], o[7], job_cap,
                                             abi.ptr(jid, abi.P_I64) if j == "x" else j,
                                             *(cnt or [C.byref(n[0]), C.byref(n[1])]), None)

        h = [e.pool for e in ps.e]
        bad = abi.COOK_E_BADARG
        assert call([h[0], h[1], h[0]], [0]) == bad                  # a handle twice
        assert call([h[0], None], [0]) == bad                        # a NULL handle
        assert call([h[0]], [0], n_users=-1) == bad
        assert call([h[0]], None, n_users=2) == bad                  # n_users without a list
        assert call(h, [0, -1]) == bad
        assert call(h, [3, 0, 3]) == bad
        assert call(h, [0], seg_cap=cap - 1) == bad
        assert call(h, [0], job_cap=2 * R_q - 1) == bad
        assert call(h, [0], pp=0, seg_cap=2 * R_q - 1) == bad
        for k in range(8):
            o = list(op)
            o[k] = None
            assert call(h, [0], o=o) == bad
        assert call(h, [0], j=None) == bad
        assert call(h, [0], cnt=[None, C.byref(n[1])]) == bad
        for x in outs + [jid]:
            assert (x == 7).all()
        assert n[0].value == n[1].value == 7
        # without by_group the list arguments are not read, and the bounds are the smaller ones
        assert call(h, [0], bg=0, seg_cap=2 * R_q, job_cap=0, o=op[:7] + [None], j=None) == abi.COOK_OK
        assert n[0].value > 0 and n[1].value == 0
        assert [digest(e) for e in ps.e] == before
        ps.check([0], True, True)
        # no row of the queried users: no device work
        ps.check([2, 9], True, True)
        ps.check([], False, True)
    finally:
        ps.close()
    e = engine.GpuEngine(pool_name="uu-empty")
    try:
        a = engine.state_user_usage([e], None, True, True)
        assert len(a["user"]) == 0 and a["stats"]["n_launches"] == 0
        with pytest.raises(CookError):
            engine.state_user_usage([e, e])
    finally:
        e.close()
