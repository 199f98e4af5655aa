"""-m gpu: cook_state_instance_stats against instance_stats_ref over a host mirror, bit for bit, and
cook_state_task_reason's fact.

The golden edges and the transcribed integration assertions replay on resident handles through
cycle.instance_stats_response.  A churn of launches, finishes, extra instances, reasons and unknown facts over three
handles, with a Zipf user past one 2048-wide sort tile, on and off the grid, checks both statuses under several windows
and entity-id bounds after every batch.  The reason fact is reset by an upsert and a launch and kept by
cook_state_patch and cook_state_task_facts; the overall count equals cook_state_user_usage's job count where every job
has one row; a twin handle shows a match after the call is unchanged; BADARGs leave the digest unchanged; each call's
transfers follow the header's formula.
"""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import instance_stats_ref as I
import resident_model as M
from cook_b200 import abi, cycle, engine
from cook_b200.engine import CookError

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instance_stats_golden.json")))
REASONS = {int(k): v for k, v in GOLDEN["reasons"].items()}
DROP = M.drop_all_but("gpus", "groups")
LO, HI = -(1 << 63), (1 << 63) - 1


def bits(x):
    return struct.unpack("<q", struct.pack("<d", float(x)))[0]


def plain(x):
    return json.loads(json.dumps(x))


def status_code(s):
    return abi.IS_UNKNOWN if s == "unknown" else abi.IS_RUNNING


class Pools:
    """Resident handles and a mirror of their running rows, {task id: row} per handle (with the reason code and the
    unknown fact), and pending rows {job id: row}."""

    def __init__(self, names):
        self.names = list(names)
        self.e = [engine.GpuEngine(pool_name=f"is-{n}") for n in self.names]
        self.run = [{} for _ in self.names]
        self.pend = [{} for _ in self.names]

    def close(self):
        for e in self.e:
            e.close()

    def apply(self, p, up=(), rm=(), run_up=(), run_rm=()):
        up, run_up = list(up), list(run_up)
        self.e[p].state_apply(M.delta(up=[(r["job_id"], r) for r in up], rm=rm, run_up=run_up, run_rm=run_rm,
                                      drop=DROP, lists=True))
        for j in rm:
            del self.pend[p][j]
        for t in run_rm:
            del self.run[p][t]
        self.pend[p].update((r["job_id"], r) for r in up)
        self.run[p].update((r["task_id"], dict(r, reason=-1, unknown=False)) for r in run_up)

    def launch(self, p, jobs, tids, starts):
        self.e[p].state_launch(jobs, tids, starts)
        for j, t, s in zip(jobs, tids, starts):
            r = self.pend[p].pop(j)
            self.run[p][t] = dict(task_id=t, job_id=j, user=r["user"], priority=r["priority"], start_time=s,
                                  cpus=r["cpus"], mem=r["mem"], gpus=r.get("gpus", 0.0), groups=list(r["groups"]),
                                  reason=-1, unknown=False)

    def reason(self, p, tids, codes):
        self.e[p].state_task_reason(tids, codes)
        for t, c in zip(tids, codes):
            self.run[p][t]["reason"] = int(c)

    def unknown(self, p, tids, flags):
        self.e[p].state_task_facts(tids, unknown=np.asarray(flags, np.uint8))
        for t, f in zip(tids, flags):
            self.run[p][t]["unknown"] = bool(f)

    def load(self, rows_by_handle):
        for p, rows in enumerate(rows_by_handle):
            self.apply(p, run_up=[dict(r, priority=50, gpus=0.0, groups=[]) for r in rows])
            rs = [r for r in rows if r.get("reason", -1) != -1]
            if rs:
                self.reason(p, [r["task_id"] for r in rs], [r["reason"] for r in rs])
            us = [r for r in rows if r.get("unknown")]
            if us:
                self.unknown(p, [r["task_id"] for r in us], [1] * len(us))

    def check(self, now, status, start, end, lo=LO, hi=HI, idx=None):
        """The call over handles idx (default all) against the restatement, bit for bit, and its transfers."""
        idx = list(range(len(self.e))) if idx is None else idx
        hs = [self.run[k] for k in idx]
        got = engine.state_instance_stats([self.e[k] for k in idx], now, status_code(status), start, end, lo, hi)
        segs, lc, lm = I.answer(hs, now, status, start, end, lo, hi)
        assert len(got["kind"]) == len(segs)
        for d, w in enumerate(segs):
            assert (int(got["kind"][d]), int(got["user"][d]), int(got["reason"][d]), int(got["count"][d])) == w[:4], d
            assert [bits(x) for x in got["total"][d]] == [bits(x) for x in w[4]], (d, w)
            assert [[bits(x) for x in m] for m in got["pct"][d]] == [[bits(x) for x in m] for m in w[5]], (d, w)
        for g, w in ((got["leaders_cpu"], lc), (got["leaders_mem"], lm)):
            assert [(u, bits(t)) for u, t in g] == [(u, bits(t)) for u, t in w]
        s = got["stats"]
        if any(hs):
            assert s["h2d_bytes"] == 0
            assert s["d2h_bytes"] == I.d2h_bytes(segs, lc, bool(segs))
        else:
            assert s["h2d_bytes"] == s["d2h_bytes"] == s["n_launches"] == 0
        return got


def digest(e):
    return {k: v for k, v in e.state_digest().items() if "buckets" not in k}


# ---- the golden scenarios on resident handles ---------------------------------------------------------------------
def edge_pools():
    h = GOLDEN["edges"]["handles"]
    ps = Pools(["a", "b", "c"])
    ps.load([h[k] for k in ("a", "b", "c")])
    return ps


def test_golden_edges():
    ps = edge_pools()
    try:
        for case in GOLDEN["edges"]["cases"]:
            q = case["request"]
            ps.check(q["now"], q["status"], q["start"], q["end"], q["lo"], q["hi"])
            a = engine.state_instance_stats(ps.e, q["now"], status_code(q["status"]), q["start"], q["end"], q["lo"],
                                            q["hi"])
            got = cycle.instance_stats_response(a, user_name=str, reason_string=REASONS.get)
            assert plain(got) == case["want"]
            for m in ("cpu-seconds", "mem-seconds"):
                assert list(got["leaders"][m].items()) == list(case["want"]["leaders"][m].items())
        # one handle, and the handles in another order: the fold order is (task id, pool index)
        now = GOLDEN["edges"]["cases"][0]["request"]["now"]
        for idx in ([0], [1], [2, 1, 0], [1, 0]):
            for status in ("running", "unknown"):
                ps.check(now, status, now - 60000, now, idx=idx)
    finally:
        ps.close()


@pytest.mark.parametrize("k", range(len(GOLDEN["transcribed"])))
def test_golden_transcribed(k):
    t = GOLDEN["transcribed"][k]
    q = t["request"]
    ps = Pools(["t"])
    try:
        ps.load(t["handles"])
        ps.check(q["now"], q["status"], q["start"], q["end"])
        r = cycle.instance_stats_response(engine.state_instance_stats(ps.e, q["now"], abi.IS_RUNNING, q["start"],
                                                                      q["end"]), user_name=str)
        assert r["overall"]["count"] == r["by-reason"][""]["count"] == r["by-user-and-reason"][str(t["user"])][""][
            "count"] == t["count"]
        for key, chk in t.get("checks", {}).items():
            assert plain(r["overall"][key]["percentiles"]) == chk["percentiles"]
            assert r["overall"][key]["total"] == pytest.approx(chk["total_approx"], abs=1e-7)
    finally:
        ps.close()


# ---- a churn past one sort tile -----------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["grid", "off"])
def test_churn(regime):
    rng = np.random.default_rng(21 if regime == "grid" else 22)
    ps = Pools(["a", "b", "c"])
    U_ = 14
    next_job, next_tid, now = [1], [10 ** 6], [M.START]

    def new_pending(n):
        user = M.zipf_users(rng, n, U_)
        cpus, mem, gpus = M.amounts(rng, regime, n)
        rows = []
        for i in range(n):
            rows.append(dict(job_id=next_job[0], user=int(user[i]), priority=50, cpus=float(cpus[i]),
                             mem=float(mem[i]), gpus=float(gpus[i]), groups=[]))
            next_job[0] += 1 + int(rng.integers(0, 2))
        return rows

    def tids(n):
        out = []
        for _ in range(n):
            next_tid[0] += 1 + int(rng.integers(0, 3))
            out.append(next_tid[0])
        return out

    def start():   # grid: whole seconds; off: any millisecond
        return now[0] - (1000 * int(rng.integers(0, 30)) if regime == "grid" else int(rng.integers(0, 30000)))

    try:
        for p in range(3):
            ps.apply(p, up=new_pending(9000 if p == 0 else 800))
        for batch in range(4):
            for p in range(3):
                pend = sorted(ps.pend[p])
                go = [int(j) for j in rng.choice(pend, min(len(pend), 7000 if batch == 0 and p == 0 else 150),
                                                 replace=False)]
                t = tids(len(go))
                rng.shuffle(t)
                now[0] += 60000
                ps.launch(p, go, t, [start() for _ in go])
                run = list(ps.run[p].values())
                extra = [dict(r, task_id=tid, start_time=start())
                         for r, tid in zip([run[k] for k in rng.choice(len(run), 40, replace=False)], tids(40))]
                fin = [int(x) for x in rng.choice(sorted(ps.run[p]), 50, replace=False)]
                ps.apply(p, run_up=extra, run_rm=fin)
                live = sorted(ps.run[p])
                rs = [int(x) for x in rng.choice(live, len(live) // 5, replace=False)]
                ps.reason(p, rs, [int(c) for c in rng.choice([-1, 1001, 1002, 2003], len(rs))])
                us = [int(x) for x in rng.choice(live, len(live) // 6, replace=False)]
                ps.unknown(p, us, [int(x) for x in rng.integers(0, 2, len(us))])
            # the same task id in a second handle
            r0 = next(iter(ps.run[0].values()))
            if r0["task_id"] not in ps.run[1]:
                ps.apply(1, run_up=[dict(r0)])
            sel = sum(1 for run in ps.run for r in run.values() if not r["unknown"])
            assert sel > 2048
            T = now[0] + 1000
            lo_tid = 10 ** 6 + 3000
            for status in ("running", "unknown"):
                ps.check(T, status, M.START - 10 ** 9, T + 1)
                ps.check(T, status, now[0] - 15000, now[0] - 5000, lo_tid, next_tid[0] - 500)
            ps.check(T, "running", M.START - 10 ** 9, T + 1, idx=[2, 0])
    finally:
        ps.close()


# ---- the reason fact ----------------------------------------------------------------------------------------------
def by_reason(ps, now):
    a = engine.state_instance_stats(ps.e, now, abi.IS_RUNNING, 0, now + 1)
    return {int(a["reason"][d]): int(a["count"][d]) for d in range(len(a["kind"])) if a["kind"][d] == abi.IS_REASON}


def test_reason_lifecycle():
    ps = Pools(["r"])
    now = M.START + 10 ** 6
    rows = [dict(task_id=10 + k, job_id=100 + k, user=k % 3, priority=50, start_time=M.START, cpus=1.0, mem=64.0,
                 gpus=0.0, groups=[]) for k in range(6)]
    try:
        ps.apply(0, up=[dict(job_id=200, user=1, priority=50, cpus=1.0, mem=8.0, gpus=0.0, groups=[])], run_up=rows)
        assert by_reason(ps, now) == {-1: 6}
        ps.reason(0, [10, 11, 12], [1001, 1001, 2003])
        assert by_reason(ps, now) == {-1: 3, 1001: 2, 2003: 1}
        # kept by the other facts and by a patch of the pending rows
        ps.e[0].state_task_facts([10, 12], max_runtime_ms=[5, -1], cancelled=[1, 0], unknown=[0, 0])
        ps.e[0].state_patch([200], allowed=[0])
        assert by_reason(ps, now) == {-1: 3, 1001: 2, 2003: 1}
        ps.check(now, "running", 0, now + 1)
        # reset by an upsert of a running id
        ps.apply(0, run_up=[rows[0]])
        assert by_reason(ps, now) == {-1: 4, 1001: 1, 2003: 1}
        # a launch writes none, even into a slot a row with a reason left
        ps.apply(0, run_rm=[12])
        ps.launch(0, [200], [12], [M.START])
        assert by_reason(ps, now) == {-1: 5, 1001: 1}
        ps.check(now, "running", 0, now + 1)
        # errors leave the facts and the digest
        before = digest(ps.e[0])
        for tid, codes in (([10, 10], [1, 1]), ([99], [1]), ([10], [-2])):
            with pytest.raises(CookError):
                ps.e[0].state_task_reason(tid, codes)
        lib = ps.e[0].lib
        assert lib.cook_state_task_reason(ps.e[0].pool, -1, None, None) == abi.COOK_E_BADARG
        assert lib.cook_state_task_reason(ps.e[0].pool, 1, None, abi.ptr(np.zeros(1, np.int32), abi.P_I32)) == \
            abi.COOK_E_BADARG
        assert digest(ps.e[0]) == before
        assert by_reason(ps, now) == {-1: 5, 1001: 1}
        # uploads 8 B per row
        ps.reason(0, [10, 11], [2003, -1])
        assert ps.e[0].last_stats(abi.PHASE_STATE)["h2d_bytes"] == 16
    finally:
        ps.close()


# ---- cross-check against cook_state_user_usage --------------------------------------------------------------------
def test_count_matches_user_usage():
    rng = np.random.default_rng(7)
    ps = Pools(["x", "y"])
    try:
        rows = M.random_rows(rng, "off", 4000, 9, 10 ** 6, [1, 2, 3])
        for p in range(2):
            ps.apply(p, run_up=[dict(r, priority=50, start_time=M.START - int(rng.integers(0, 10 ** 6)), groups=[])
                                for r in rows[p::2]])
            live = sorted(ps.run[p])
            ps.unknown(p, live[::7], [1] * len(live[::7]))
        now = M.START + 1
        u = engine.state_user_usage(ps.e, None, False, False)
        jobs = {int(u["user"][d]): int(u["jobs"][d]) for d in range(len(u["user"]))}
        counts = {}
        for status in ("running", "unknown"):
            a = ps.check(now, status, 0, now)
            for d in range(len(a["kind"])):
                if a["kind"][d] == abi.IS_USER_REASON:
                    counts[int(a["user"][d])] = counts.get(int(a["user"][d]), 0) + int(a["count"][d])
        assert counts == jobs
    finally:
        ps.close()


# ---- nothing resident changes -------------------------------------------------------------------------------------
def test_match_in_between():
    """Two handles with the same rows, ranked alike: one answers instance stats around its match.  Queue, digest,
    the usage the match read and the next match are those of the twin."""
    t = M.c2(5)
    pend, run = M.pool_rows(t)
    twins = [M.Pool.of_trace(t, name=f"is-twin-{k}") for k in range(2)]
    try:
        for p in twins:
            p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
            p.rank()
        a, b = twins
        now = M.START + 10 ** 9
        engine.state_instance_stats([a.gpu], now, abi.IS_RUNNING, 0, now)
        ga = a.gpu.state_match(a.offers, a.users, a.params, max_ports=a.max_ports, derived=True)
        gb = b.gpu.state_match(b.offers, b.users, b.params, max_ports=b.max_ports, derived=True)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ga[k], gb[k]), k
        engine.state_instance_stats([a.gpu], now, abi.IS_UNKNOWN, 0, now)
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
        R = sum(len(r) for r in ps.run)
        cap = 1 + 2 * R
        now = GOLDEN["edges"]["cases"][0]["request"]["now"]
        outs = [np.full(cap, 7, np.int32), np.full(cap, 7, np.int32), np.full(cap, 7, np.int32),
                np.full(cap, 7, np.int64), np.full(3 * cap, 7.0), np.full(15 * cap, 7.0),
                np.full(20, 7, np.int32), np.full(20, 7.0)]
        types = [abi.P_I32, abi.P_I32, abi.P_I32, abi.P_I64, abi.P_F64, abi.P_F64, abi.P_I32, abi.P_F64]
        op = [abi.ptr(o, t) for o, t in zip(outs, types)]
        n = [C.c_int32(7), C.c_int32(7)]

        def call(handles, status=abi.IS_RUNNING, start=0, end=now, t_now=now, seg_cap=cap, o=None, cnt=None):
            hs = (C.c_void_p * len(handles))(*handles)
            return lib.cook_state_instance_stats(hs, len(handles), t_now, status, start, end, LO, HI, seg_cap,
                                                 *(o or op), *(cnt or [C.byref(n[0]), C.byref(n[1])]), None)

        h = [e.pool for e in ps.e]
        bad = abi.COOK_E_BADARG
        assert call([h[0], h[1], h[0]]) == bad                     # a handle twice
        assert call([h[0], None]) == bad                           # a NULL handle
        assert call(h, status=2) == bad
        assert call(h, start=now, end=now) == bad                  # end <= start
        assert call(h, seg_cap=cap - 1) == bad
        for k in range(8):
            o = list(op)
            o[k] = None
            assert call(h, o=o) == bad
        assert call(h, cnt=[None, C.byref(n[1])]) == bad
        assert call(h, cnt=[C.byref(n[0]), None]) == bad
        # a selected row that starts after now; one that is not selected does not matter
        assert call(h, t_now=now - 1500) == bad
        for x in outs:
            assert (x == 7).all()
        assert n[0].value == n[1].value == 7
        assert call(h, t_now=now - 1500, end=now - 2000) == abi.COOK_OK
        assert n[0].value > 0
        assert [digest(e) for e in ps.e] == before
        # nothing selected: empty results after the selection
        ps.check(now, "unknown", now - 10, now)
    finally:
        ps.close()
    e = engine.GpuEngine(pool_name="is-empty")
    try:
        a = engine.state_instance_stats([e], M.START, abi.IS_RUNNING, 0, M.START)
        assert len(a["kind"]) == 0 and a["leaders_cpu"] == [] and a["stats"]["n_launches"] == 0
        with pytest.raises(CookError):
            engine.state_instance_stats([e, e], M.START, abi.IS_RUNNING, 0, M.START)
    finally:
        e.close()
