"""-m gpu: the finished-instance history (cook_state_history_seed, cook_state_finish_history,
cook_state_history_advance) and cook_state_history_stats against history_ref over a host mirror, bit for bit.

The golden edges and the transcribed integration assertions replay on seeded handles through
cycle.instance_stats_response.  A churn of launches, running upserts, reason facts, successes and failures (with and
without reason codes) and advances over three handles, with a Zipf user past one 2048-wide sort tile, on and off the
grid, checks both statuses under several windows and id bounds after every batch.  A twin handle fed cook_state_finish
shows the history changes nothing else; a fresh handle seeded with the mirror's rows answers alike; the horizon rules,
a reset, seg_cap's retry, BADARGs and each call's transfers are checked.
"""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import history_ref as Hr
import resident_model as M
from cook_b200 import abi, cycle, engine
from cook_b200.engine import CookError

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "history_stats_golden.json")))
REASONS = {int(k): v for k, v in GOLDEN["reasons"].items()}
DROP = M.drop_all_but("gpus", "groups")
LO, HI = -(1 << 63), (1 << 63) - 1
COLS = ("task_id", "user", "start", "end", "cpus", "mem", "success", "reason")


def bits(x):
    return struct.unpack("<q", struct.pack("<d", float(x)))[0]


def plain(x):
    return json.loads(json.dumps(x))


def status_code(s):
    return abi.IS_SUCCESS if s == Hr.SUCCESS else abi.IS_FAILED


def seed(e, h, since, rows):
    """Seed engine e and mirror h alike."""
    cols = {k: [r[k] for r in rows] for k in COLS}
    e.state_history_seed(since, cols["task_id"], cols["user"], cols["start"], cols["end"], cols["cpus"], cols["mem"],
                         [int(x) for x in cols["success"]], cols["reason"])
    h.seed(since, rows)


def digest(e):
    return {k: v for k, v in e.state_digest().items() if "buckets" not in k}


def check(engines, hists, status, start, end, lo=LO, hi=HI, seg_cap=256):
    """The call against the restatement, bit for bit, and its transfers."""
    got = engine.state_history_stats(engines, status_code(status), start, end, lo, hi, seg_cap=seg_cap)
    segs, lc, lm = Hr.answer(hists, status, start, end, lo, hi)
    assert len(got["kind"]) == len(segs)
    for d, w in enumerate(segs):
        assert (int(got["kind"][d]), int(got["user"][d]), int(got["reason"][d]), int(got["count"][d])) == w[:4], d
        assert [bits(x) for x in got["total"][d]] == [bits(x) for x in w[4]], (d, w)
        assert [[bits(x) for x in m] for m in got["pct"][d]] == [[bits(x) for x in m] for m in w[5]], (d, w)
    for g, w in ((got["leaders_cpu"], lc), (got["leaders_mem"], lm)):
        assert [(u, bits(t)) for u, t in g] == [(u, bits(t)) for u, t in w]
    s = got["stats"]
    H = sum(1 for h in hists if h.rows)
    assert s["h2d_bytes"] == 0
    if len(segs) <= seg_cap:
        assert s["d2h_bytes"] == Hr.d2h_bytes(H, segs, lc, bool(segs))
    if not H:
        assert s["n_launches"] == 0
    return got


class Pools:
    """Resident handles, a mirror of their running rows {task id: row} (with the reason fact) and pending rows, and
    each handle's history restated (history_ref.History)."""

    def __init__(self, names):
        self.e = [engine.GpuEngine(pool_name=f"hs-{n}") for n in names]
        self.run = [{} for _ in names]
        self.pend = [{} for _ in names]
        self.h = [Hr.History() for _ in names]

    def close(self):
        for e in self.e:
            e.close()

    def apply(self, p, up=(), run_up=(), run_rm=()):
        up, run_up = list(up), list(run_up)
        self.e[p].state_apply(M.delta(up=[(r["job_id"], r) for r in up], run_up=run_up, run_rm=run_rm, drop=DROP,
                                      lists=True))
        for t in run_rm:
            del self.run[p][t]
        self.pend[p].update((r["job_id"], r) for r in up)
        self.run[p].update((r["task_id"], dict(r, reason=-1)) for r in run_up)

    def launch(self, p, jobs, tids, starts):
        self.e[p].state_launch(jobs, tids, starts)
        for j, t, s in zip(jobs, tids, starts):
            r = self.pend[p].pop(j)
            self.run[p][t] = dict(task_id=t, job_id=j, user=r["user"], priority=r["priority"], start_time=s,
                                  cpus=r["cpus"], mem=r["mem"], gpus=r.get("gpus", 0.0), groups=list(r["groups"]),
                                  reason=-1)

    def reason(self, p, tids, codes):
        self.e[p].state_task_reason(tids, codes)
        for t, c in zip(tids, codes):
            self.run[p][t]["reason"] = int(c)

    def finish(self, p, tids, end, success, reason=None):
        self.e[p].state_finish_history(tids, end, success, reason)
        self.h[p].finish(self.run[p], tids, end, success, reason)
        for t in tids:
            del self.run[p][t]

    def advance(self, p, since):
        self.e[p].state_history_advance(since)
        self.h[p].advance(since)

    def check(self, status, start, end, lo=LO, hi=HI, idx=None):
        idx = list(range(len(self.e))) if idx is None else idx
        return check([self.e[k] for k in idx], [self.h[k] for k in idx], status, start, end, lo, hi)


# ---- the golden scenarios on resident handles ---------------------------------------------------------------------
def edge_pools():
    h = GOLDEN["edges"]["handles"]
    ps = Pools(["a", "b", "c"])
    for p, k in enumerate(("a", "b", "c")):
        seed(ps.e[p], ps.h[p], GOLDEN["since"], h[k])
    return ps


def test_golden_edges():
    ps = edge_pools()
    try:
        for case in GOLDEN["edges"]["cases"]:
            q = case["request"]
            ps.check(q["status"], q["start"], q["end"], q["lo"], q["hi"])
            a = engine.state_history_stats(ps.e, status_code(q["status"]), q["start"], q["end"], q["lo"], q["hi"])
            got = cycle.instance_stats_response(a, user_name=str, reason_string=REASONS.get)
            assert plain(got) == case["want"]
            for m in ("cpu-seconds", "mem-seconds"):
                assert list(got["leaders"][m].items()) == list(case["want"]["leaders"][m].items())
        # one handle, and the handles in another order: the fold order is (task id, pool index, position)
        s0 = GOLDEN["since"]
        for idx in ([0], [1], [2, 1, 0], [1, 0]):
            for status in (Hr.SUCCESS, Hr.FAILED):
                ps.check(status, s0, s0 + 10 ** 8, idx=idx)
    finally:
        ps.close()


@pytest.mark.parametrize("k", range(len(GOLDEN["transcribed"])))
def test_golden_transcribed(k):
    t = GOLDEN["transcribed"][k]
    q = t["request"]
    ps = Pools(["t"])
    try:
        seed(ps.e[0], ps.h[0], t["since"], t["rows"])
        ps.check(q["status"], q["start"], q["end"])
        r = cycle.instance_stats_response(engine.state_history_stats(ps.e, status_code(q["status"]), q["start"],
                                                                     q["end"]), user_name=str,
                                          reason_string=REASONS.get)
        key = t["reason"]
        assert r["overall"]["count"] == r["by-reason"][key]["count"] == \
            r["by-user-and-reason"][str(t["user"])][key]["count"] == t["count"]
        for m, chk in t["checks"].items():
            assert plain(r["overall"][m]["percentiles"]) == chk["percentiles"]
            assert r["overall"][m]["total"] == pytest.approx(chk["total_approx"], abs=1e-7)
    finally:
        ps.close()


def test_golden_ops():
    """The table's seed, finish (both reason paths, a row one ms before the horizon) and advance on a handle."""
    ops = GOLDEN["ops"]
    ps = Pools(["o"])
    try:
        run = [dict(task_id=int(t), job_id=int(t) + 10 ** 6, priority=50, gpus=0.0, groups=[], **r)
               for t, r in ops["running"].items()]
        ps.apply(0, run_up=[{k: v for k, v in r.items() if k != "reason"} for r in run])
        ps.reason(0, [r["task_id"] for r in run if r["reason"] != -1], [r["reason"] for r in run if r["reason"] != -1])
        for s in ops["steps"]:
            if s["op"] == "seed":
                seed(ps.e[0], ps.h[0], s["since"], s["rows"])
            elif s["op"] == "finish":
                ps.finish(0, s["task_id"], s["end"], s["success"], s["reason"])
            else:
                ps.advance(0, s["since"])
            assert [[r["task_id"], r["reason"], int(r["success"])] for r in ps.h[0].rows] == s["want"]
            for status in (Hr.SUCCESS, Hr.FAILED):
                ps.check(status, ps.h[0].since, ps.h[0].since + 10 ** 6)
    finally:
        ps.close()


# ---- a churn past one sort tile -----------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["grid", "off"])
def test_churn(regime):
    rng = np.random.default_rng(31 if regime == "grid" else 32)
    ps = Pools(["a", "b", "c"])
    U_ = 14
    next_job, next_tid, now = [1], [10 ** 6], [M.START]
    since0 = M.START - 10 ** 6

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

    def ends(p, ts):
        return [ps.run[p][t]["start_time"] + (1000 * int(rng.integers(0, 90)) if regime == "grid"
                                              else int(rng.integers(0, 90000))) for t in ts]

    try:
        for p in range(3):
            seed(ps.e[p], ps.h[p], since0, [])
            ps.apply(p, up=new_pending(9000 if p == 0 else 800))
        for batch in range(4):
            for p in range(3):
                pend = sorted(ps.pend[p])
                go = [int(j) for j in rng.choice(pend, min(len(pend), 3000 if batch < 2 and p == 0 else 150),
                                                 replace=False)]
                t = tids(len(go))
                rng.shuffle(t)
                now[0] += 60000
                ps.launch(p, go, t, [start() for _ in go])
                run = list(ps.run[p].values())
                extra = [dict(r, task_id=tid, start_time=start())
                         for r, tid in zip([run[k] for k in rng.choice(len(run), 40, replace=False)], tids(40))]
                ps.apply(p, run_up=extra)
                live = sorted(ps.run[p])
                rs = [int(x) for x in rng.choice(live, len(live) // 5, replace=False)]
                ps.reason(p, rs, [int(c) for c in rng.choice([-1, 1001, 1002, 2003], len(rs))])
                live = sorted(ps.run[p])
                fin = [int(x) for x in rng.choice(live, min(len(live), 2500 if p == 0 and batch < 2 else 120),
                                                  replace=False)]
                half = len(fin) // 2
                for part, with_reason in ((fin[:half], False), (fin[half:], True)):
                    ok = [int(x) for x in rng.integers(0, 2, len(part))]
                    rc = [int(c) for c in rng.choice([-1, 3001, 1001], len(part))] if with_reason else None
                    ps.finish(p, part, ends(p, part), ok, rc)
            if batch == 2:   # an advance on every handle past the first batch's rows
                for p in range(3):
                    ps.advance(p, M.START + 200000)
            # the same task id in a second handle's history
            if batch == 1:
                r0 = ps.h[0].rows[0]
                ps.e[1].state_history_seed(ps.h[1].since, *[[r[k] if k != "success" else int(r[k])
                                                             for r in ps.h[1].rows + [r0]] for k in COLS])
                ps.h[1].seed(ps.h[1].since, ps.h[1].rows + [dict(r0)])
            sel = sum(1 for h in ps.h for r in h.rows if r["success"])
            assert sel > 2048 or batch != 1   # past one tile before the advance
            s0 = max(h.since for h in ps.h)
            lo_tid = 10 ** 6 + 3000
            for status in (Hr.SUCCESS, Hr.FAILED):
                ps.check(status, s0, now[0] + 1)
                ps.check(status, now[0] - 90000, now[0] - 20000, lo_tid, next_tid[0] - 500)
            ps.check(Hr.SUCCESS, s0, now[0] + 1, idx=[2, 0])
    finally:
        ps.close()


# ---- nothing else changes -----------------------------------------------------------------------------------------
def test_twin_finish_changes_nothing_else():
    """Two handles with the same rows: one finishes with cook_state_finish, the other (history on) with
    cook_state_finish_history.  Every other answer is the twin's."""
    t = M.c2(5)
    pend, run = M.pool_rows(t)
    twins = [M.Pool.of_trace(t, name=f"hs-twin-{k}") for k in range(2)]
    try:
        for p in twins:
            p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
        a, b = twins
        b.gpu.state_history_seed(0)
        ids = sorted(run)[::3]
        end = [run[i]["start_time"] + 5000 for i in ids]
        ok = [k % 2 for k in range(len(ids))]
        a.gpu.state_finish(ids, end, ok)
        b.gpu.state_finish_history(ids, end, ok, None)
        for p in twins:
            p.rank()
        now = M.START + 10 ** 9
        assert digest(a.gpu) == digest(b.gpu)
        copies = [engine.GpuEngine(pool_name=f"hs-copy-{k}") for k in range(2)]   # the exports, as copies
        try:
            for c, p in zip(copies, twins):
                c.state_apply(abi.make_delta(reset=True, **p.gpu.state_export()))
            for x, y in ((a.gpu, b.gpu), (copies[0], copies[1])):
                dx, dy = x.state_digest(64), y.state_digest(64)
                assert set(dx) == set(dy) and all(np.array_equal(dx[k], dy[k]) for k in dx)
        finally:
            for c in copies:
                c.close()
        assert np.array_equal(a.gpu.state_queue(), b.gpu.state_queue())
        sa = engine.state_sweep([a.gpu], now, 1000, 10 ** 9)
        sb = engine.state_sweep([b.gpu], now, 1000, 10 ** 9)
        for k in ("linger", "cancel", "straggler"):
            assert sa[k] == sb[k], k
        ua, ub = engine.state_user_usage([a.gpu], None, True, True), engine.state_user_usage([b.gpu], None, True, True)
        for k in ua:
            if k != "stats":
                x, y = ua[k], ub[k]
                assert np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y, k
        ia = engine.state_instance_stats([a.gpu], now, abi.IS_RUNNING, 0, now)
        ib = engine.state_instance_stats([b.gpu], now, abi.IS_RUNNING, 0, now)
        for k in ("kind", "user", "reason", "count", "total", "pct"):
            assert np.array_equal(ia[k], ib[k]), k
        assert ia["leaders_cpu"] == ib["leaders_cpu"] and ia["leaders_mem"] == ib["leaders_mem"]
        ga = a.gpu.state_match(a.offers, a.users, a.params, max_ports=a.max_ports, derived=True)
        gb = b.gpu.state_match(b.offers, b.users, b.params, max_ports=b.max_ports, derived=True)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ga[k], gb[k]), k
        # the history holds exactly the finished rows
        got = engine.state_history_stats([b.gpu], abi.IS_SUCCESS, 0, now)
        got_f = engine.state_history_stats([b.gpu], abi.IS_FAILED, 0, now)
        n = lambda g: int(g["count"][0]) if len(g["kind"]) else 0
        assert n(got) + n(got_f) == len(ids)
        # a's history is off
        with pytest.raises(CookError):
            engine.state_history_stats([a.gpu], abi.IS_SUCCESS, 0, now)
    finally:
        for p in twins:
            p.close()


def test_seed_round_trip():
    """A fresh handle seeded with the restatement's rows at the same horizon answers identically."""
    ps = edge_pools()
    fresh = engine.GpuEngine(pool_name="hs-fresh")
    try:
        rows = [r for h in ps.h[:1] for r in h.rows]
        h = Hr.History()
        seed(fresh, h, ps.h[0].since, rows)
        for status in (Hr.SUCCESS, Hr.FAILED):
            a = engine.state_history_stats([ps.e[0]], status_code(status), ps.h[0].since, ps.h[0].since + 10 ** 8)
            b = check([fresh], [h], status, ps.h[0].since, ps.h[0].since + 10 ** 8)
            for k in ("kind", "user", "reason", "count"):
                assert np.array_equal(a[k], b[k])
            assert [bits(x) for x in a["total"].ravel()] == [bits(x) for x in b["total"].ravel()]
            assert [bits(x) for x in a["pct"].ravel()] == [bits(x) for x in b["pct"].ravel()]
    finally:
        fresh.close()
        ps.close()


# ---- the horizon rules, the reset, seg_cap ------------------------------------------------------------------------
def test_horizon_and_reset():
    ps = Pools(["h"])
    e = ps.e[0]
    s0 = M.START
    try:
        with pytest.raises(CookError):     # off until seeded
            engine.state_history_stats([e], abi.IS_SUCCESS, s0, s0 + 1)
        with pytest.raises(CookError):
            e.state_history_advance(s0)
        seed(e, ps.h[0], s0, [])
        a = check([e], ps.h, Hr.SUCCESS, s0, s0 + 1)   # n = 0: an empty history at that horizon
        assert len(a["kind"]) == 0 and a["stats"]["n_launches"] == 0
        rows = [dict(task_id=10 + k, job_id=100 + k, user=k % 3, priority=50, start_time=s0 - 1 + k, cpus=1.0,
                     mem=8.0, gpus=0.0, groups=[]) for k in range(4)]
        ps.apply(0, run_up=rows)
        ps.finish(0, [10, 11, 12], [s0 + 100, s0 + 100, s0 + 100], [1, 1, 0])
        assert [r["task_id"] for r in ps.h[0].rows] == [11, 12]   # 10 started one ms before the horizon
        check([e], ps.h, Hr.SUCCESS, s0, s0 + 10)
        with pytest.raises(CookError):     # a window before the horizon is refused
            engine.state_history_stats([e], abi.IS_SUCCESS, s0 - 1, s0 + 10)
        with pytest.raises(CookError):     # an advance backwards
            e.state_history_advance(s0 - 1)
        ps.advance(0, s0 + 1)              # drops exactly 11
        assert [r["task_id"] for r in ps.h[0].rows] == [12]
        assert e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 0
        assert e.last_stats(abi.PHASE_STATE)["d2h_bytes"] == 4
        check([e], ps.h, Hr.FAILED, s0 + 1, s0 + 10)
        ps.advance(0, s0 + 1)              # the same horizon: nothing to drop, nothing transferred
        assert e.last_stats(abi.PHASE_STATE)["d2h_bytes"] == 0
        # a reset empties the history and turns it off; a finish then keeps nothing
        e.state_apply(M.delta(reset=True, drop=DROP))
        ps.run[0].clear()
        ps.h[0].reset()
        with pytest.raises(CookError):
            engine.state_history_stats([e], abi.IS_FAILED, s0, s0 + 10)
        with pytest.raises(CookError):
            e.state_history_advance(s0 + 2)
        ps.apply(0, run_up=rows[3:])
        ps.finish(0, [13], [s0 + 100], [1])
        seed(e, ps.h[0], s0, [])
        check([e], ps.h, Hr.SUCCESS, s0, s0 + 10)
        assert ps.h[0].rows == []
    finally:
        ps.close()


def test_seg_cap_retry():
    ps = edge_pools()
    lib = ps.e[0].lib
    try:
        s0 = GOLDEN["since"]
        segs, _, _ = Hr.answer(ps.h, Hr.FAILED, s0, s0 + 10 ** 8)
        need = len(segs)
        cap = need - 1
        outs = [np.full(cap, 7, np.int32), np.full(cap, 7, np.int32), np.full(cap, 7, np.int32),
                np.full(cap, 7, np.int64), np.full(3 * cap, 7.0), np.full(15 * cap, 7.0),
                np.full(20, 7, np.int32), np.full(20, 7.0)]
        types = [abi.P_I32, abi.P_I32, abi.P_I32, abi.P_I64, abi.P_F64, abi.P_F64, abi.P_I32, abi.P_F64]
        n = [C.c_int32(-5), C.c_int32(-5)]
        st = abi.PhaseStats()
        st.n_launches = -5
        hs = (C.c_void_p * 3)(*[e.pool for e in ps.e])
        rc = lib.cook_state_history_stats(hs, 3, abi.IS_FAILED, s0, s0 + 10 ** 8, LO, HI, cap,
                                          *[abi.ptr(o, t) for o, t in zip(outs, types)], C.byref(n[0]),
                                          C.byref(n[1]), C.byref(st))
        assert rc == abi.COOK_E_TOO_LARGE
        assert n[0].value == need and n[1].value == -5 and st.n_launches == -5
        for x in outs:
            assert (x == 7).all()
        # engine.state_history_stats retries with the count; check() with a small first capacity
        check(ps.e, ps.h, Hr.FAILED, s0, s0 + 10 ** 8, seg_cap=1)
        check(ps.e, ps.h, Hr.FAILED, s0, s0 + 10 ** 8, seg_cap=need)
    finally:
        ps.close()


# ---- errors and transfers -----------------------------------------------------------------------------------------
def test_badargs_leave_the_digest():
    ps = edge_pools()
    e = ps.e[0]
    lib = e.lib
    s0 = GOLDEN["since"]
    try:
        rows = [dict(task_id=900 + k, job_id=9000 + k, user=1, priority=50, start_time=s0 + 1000 * k, cpus=1.0,
                     mem=8.0, gpus=0.0, groups=[]) for k in range(3)]
        ps.apply(0, run_up=rows)
        before = [digest(x) for x in ps.e]
        answers = lambda: [engine.state_history_stats(ps.e, c, s0, s0 + 10 ** 8) for c in (abi.IS_SUCCESS, abi.IS_FAILED)]
        a0 = answers()
        bad = abi.COOK_E_BADARG
        # finish_history: finish's cases, then its own
        for args in (([900, 900], [s0 + 5000] * 2, [1, 1], None),          # task id twice
                     ([999], [s0 + 5000], [1], None),                       # not live
                     ([901], [s0 + 999], [0], None),                        # a failed row that ends before its start
                     ([900], [s0 + 5000], [1], [-2])):                      # a reason below -1
            with pytest.raises(CookError):
                e.state_finish_history(*args)
        i64 = lambda *v: abi.ptr(np.array(v, np.int64), abi.P_I64)
        assert lib.cook_state_finish_history(e.pool, -1, None, None, None, None) == bad
        assert lib.cook_state_finish_history(e.pool, 1, i64(900), None, abi.ptr(np.ones(1, np.uint8), abi.P_U8),
                                             None) == bad
        assert lib.cook_state_finish_history(e.pool, 1, i64(900), i64(s0 + 5000), None, None) == bad
        # seed
        ok = dict(task_id=[1], user=[0], start_ms=[s0], end_ms=[s0 + 1], cpus=[1.0], mem=[1.0], success=[1],
                  reason_code=[-1])
        for over in (dict(start_ms=[s0 - 1], end_ms=[s0]), dict(end_ms=[s0 - 1]), dict(user=[-1]),
                     dict(reason_code=[-2]), dict(cpus=[-1.0]), dict(cpus=[-0.0]), dict(mem=[float("nan")]),
                     dict(mem=[float("inf")]), dict(task_id=[900]),
                     dict(task_id=[1, 1], user=[0, 0], start_ms=[s0] * 2, end_ms=[s0 + 1] * 2, cpus=[1.0] * 2,
                          mem=[1.0] * 2, success=[1, 1], reason_code=[-1, -1])):
            with pytest.raises(CookError):
                e.state_history_seed(s0, **{**ok, **over})
        assert lib.cook_state_history_seed(e.pool, s0, -1, *([None] * 8)) == bad
        assert lib.cook_state_history_seed(e.pool, s0, 1, i64(1), *([None] * 7)) == bad
        # stats
        cap = 64
        outs = [np.full(cap, 7, np.int32), np.full(cap, 7, np.int32), np.full(cap, 7, np.int32),
                np.full(cap, 7, np.int64), np.full(3 * cap, 7.0), np.full(15 * cap, 7.0),
                np.full(20, 7, np.int32), np.full(20, 7.0)]
        types = [abi.P_I32, abi.P_I32, abi.P_I32, abi.P_I64, abi.P_F64, abi.P_F64, abi.P_I32, abi.P_F64]
        op = [abi.ptr(o, t) for o, t in zip(outs, types)]
        n = [C.c_int32(7), C.c_int32(7)]
        h = [x.pool for x in ps.e]

        def call(handles, status=abi.IS_SUCCESS, start=s0, end=s0 + 10 ** 8, seg_cap=cap, o=None, cnt=None):
            hs = (C.c_void_p * len(handles))(*handles)
            return lib.cook_state_history_stats(hs, len(handles), status, start, end, LO, HI, seg_cap, *(o or op),
                                                *(cnt or [C.byref(n[0]), C.byref(n[1])]), None)

        assert call([h[0], h[1], h[0]]) == bad
        assert call([h[0], None]) == bad
        for st_ in (abi.IS_RUNNING, abi.IS_UNKNOWN, 4, -1):
            assert call(h, status=st_) == bad
        assert call(h, start=s0 + 5, end=s0 + 5) == bad
        assert call(h, start=s0 - 1) == bad                         # before the horizon
        assert call(h, seg_cap=-1) == bad
        for k in range(8):
            o = list(op)
            o[k] = None
            assert call(h, o=o) == bad
        assert call(h, cnt=[None, C.byref(n[1])]) == bad
        assert call(h, cnt=[C.byref(n[0]), None]) == bad
        # cook_state_instance_stats still refuses the two statuses
        R = sum(len(r) for r in ps.run)
        hs = (C.c_void_p * 3)(*h)
        assert lib.cook_state_instance_stats(hs, 3, s0 + 10 ** 6, abi.IS_SUCCESS, 0, s0, LO, HI, 1 + 2 * R, *op,
                                             C.byref(n[0]), C.byref(n[1]), None) == bad
        for x in outs:
            assert (x == 7).all()
        assert n[0].value == n[1].value == 7
        assert [digest(x) for x in ps.e] == before
        a1 = answers()
        for x, y in zip(a0, a1):
            for k in ("kind", "user", "reason", "count", "total", "pct"):
                assert np.array_equal(x[k], y[k])
        # the transfers of a finish_history: cook_state_finish's 13 n, plus 4 n with reason codes and a row kept
        e.state_finish_history([900], [s0 + 5000], [1])
        assert e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 13
        e.state_finish_history([901, 902], [s0 + 5000] * 2, [0, 1], [3001, -1])
        assert e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 13 * 2 + 4 * 2
        # and of a seed: 49 B per row
        e.state_history_seed(s0, **ok)
        assert e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 49
        e.state_history_seed(s0)
        assert e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 0
    finally:
        ps.close()
