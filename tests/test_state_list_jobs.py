"""The job listing on resident handles (cook_state_list_facts, cook_state_list_jobs): the golden scenarios replayed,
a churn over three handles past one sort tile checked bit for bit against list_ref after every batch, the facts
through launch, requeue and upserts, the BADARGs, the TOO_LARGE retry, the transfer formulas, and that the call
changes nothing resident."""
import ctypes as C

import numpy as np
import pytest

import list_ref as L
import resident_model as M
import test_list_jobs_reference as R
from cook_b200 import abi, cycle, engine
from cook_b200.engine import CookError, GpuEngine

pytestmark = pytest.mark.gpu

START = M.START
MAXI = (1 << 31) - 1


def prow(user):
    return dict(M.DEFAULTS, user=user, priority=50, cpus=1.0, mem=1024.0, novel=[], attr=[], groups=[])


def rrow(user, jid, tid):
    return dict(user=user, priority=50, start_time=START, task_id=tid, job_id=jid, cpus=1.0, mem=1024.0, gpus=0.0,
                host=-1, groups=[])


def upsert(e, pend=(), run=()):
    """Pending upserts [(job id, user)] and running upserts [(task id, job id, user)] in one batch."""
    e.state_apply(M.delta(up=[(j, prow(u)) for j, u in pend], run_up=[rrow(u, j, t) for t, j, u in run]))


def facts(e, rows):
    """cook_state_list_facts of [(job id, (submit, pool, executor))]."""
    if rows:
        e.state_list_facts([j for j, _ in rows], [f[0] for _, f in rows], [f[1] for _, f in rows],
                           [f[2] for _, f in rows])


def bad(fn, *a, code=abi.COOK_E_BADARG, **k):
    with pytest.raises(CookError) as ei:
        fn(*a, **k)
    assert ei.value.code == code


def device_entries(ans):
    return [(int(s), int(j), int(t), int(p)) for s, j, t, p in
            zip(ans["state"], ans["job_id"], ans["submit_ms"], ans["pool"])]


def ask(engines, q):
    return engine.state_list_jobs(engines, q["user"], q["states"], q["start"], q["end"], q["lo"], q["hi"], q["pool"],
                                  q["handle_pool"] if q["pool"] != -1 else None, q["include_custom_executor"],
                                  q["limit"])


# ---- the golden scenarios -------------------------------------------------------------------------------------
def scenario_handles(scenario):
    """One engine per handle of the scenario, its rows and facts written as the shim would."""
    es = []
    for k, h in enumerate(scenario["handles"]):
        e = GpuEngine(pool_name=f"lj{k}")
        e.state_retry_config()
        pend = [(j, u) for u, j, _ in h["pending"]]
        run, parked, unknown = [], [], []
        for r in h["running"]:
            row, d = (r["row"], r) if isinstance(r, dict) else (r, {})
            if d.get("parked"):
                parked.append(row)
            else:
                run.append(row)
                if d.get("unknown"):
                    unknown.append(row[2])
        upsert(e, pend + [(j, u) for u, j, _, _ in parked], [(t, j, u) for u, j, t, _ in run])
        facts(e, [(j, tuple(f)) for _, j, f in h["pending"] if f])
        facts(e, sorted({(j, tuple(f)) for u, j, _, f in run if f}))
        facts(e, [(j, tuple(f)) for u, j, _, f in parked])
        if parked:   # a launch with retry facts parks the pending slot and copies the facts to the task
            e.state_retry_facts([j for _, j, _, _ in parked], [3] * len(parked), [0] * len(parked))
            e.state_launch([j for _, j, _, _ in parked], [t for _, _, t, _ in parked], [START] * len(parked))
        if unknown:
            e.state_task_facts(unknown, unknown=[1] * len(unknown))
        es.append(e)
    return es


@pytest.mark.parametrize("scenario", R.GOLDEN["scenarios"], ids=[s["name"] for s in R.GOLDEN["scenarios"]])
def test_golden(scenario):
    es = scenario_handles(scenario)
    try:
        for qd in scenario["queries"]:
            hs, q = R.ref_query(scenario, qd)
            if not q["states"]:
                continue
            ans = ask(es, q)
            want, missing = L.list_jobs(hs, q)
            assert device_entries(ans) == want
            assert ans["missing"] == missing
            got = cycle.list_jobs_response(ans, states=qd["states"], limit=qd["limit"],
                                           completed={k: [tuple(e) for e in v] for k, v in qd.get("completed", {}).items()},
                                           uncommitted=[tuple(e) for e in qd.get("uncommitted", [])])
            R.check(qd, got, ans["missing"])
    finally:
        for e in es:
            e.close()


# ---- a churn over three handles -------------------------------------------------------------------------------
class Model:
    """One handle's rows as list_ref sees them: pending {job id: (user, facts)}, running {task id: (user, job id,
    facts)}."""

    def __init__(self):
        self.pend, self.run = {}, {}

    def rows(self):
        return {"pending": [(u, j, f) for j, (u, f) in self.pend.items()],
                "running": [(u, j, t, f) for t, (u, j, f) in self.run.items()]}

    def set_facts(self, j, f):
        if j in self.pend:
            self.pend[j] = (self.pend[j][0], f)
        for t, (u, jj, _) in list(self.run.items()):
            if jj == j:
                self.run[t] = (u, j, f)


def random_facts(rng, n_pools):
    return (int(START + rng.integers(0, 10_000)), int(rng.integers(-1, n_pools + 1)), int(rng.integers(-1, 2)))


def test_churn_against_the_restatement():
    rng = np.random.default_rng(7)
    H, U, P = 3, 3, 4
    es = [GpuEngine(pool_name=f"churn{k}") for k in range(H)]
    ms = [Model() for _ in range(H)]
    hp = [0, 1, 2]
    next_jid, next_tid = [1000], [1]
    try:
        for batch in range(8):
            for e, m in zip(es, ms):
                # new pending jobs (some users heavy), replacements (facts cleared), removals
                n_new = 1500 if batch == 0 else 200
                new = [(next_jid[0] + i, int(rng.choice(U, p=[0.8, 0.15, 0.05]))) for i in range(n_new)]
                next_jid[0] += n_new
                old = list(m.pend)
                repl = [(j, m.pend[j][0]) for j in rng.choice(old, min(30, len(old)), replace=False).tolist()] if old else []
                rest = [j for j in old if j not in {r for r, _ in repl}]
                rm = rng.choice(rest, min(20, len(rest)), replace=False).tolist() if rest else []
                # running upserts: new tasks of new jobs (several per job), and a task re-upserted (facts cleared)
                run_new = []
                for i in range(100):
                    j, u = next_jid[0] + i, int(rng.integers(U))
                    for _ in range(int(rng.integers(1, 3))):
                        run_new.append((next_tid[0], j, u))
                        next_tid[0] += 1
                next_jid[0] += 100
                rerun = [(t, m.run[t][1], m.run[t][0]) for t in list(m.run)[:5]]
                e.state_apply(M.delta(up=[(j, prow(u)) for j, u in new + repl], rm=rm,
                                      run_up=[rrow(u, j, t) for t, j, u in run_new + rerun]))
                for j in rm:
                    del m.pend[j]
                for j, u in new + repl:
                    m.pend[j] = (u, None)
                for t, j, u in run_new + rerun:
                    m.run[t] = (u, j, None)
                # facts for most jobs, the three columns together
                jobs = sorted(set(m.pend) | {j for _, j, _ in m.run.values()})
                pick = [j for j in jobs if rng.random() < 0.9]
                fs = [(j, random_facts(rng, P)) for j in pick]
                facts(e, fs)
                for j, f in fs:
                    m.set_facts(j, f)
                # launches: the task takes the job's facts
                ready = list(m.pend)
                lj = rng.choice(ready, min(50, len(ready)), replace=False).tolist()
                tids = list(range(next_tid[0], next_tid[0] + len(lj)))
                next_tid[0] += len(lj)
                e.state_launch(lj, tids, [START] * len(lj))
                for j, t in zip(lj, tids):
                    u, f = m.pend.pop(j)
                    m.run[t] = (u, j, f)
            assert sum(sum(1 for u, _ in m.pend.values() if u == 0) for m in ms) > 2048   # past one sort tile
            rows = [m.rows() for m in ms]
            for _ in range(12):
                a, b = sorted(rng.integers(START - 100, START + 10_100, 2).tolist())
                lo, hi = sorted(rng.integers(900, next_jid[0] + 100, 2).tolist())
                if rng.random() < 0.4:
                    lo, hi = -(1 << 63), (1 << 63) - 1
                pool = int(rng.integers(-1, P))
                q = L.query(int(rng.integers(U)), int(rng.integers(1, 4)), a, b + 1, lo, hi, pool, hp,
                            bool(rng.integers(2)), int(rng.choice([0, 1, 150, MAXI, int(rng.integers(1, 3000))])))
                ans = ask(es, q)
                want, missing = L.list_jobs(rows, q)
                assert device_entries(ans) == want
                assert ans["missing"] == missing
    finally:
        for e in es:
            e.close()


# ---- the facts' life ------------------------------------------------------------------------------------------
def one(e, states=abi.LJ_WAITING | abi.LJ_RUNNING, user=0):
    ans = engine.state_list_jobs([e], user, states, START, START + 10_000)
    return device_entries(ans), ans["missing"]


def test_facts_survive_launch_and_requeue_and_upserts_clear_them():
    e = GpuEngine(pool_name="life")
    try:
        e.state_retry_config()
        upsert(e, [(1, 0), (2, 0), (3, 0)], [(50, 4, 0)])
        facts(e, [(1, (START + 1, -1, 0)), (2, (START + 2, -1, 0)), (3, (START + 3, -1, 0)), (4, (START + 4, -1, 0))])
        W, Rn = abi.LJ_WAITING, abi.LJ_RUNNING
        assert one(e) == ([(W, 1, START + 1, 0), (W, 2, START + 2, 0), (W, 3, START + 3, 0), (Rn, 4, START + 4, 0)], 0)
        # a NULL column is left unchanged
        e.state_list_facts([1], submit_ms=[START + 9])
        assert one(e, W)[0][0] == (W, 1, START + 9, 0)
        # launch: the task takes the facts; job 2 has retry facts, so its slot parks
        e.state_retry_facts([2], [3], [0])
        e.state_launch([1, 2], [60, 61], [START, START])
        assert one(e) == ([(W, 3, START + 3, 0), (Rn, 1, START + 9, 0), (Rn, 2, START + 2, 0), (Rn, 4, START + 4, 0)], 0)
        # a failure with retries left requeues job 2 in place: its facts stay
        out, _ = e.state_status([61], [0], [START + 100])
        assert out.tolist() == [abi.JOB_WAITING]
        assert one(e) == ([(W, 2, START + 2, 0), (W, 3, START + 3, 0), (Rn, 1, START + 9, 0), (Rn, 4, START + 4, 0)], 0)
        # upserts write "no facts": a pending replacement, a running re-upsert
        upsert(e, [(3, 0)], [(50, 4, 0)])
        assert one(e) == ([(W, 2, START + 2, 0), (Rn, 1, START + 9, 0)], 2)
    finally:
        e.close()


# ---- arguments, sizes, transfers ------------------------------------------------------------------------------
def raw_list(es, user=0, states=3, pool=-1, handle_pool=None, inc=1, limit=MAXI, cap=64, outs=True):
    handles = (C.c_void_p * len(es))(*[e.pool if e is not None else None for e in es])
    st, pi = np.zeros(max(cap, 1), np.int32), np.zeros(max(cap, 1), np.int32)
    jid, sub = np.zeros(max(cap, 1), np.int64), np.zeros(max(cap, 1), np.int64)
    n, miss = C.c_int32(-5), C.c_int32(-5)
    hp = np.ascontiguousarray(handle_pool, np.int32) if handle_pool is not None else None
    rc = es[0].lib.cook_state_list_jobs(handles, len(es), user, states, START, START + 10_000, -(1 << 63), (1 << 63) - 1,
                                        pool, abi.ptr(hp, abi.P_I32) if hp is not None else None, inc, limit, cap,
                                        abi.ptr(st, abi.P_I32) if outs else None, abi.ptr(jid, abi.P_I64),
                                        abi.ptr(sub, abi.P_I64), abi.ptr(pi, abi.P_I32), C.byref(n), C.byref(miss), None)
    return rc, n.value, miss.value


def test_badargs_too_large_transfers_and_no_change():
    a, b = GpuEngine(pool_name="a"), GpuEngine(pool_name="b")
    try:
        upsert(a, [(j, 0) for j in range(1, 11)] + [(99, 1)], [(100 + j, 20 + j, 0) for j in range(5)] +
               [(200, 20, 0)])
        upsert(b, [(5, 0)])
        lib = a.lib
        # ---- list facts
        bad(a.state_list_facts, [77], [START], [-1], [0])                 # not live
        bad(a.state_list_facts, [1, 1], [START] * 2, [-1] * 2, [0] * 2)   # twice
        bad(a.state_list_facts, [1], [START], [-1], [2])                  # executor outside {-1, 0, 1}
        bad(a.state_list_facts, [1], [START], [-1], [-2])
        bad(a.state_list_facts, [1], [START], [-2], [0])                  # submit pool below -1
        assert lib.cook_state_list_facts(a.pool, -1, None, None, None, None) == abi.COOK_E_BADARG
        assert lib.cook_state_list_facts(a.pool, 1, None, None, None, None) == abi.COOK_E_BADARG
        # uploads (P + R) * (4 + 8 + 4 + 1): job 20 has a running row twice over, job 1 a pending row
        facts(a, [(1, (START + 1, -1, 0)), (20, (START + 2, 0, 1))])
        assert a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == (1 + 2) * 17
        a.state_list_facts([1, 20], custom_executor=[0, 0])
        assert a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 3 * (4 + 1)
        facts(a, [(j, (START + j, -1, 0)) for j in range(2, 11)] + [(20 + j, (START + 20 + j, -1, 0)) for j in range(1, 5)])
        # ---- list jobs
        for kw in (dict(states=0), dict(states=4), dict(user=-1), dict(pool=-2), dict(pool=0), dict(inc=2),
                   dict(limit=-1), dict(cap=-1), dict(outs=False)):
            assert raw_list([a, b], **kw) == (abi.COOK_E_BADARG, -5, -5), kw
        assert raw_list([a, a])[0] == abi.COOK_E_BADARG
        assert raw_list([a, None])[0] == abi.COOK_E_BADARG
        # 10 waiting and 5 running entries; b's job 5 has no facts, so it is missing
        assert raw_list([a, b], cap=64)[1:] == (15, 1)
        assert raw_list([a, b], cap=4) == (abi.COOK_E_TOO_LARGE, 15, -5)
        assert raw_list([a, b], limit=3, cap=6)[:2] == (abi.COOK_OK, 6)
        assert raw_list([a, b], user=7) == (abi.COOK_OK, 0, 0)   # no row of the user: no device work
        digest = lambda e: {k: v for k, v in e.state_digest().items() if not k.endswith("_buckets")}
        d0 = (digest(a), digest(b))
        ans = engine.state_list_jobs([a, b], 0, 3, START, START + 10_000, cap=2)   # retried with the count
        assert len(ans["job_id"]) == 15 and ans["missing"] == 1
        assert ans["stats"]["h2d_bytes"] == 0 and ans["stats"]["d2h_bytes"] == 12 + 20 * 15
        assert (digest(a), digest(b)) == d0
        ans = engine.state_list_jobs([a, b], 7, 3, START, START + 10_000)
        assert ans["stats"]["n_launches"] == 0 and ans["stats"]["d2h_bytes"] == 0
        ans = engine.state_list_jobs([a, b], 0, abi.LJ_RUNNING, START, START + 10_000, pool_code=1, handle_pool=[0, 1])
        assert device_entries(ans) == []   # job 20's submit pool is 0, a's pool is 0, b holds none running
        ans = engine.state_list_jobs([a, b], 0, abi.LJ_RUNNING, START, START + 10_000, pool_code=0, handle_pool=[1, 2])
        assert [j for _, j, _, _ in device_entries(ans)] == [20]
    finally:
        a.close()
        b.close()
