"""The completed-job log on resident handles (cook_state_completed_seed / _record / _advance) and its listing
(cook_state_list_completed): the golden scenarios replayed, mixed-state queries answered with cook_state_list_jobs
through cycle.list_jobs_response; a churn over three handles past one sort tile checked bit for bit against
completed_ref after every batch; a seed round trip; the horizon, reset and off-log refusals; the cap retry; the
BADARGs; the transfer formulas; and that nothing else changes."""
import ctypes as C

import numpy as np
import pytest

import completed_ref as CR
import list_ref as L
import resident_model as M
import test_list_completed_reference as R
import test_list_jobs_reference as LJ
from cook_b200 import abi, cycle, engine
from cook_b200.engine import CookError, GpuEngine
from test_state_list_jobs import device_entries, facts, upsert

pytestmark = pytest.mark.gpu

START = M.START
MAXI = (1 << 31) - 1
LO, HI = -(1 << 63), (1 << 63) - 1
STATES = (CR.L_SUCCESS, CR.L_FAILED, CR.L_COMPLETED)


def cols(rows):
    """Records -> the seven columns of state_completed_seed / _record."""
    rows = [tuple(r) for r in rows]
    return [[r[c] for r in rows] for c in range(7)]


def seed(e, lg, since, rows):
    e.state_completed_seed(since, *cols(rows))
    lg.update(CR.seed(since, rows))


def record(e, lg, rows):
    e.state_completed_record(*cols(rows))
    CR.record(lg, rows)


def ask(es, q, state):
    a = engine.state_list_completed(es, q["user"], state, q["start"], q["end"], q["lo"], q["hi"], q["pool"],
                                    q["handle_pool"] if q["pool"] != -1 else None, q["include_custom_executor"],
                                    q["limit"])
    return [(int(j), int(t), int(p)) for j, t, p in zip(a["job_id"], a["submit_ms"], a["pool"])], a


def bad(fn, *a, code=abi.COOK_E_BADARG, **k):
    with pytest.raises(CookError) as ei:
        fn(*a, **k)
    assert ei.value.code == code


# ---- the golden scenarios -------------------------------------------------------------------------------------
@pytest.mark.parametrize("scenario", R.GOLDEN["scenarios"], ids=[s["name"] for s in R.GOLDEN["scenarios"]])
def test_golden(scenario):
    es, lgs = [], R.logs(scenario)
    try:
        for k, h in enumerate(scenario["handles"]):
            e = GpuEngine(pool_name=f"lc{k}")
            es.append(e)
            if h["pending"]:
                upsert(e, [(j, u) for u, j, _ in h["pending"]])
                facts(e, [(j, tuple(f)) for _, j, f in h["pending"]])
            e.state_completed_seed(h["since"], *cols(h["seed"]))
            for b in h["record"]:
                e.state_completed_record(*cols(b))
        for qd in scenario["queries"]:
            q, done = R.query(scenario, qd)
            if qd.get("refused"):
                for s in done:
                    bad(ask, es, q, CR.NAMES[s])
                continue
            completed = {}
            for s in done:
                got, _ = ask(es, q, CR.NAMES[s])
                assert got == CR.list_completed(lgs, q, CR.NAMES[s])
                completed[s] = [(j, t) for j, t, _ in got]
            ans = {"state": [], "job_id": [], "submit_ms": [], "pool": []}
            if q["states"]:
                ans = engine.state_list_jobs(es, q["user"], q["states"], q["start"], q["end"], q["lo"], q["hi"],
                                             q["pool"], q["handle_pool"] if q["pool"] != -1 else None,
                                             q["include_custom_executor"], q["limit"])
                assert device_entries(ans) == L.list_jobs(R.active_rows(scenario), q)[0]
            got = cycle.list_jobs_response(ans, states=qd["states"], limit=qd["limit"], completed=completed)
            LJ.check(qd, got, None)
    finally:
        for e in es:
            e.close()


# ---- a churn over three handles -------------------------------------------------------------------------------
def check_all(es, lgs, rng, U, hp, jid_hi, n_queries=6):
    horizon = max(lg["since"] for lg in lgs)
    for _ in range(n_queries):
        a, b = sorted(rng.integers(horizon, horizon + 40_000, 2).tolist())
        lo, hi = sorted(rng.integers(0, jid_hi + 100, 2).tolist())
        if rng.random() < 0.4:
            lo, hi = LO, HI
        q = L.query(int(rng.choice(U, p=[0.85, 0.1, 0.05])), 0, a, b + 1, lo, hi, int(rng.integers(-1, 4)), hp,
                    bool(rng.integers(2)), int(rng.choice([0, 1, 150, MAXI, int(rng.integers(1, 4000))])))
        for s in STATES:
            got, _ = ask(es, q, s)
            assert got == CR.list_completed(lgs, q, s), (q, s)


def test_churn_against_the_restatement():
    rng = np.random.default_rng(11)
    H, U = 3, 3
    hp = [0, 1, 2]
    es = [GpuEngine(pool_name=f"lc-churn{k}") for k in range(H)]
    lgs = [{} for _ in range(H)]
    since = START
    stamp = [100]
    jobs = {}    # job id -> (user, submit, spool, exec)
    try:
        for e, lg in zip(es, lgs):
            seed(e, lg, since, [])
        next_jid = 1
        for batch in range(10):
            for k, (e, lg) in enumerate(zip(es, lgs)):
                stamp[0] += 1
                rows, seen = [], set()
                # new completions (the first batch past one sort tile for user 0 over the handles)
                for _ in range(1500 if batch == 0 else 300):
                    j = next_jid
                    next_jid += 1
                    jobs[j] = (int(rng.choice(U, p=[0.85, 0.1, 0.05])), int(since + rng.integers(-50, 40_000)),
                               int(rng.integers(-1, 3)), int(rng.integers(-1, 2)))
                    u, sub, sp, ex = jobs[j]
                    rows.append((j, stamp[0], u, sub, sp, ex, int(rng.choice([CR.SUCCESS, CR.FAILED]))))
                    seen.add(j)
                # reopens, success flips and moves of older jobs, some stamped late or equal; exact re-sends
                for j in (rng.choice(next_jid - 1, min(200, next_jid - 1), replace=False) + 1).tolist():
                    if j in seen:
                        continue
                    seen.add(j)
                    u, sub, sp, ex = jobs[j]
                    kind = int(rng.choice([CR.SUCCESS, CR.FAILED, CR.REOPENED]))
                    st = stamp[0] if rng.random() < 0.8 else stamp[0] - int(rng.integers(1, 5))   # some late, some equal
                    rows.append((j, st, u, sub, sp, ex, kind))
                for i in rng.choice(len(lg["rows"]), min(20, len(lg["rows"])), replace=False).tolist():
                    if lg["rows"][i][0] not in seen:
                        seen.add(lg["rows"][i][0])
                        rows.append(lg["rows"][i])
                perm = rng.permutation(len(rows))
                record(e, lg, [rows[i] for i in perm])
            if batch % 3 == 2:
                since += 2000
                for e, lg in zip(es, lgs):
                    e.state_completed_advance(since)
                    CR.advance(lg, since)
            assert sum(sum(1 for r in lg["rows"] if r[2] == 0) for lg in lgs) > 2048   # past one sort tile
            check_all(es, lgs, rng, U, hp, next_jid)
    finally:
        for e in es:
            e.close()


def test_seed_round_trip():
    """Handles seeded with the restatement's rows answer the same as the ones built by record calls."""
    rng = np.random.default_rng(3)
    a, b = [GpuEngine(pool_name=f"rt-a{k}") for k in range(2)], [GpuEngine(pool_name=f"rt-b{k}") for k in range(2)]
    la, lb = [{}, {}], [{}, {}]
    try:
        for k in range(2):
            seed(a[k], la[k], START, [])
            for t in range(4):
                # a job's user, submit time and executor are fixed; its kind and stamp change
                rows = [(int(j), 10 * t + k, int(j % 2), int(START - 5 + (j * 7919) % 5005), -1, int(j % 3 - 1),
                         int(rng.integers(1, 4))) for j in rng.choice(3000, 700, replace=False)]
                record(a[k], la[k], rows)
            a[k].state_completed_advance(START + 100)
            CR.advance(la[k], START + 100)
            latest = {}   # one record per job, as a seed read from one database value holds
            for r in la[k]["rows"]:
                if r[0] not in latest or r[1] >= latest[r[0]][1]:
                    latest[r[0]] = r
            seed(b[k], lb[k], START + 100, [latest[j] for j in sorted(latest)])
        for _ in range(8):
            q = L.query(int(rng.integers(2)), 0, START + 100, START + int(rng.integers(200, 6000)),
                        limit=int(rng.choice([1, 150, MAXI])), include_custom_executor=bool(rng.integers(2)))
            for s in STATES:
                assert ask(a, q, s)[0] == ask(b, q, s)[0] == CR.list_completed(la, q, s) == CR.list_completed(lb, q, s)
    finally:
        for e in a + b:
            e.close()


# ---- refusals, retries, arguments, transfers --------------------------------------------------------------------
REC = (5, 1, 0, START + 10, -1, 0, CR.SUCCESS)


def raw(es, user=0, state=CR.L_COMPLETED, start=START, pool=-1, handle_pool=None, inc=1, limit=MAXI, cap=64,
        outs=True):
    handles = (C.c_void_p * len(es))(*[e.pool if e is not None else None for e in es])
    m = max(cap, 1)
    jid, sub, pi = np.zeros(m, np.int64), np.zeros(m, np.int64), np.zeros(m, np.int32)
    n = C.c_int32(-5)
    hp = np.ascontiguousarray(handle_pool, np.int32) if handle_pool is not None else None
    st = abi.PhaseStats()
    rc = es[0].lib.cook_state_list_completed(handles, len(es), user, state, start, START + 10_000, LO, HI, pool,
                                             abi.ptr(hp, abi.P_I32) if hp is not None else None, inc, limit, cap,
                                             abi.ptr(jid, abi.P_I64) if outs else None, abi.ptr(sub, abi.P_I64),
                                             abi.ptr(pi, abi.P_I32), C.byref(n), C.byref(st))
    return rc, n.value, st.as_dict()


def test_refusals_badargs_cap_and_transfers():
    a, b = GpuEngine(pool_name="lc-a"), GpuEngine(pool_name="lc-b")
    la, lb = {}, {}
    try:
        # off until seeded: every call but the seed is refused
        assert raw([a])[0] == abi.COOK_E_BADARG
        bad(a.state_completed_record, *cols([REC]))
        bad(a.state_completed_advance, START)
        # the seed's BADARGs, before any change
        for r in ((5, 1, 0, START - 1, -1, 0, 1), (5, 1, -1, START, -1, 0, 1), (5, -1, 0, START, -1, 0, 1),
                  (5, 1, 0, START, -1, 0, 0), (5, 1, 0, START, -1, 0, 4), (5, 1, 0, START, -1, 2, 1),
                  (5, 1, 0, START, -1, -2, 1), (5, 1, 0, START, -2, 0, 1)):
            bad(a.state_completed_seed, START, *cols([r]))
        bad(a.state_completed_seed, START, *cols([REC, REC]))
        assert a.lib.cook_state_completed_seed(a.pool, START, -1, *[None] * 7) == abi.COOK_E_BADARG
        assert a.lib.cook_state_completed_seed(a.pool, START, 1, *[None] * 7) == abi.COOK_E_BADARG
        assert raw([a])[0] == abi.COOK_E_BADARG   # still off
        # seed: 34 B per row
        rows = [(j, 1, j % 2, START + j, -1, 0, CR.SUCCESS if j % 3 else CR.FAILED) for j in range(1, 41)]
        seed(a, la, START, rows)
        assert a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 34 * 40
        seed(b, lb, START, [])
        assert b.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 0
        # record: 34 B per row kept; a row before the horizon is skipped; the row checks and a job id twice refused
        record(a, la, [(41, 2, 0, START - 1, -1, 0, 1), (42, 2, 0, START, -1, 0, 1), (3, 2, 1, START + 3, -1, 0, 3)])
        assert a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 34 * 2
        assert [r[0] for r in la["rows"][-2:]] == [42, 3]
        before = raw([a], cap=64)[:2]
        for r in ((7, 3, 0, START, -1, 0, 9), (7, -3, 0, START, -1, 0, 1), (7, 3, 0, START, -3, 0, 1)):
            bad(a.state_completed_record, *cols([r]))
        bad(a.state_completed_record, *cols([(7, 3, 0, START, -1, 0, 1), (7, 4, 0, START, -1, 0, 1)]))
        assert raw([a], cap=64)[:2] == before
        # listing BADARGs, nothing written
        for kw in (dict(state=0), dict(state=4), dict(user=-1), dict(pool=-2), dict(pool=0), dict(inc=2),
                   dict(limit=-1), dict(cap=-1), dict(outs=False), dict(start=START - 1)):
            assert raw([a, b], **kw)[:2] == (abi.COOK_E_BADARG, -5), kw
        assert raw([a, a])[0] == abi.COOK_E_BADARG
        assert raw([a, None])[0] == abi.COOK_E_BADARG
        # the cap: TOO_LARGE writes only the count; the engine retries once with it
        q = L.query(0, 0, START, START + 10_000)
        want = CR.list_completed([la, lb], dict(q, handle_pool=None), CR.L_COMPLETED)
        assert raw([a, b], cap=len(want))[:2] == (abi.COOK_OK, len(want))
        assert raw([a, b], cap=len(want) - 1)[:2] == (abi.COOK_E_TOO_LARGE, len(want))
        got, ans = ask([a, b], dict(q, handle_pool=None), CR.L_COMPLETED)
        got2 = engine.state_list_completed([a, b], 0, CR.L_COMPLETED, START, START + 10_000, cap=2)
        assert got == want and got2["job_id"].tolist() == [j for j, _, _ in want]
        # the listing: nothing up, 4 + 20 per entry down
        for s in STATES:
            st = raw([a, b], state=s)[2]
            n = len(CR.list_completed([la, lb], dict(q, handle_pool=None), s))
            assert st["h2d_bytes"] == 0 and st["d2h_bytes"] == 4 + 20 * n
        rc, n, st = raw([a, b], user=9)   # no record of the user: no device work
        assert (rc, n, st["n_launches"], st["d2h_bytes"]) == (abi.COOK_OK, 0, 0, 0)
        # advance: a 4 B download when rows may leave, nothing otherwise; backwards and off refused
        a.state_completed_advance(START + 20)
        CR.advance(la, START + 20)
        assert a.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 0 and a.last_stats(abi.PHASE_STATE)["d2h_bytes"] == 4
        a.state_completed_advance(START + 20)
        assert a.last_stats(abi.PHASE_STATE)["d2h_bytes"] == 0
        bad(a.state_completed_advance, START + 19)
        assert raw([a, b])[0] == abi.COOK_E_BADARG               # a's horizon is after start
        assert raw([a, b], start=START + 20)[1] == len(CR.list_completed([la, lb], dict(q, start=START + 20,
                                                                                        handle_pool=None), 3))
        # a reset empties the log and turns it off
        a.state_apply(M.delta(reset=True))
        assert raw([a], start=START + 20)[0] == abi.COOK_E_BADARG
        bad(a.state_completed_record, *cols([REC]))
        seed(a, la, START, [])
        assert raw([a])[:2] == (abi.COOK_OK, 0)
    finally:
        a.close()
        b.close()


# ---- nothing else changes -----------------------------------------------------------------------------------------
def digest(e):
    return {k: v for k, v in e.state_digest().items() if "buckets" not in k}


def test_twin_without_a_log_answers_the_same():
    """Two handles with the same rows; one also holds a completed-job log, fed and listed.  Every other answer is the
    twin's, and the listing changes nothing resident."""
    t = M.c2(5)
    pend, run = M.pool_rows(t)
    twins = [M.Pool.of_trace(t, name=f"lc-twin-{k}") for k in range(2)]
    try:
        for p in twins:
            p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
        a, b = twins
        ids = sorted(pend)
        for p in twins:
            p.gpu.state_list_facts(ids, [START + (j % 1000) for j in ids], [-1] * len(ids), [0] * len(ids))
        users = {j: r["user"] for j, r in pend.items()}
        b.gpu.state_completed_seed(START, *cols([(j, 1, users[j], START + (j % 1000), -1, 0, 1) for j in ids[::2]]))
        b.gpu.state_completed_record(*cols([(j, 2, users[j], START + (j % 1000), -1, 0, 3) for j in ids[::4]]))
        for p in twins:
            p.rank()
        d0 = digest(b.gpu)
        assert digest(a.gpu) == d0
        q0 = b.gpu.state_queue()
        lj = lambda e, u: device_entries(engine.state_list_jobs([e], u, 3, START, START + 1000))
        for u in sorted(set(users.values()))[:5]:
            for s in STATES:
                engine.state_list_completed([b.gpu], u, s, START, START + 1000)
            assert lj(a.gpu, u) == lj(b.gpu, u)
        assert digest(b.gpu) == d0
        assert np.array_equal(q0, b.gpu.state_queue()) and np.array_equal(a.gpu.state_queue(), q0)
        ga = a.gpu.state_match(a.offers, a.users, a.params, max_ports=a.max_ports, derived=True)
        gb = b.gpu.state_match(b.offers, b.users, b.params, max_ports=b.max_ports, derived=True)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ga[k], gb[k]), k
        with pytest.raises(CookError):   # a's log is off
            engine.state_list_completed([a.gpu], 0, CR.L_COMPLETED, START, START + 1000)
    finally:
        for p in twins:
            p.close()
