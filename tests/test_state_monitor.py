"""cook_state_user_stats: the monitor's per-user stats and user counts (set-stats-counters!) and the queue lengths
(jobs->queue-lengths) from the live rows of one resident pool or of the pools of a quota group.

CPU: monitor_ref.py on the reference's known answers (test-set-stats-counters!, every step, "accum" included, and
query-queue-lengths, in tests/golden/monitor_golden.json) and on hand-computed cases for each quirk; cycle.monitor_stats
and cycle.queue_lengths against the restatement through its CPU stand-in.
GPU (-m gpu): bit equality with the stand-in after every batch of a churn on C2 and config-#3 trace pools and on
Zipf-user tables on and off the grid; three handles as a quota group; the running part against cook_state_usage and
the waiting jobs against the host's live counts; the golden scenario replayed through cook_state_apply /
cook_state_launch; nothing resident changes; the transfers; the errors.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

import fold_ref as F
import monitor_ref as M
from cook_b200 import abi, cycle, engine, traces
from resident_model import START, Pool, c2, c3, churn, drop_all_but, keyed, pending_rows, pool_rows, random_rows

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "monitor_golden.json")))
BIG = float(np.finfo(np.float64).max)
LONG_MAX = 2 ** 63 - 1
CODES = list(range(8))   # novel-host codes pending_rows draws from (the handles here drop the lists)


# ---- the golden scenario ---------------------------------------------------------------------------------------
def golden_users():
    """User names by code, in first-seen order of the scenario's jobs."""
    names = []
    for j in GOLDEN["monitor"]["jobs"].values():
        if j["user"] not in names:
            names.append(j["user"])
    return names


def golden_rows(step):
    """The step's pending rows (id: the job's number) and running rows (id: 100 + the job's number)."""
    jobs = GOLDEN["monitor"]["jobs"]
    row = lambda j, pool, base: dict(jobs[j], id=base + int(j[3:]), pool=pool)
    return ([row(j, p, 0) for j, p in step["pending"].items()], [row(j, p, 100) for j, p in step["running"].items()])


def golden_tables(step):
    m = GOLDEN["monitor"]
    return dict(m["default_share"], **(step.get("share") or {})), dict(m["default_quota"], **(step.get("quota") or {}))


def check_counters(got, call):
    for state, user, want in call["counters"]:
        entry = got[state].get(user, {})
        assert [entry.get(k, 0) for k in ("jobs", "cpus", "mem")] == want, (call["pool"], state, user)
    for k, v in call.get("users", {}).items():
        assert got["users"][k] == v, (call["pool"], k)


@pytest.mark.parametrize("step", range(len(GOLDEN["monitor"]["steps"])))
def test_golden_set_stats_counters(step):
    s = GOLDEN["monitor"]["steps"][step]
    pend, run = golden_rows(s)
    share, quota = golden_tables(s)
    for call in s["calls"]:
        got = M.set_stats_counters(pend, run, call["pool"], lambda u: share, lambda u: quota, golden_users(),
                                   GOLDEN["monitor"]["grouping"])
        check_counters(got, call)


def test_golden_queue_lengths():
    q = GOLDEN["queue_lengths"]
    rows = [dict(pool=p, user=u) for p, u in q["pending"]]
    assert M.queue_lengths(rows) == q["expect"]


# ---- the quirks, by hand -------------------------------------------------------------------------------------------
def _rows(spec, base):
    """[(user, cpus, mem)] -> rows with ascending ids in one pool."""
    return [dict(id=base + i, user=u, pool="p", cpus=c, mem=m) for i, (u, c, m) in enumerate(spec)]


def _counters(pend, run, shares=None, quota=None):
    shares = shares or {}
    quota = quota or {}
    dq = {"count": 2147483647, "cpus": BIG, "mem": BIG, "gpus": BIG}
    return M.set_stats_counters(pend, run, "p", lambda u: shares.get(u, {"cpus": BIG, "mem": BIG}),
                                lambda u: quota.get(u, dq), sorted({r["user"] for r in pend + run}))


def test_starved_jobs_of_a_running_user():
    """:jobs is only in the running map: a running user's starved jobs are min(running jobs, waiting jobs)."""
    run = _rows([("a", 1.0, 10.0)] * 3, 0)
    pend = _rows([("a", 2.0, 1.0)] * 5 + [("b", 1.0, 1.0)] * 4, 100)
    got = _counters(pend, run, shares={"a": {"cpus": 100.0, "mem": 100.0}, "b": {"cpus": 100.0, "mem": 100.0}})
    assert got["starved"]["a"] == {"jobs": 3, "cpus": 10, "mem": 5}
    assert got["starved"]["b"] == {"jobs": 4, "cpus": 4, "mem": 4}   # not running: the waiting jobs
    assert got["starved"]["all"] == {"jobs": 7, "cpus": 14, "mem": 9}


def test_share_zero_and_max():
    pend = _rows([("a", 1.0, 8.0), ("b", 1.0, 8.0)], 0)
    got = _counters(pend, [], shares={"a": {"cpus": 0.0, "mem": 0.0}})
    assert "a" not in got["starved"] and got["starved"]["b"] == {"jobs": 1, "cpus": 1, "mem": 8}
    assert got["users"] == {"total": 2, "starved": 1, "waiting-under-quota": 2, "hungry": 1, "satisfied": 0}
    # a share at MAX_VALUE minus the running amount is still huge: min picks the waiting amount
    run = _rows([("b", 3.0, 5.0)], 50)
    assert _counters(pend, run)["starved"]["b"] == {"jobs": 1, "cpus": 1, "mem": 8}


def test_quota_rest_keys():
    """A quota key beyond count, cpus and mem at 0 keeps the user out of waiting-under-quota (0.0 < 0 fails); the
    stand-in's rest_ok is that verdict."""
    pend = _rows([(0, 1.0, 8.0), (1, 1.0, 8.0)], 0)
    q = {"count": 10, "cpus": 10.0, "mem": 100.0, "gpus": 0.0}
    got = M.set_stats_counters(pend, [], "p", lambda u: {"cpus": BIG, "mem": BIG},
                               lambda u: dict(q, gpus=1.0) if u == 1 else q, [0, 1])
    assert 0 not in got["waiting-under-quota"] and got["waiting-under-quota"][1]["gpus"] == 1
    one = np.ones(2)
    s = M.user_stats(pend, [], 2, one * BIG, one * BIG, one * 10, one * 10, one * 100, rest_ok=np.array([0, 1]))
    assert s["member"].tolist() == [0b0110, 0b1110]
    assert s["jobs"][abi.STATS_WUQ].tolist() == [0, 1] and s["users"]["waiting-under-quota"] == 1


def test_satisfied_hungry_and_empty():
    run = _rows([("a", 1.0, 1.0), ("c", 1.0, 1.0)], 0)
    pend = _rows([("b", 1.0, 1.0), ("c", 1.0, 1.0)], 100)
    got = _counters(pend, run, shares={"b": {"cpus": 0.0, "mem": 1.0}})
    # a: runs only (satisfied); b: waits with a zero cpus share (hungry); c: runs and waits, starved
    assert got["users"] == {"total": 3, "starved": 1, "waiting-under-quota": 2, "hungry": 1, "satisfied": 1}
    assert set(got["running"]) == {"a", "c", "all"} and set(got["starved"]) == {"c", "all"}
    empty = _counters([], [])
    for s in M.STATES:
        assert empty[s] == {"all": {"cpus": 0, "mem": 0, "jobs": 0}}
    assert set(empty["users"].values()) == {0}


def test_counter_value():
    for x, want in ((float(LONG_MAX), LONG_MAX), (1e300, LONG_MAX), (2.0 ** 62, 2 ** 62), (7.9, 7), (3, 3),
                    (np.int64(LONG_MAX), LONG_MAX), (10000097.0, 10000097)):
        assert cycle.counter_value(x) == M.counter(x) == want


# ---- the layers above, through the CPU stand-in ------------------------------------------------------------------
def _table(rng, U, run):
    """Shares and quotas that put users in every state: some run above their share or quota, some far below."""
    used = {u: sum(r["cpus"] for r in run if r["user"] == u) for u in range(U)}
    around = np.array([used[u] for u in range(U)]) + rng.choice([-1.0, 0.5, 4.0], U)
    return dict(div_cpus=np.where(rng.random(U) < 0.3, BIG, np.maximum(around, 0.0)),
                div_mem=np.where(rng.random(U) < 0.2, 0.0, BIG),
                quota_count=rng.integers(0, 40, U).astype(float), quota_cpus=np.where(rng.random(U) < 0.5, BIG, around),
                quota_mem=np.full(U, BIG), rest_ok=(rng.random(U) < 0.8).astype(np.uint8))


@pytest.mark.parametrize("regime", ["grid", "off"])
def test_monitor_stats_through_the_stand_in(regime):
    rng = np.random.default_rng({"grid": 3, "off": 4}[regime])
    U = 12
    names = [f"user-{(7 * u) % U:02d}" for u in range(U)]
    run = [dict(r, id=r["task_id"]) for r in random_rows(rng, regime, 300, U - 1, 10, [-1])]
    pend = [dict(r, id=r["job_id"]) for r in pending_rows(rng, regime, 400, U - 4, 10_000, CODES)]
    t = _table(rng, U, run)
    raw = M.user_stats(pend, run, U, **t)
    extra = [{"gpus": float(u), "launch-rate-saved": 10000097.0, "launch-rate-per-minute": 600013.0} for u in range(U)]
    got = cycle.monitor_stats(raw, names, extra)
    # the restatement over named rows, with the whole quota maps
    nm = lambda rows: [dict(r, user=names[r["user"]], pool="p") for r in rows]
    code = {n: u for u, n in enumerate(names)}
    shares = lambda n: {"cpus": t["div_cpus"][code[n]], "mem": t["div_mem"][code[n]]}
    quota = lambda n: dict({"count": t["quota_count"][code[n]], "cpus": t["quota_cpus"][code[n]],
                            "mem": t["quota_mem"][code[n]]}, **(extra[code[n]] if t["rest_ok"][code[n]] else
                                                             dict(extra[code[n]], gpus=0.0)))
    want = M.set_stats_counters(nm(pend), nm(run), "p", shares, quota, names)
    assert got == want
    assert {s: len(got[s]) - 1 for s in M.STATES} == {s: int(((raw["member"] >> i) & 1).sum())
                                                      for i, s in enumerate(M.STATES)}
    assert all(0 < got["users"][k] for k in ("starved", "waiting-under-quota", "hungry", "satisfied"))


def test_queue_lengths_through_the_stand_in():
    rng = np.random.default_rng(5)
    U, names = 6, ["alice", "bob", "carol", "dave", "erin", "frank"]
    one = np.ones(U)
    pools = {"p1": pending_rows(rng, "grid", 50, 4, 0, CODES), "p2": pending_rows(rng, "grid", 20, 2, 500, CODES), "p3": []}
    stats = {p: M.user_stats([dict(r, id=r["job_id"]) for r in rows], [], U, one, one, one, one, one)
             for p, rows in pools.items()}
    want = M.queue_lengths([dict(pool=p, user=names[r["user"]]) for p, rows in pools.items() for r in rows])
    assert cycle.queue_lengths(stats, names) == want
    assert "p3" not in want["pool->queue-length"]


# ---- GPU -----------------------------------------------------------------------------------------------------------
def users_of(t, U):
    return abi.make_users(U, div_cpus=t["div_cpus"], div_mem=t["div_mem"],
                          quota={"count": t["quota_count"], "cpus": t["quota_cpus"], "mem": t["quota_mem"]})


def want_of(pools, U, t):
    pend = [dict(r, id=j) for p in pools for j, r in p.pend.items()]
    run = [dict(r, id=k) for p in pools for k, r in p.run.items()]
    return M.user_stats(pend, run, U, **t)


def check(pools, U, t, rest=True):
    """state_user_stats over the pools' handles against the stand-in over their rows, bit for bit, the transfers in the
    call's own statistics, and no cook_last_stats slot of pools[0] touched.  rest: pass t's quota_rest_ok (else NULL,
    every flag 1)."""
    slots = [pools[0].gpu.last_stats(k) for k in range(abi.PHASE_AUDIT + 1)]
    got = engine.state_user_stats([p.gpu for p in pools], users_of(t, U), t["rest_ok"] if rest else None)
    assert [pools[0].gpu.last_stats(k) for k in range(abi.PHASE_AUDIT + 1)] == slots
    want = want_of(pools, U, t if rest else dict(t, rest_ok=None))
    assert np.array_equal(got["member"], want["member"])
    assert np.array_equal(got["jobs"], want["jobs"])
    assert F.same_bits(got["cpus"], want["cpus"]) and F.same_bits(got["mem"], want["mem"])
    for s in M.STATES:
        assert got["all"][s][0] == want["all"][s][0], s
        assert F.same_bits(np.array(got["all"][s][1:]), np.array(want["all"][s][1:])), s
    assert got["users"] == want["users"]
    st = got["stats"]
    live = any(p.pend or p.run for p in pools)
    assert st["h2d_bytes"] == ((41 if rest else 40) * U if live else 0)
    assert st["d2h_bytes"] == (97 * U + 136 if live else 0)
    assert (st["n_launches"] > 0) == live
    return got


def stats_pool(name):
    return Pool(name, drop=drop_all_but("gpus"), send_hosts=True)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["grid", "off", "mixed"])
def test_churn_zipf(regime):
    rng = np.random.default_rng({"grid": 21, "off": 22, "mixed": 23}[regime])
    U = 40
    p = stats_pool("monitor")
    tid, jid = [1_000], [5_000_000]

    def runs(n):
        rows = random_rows(rng, regime, n, U, tid[0], list(range(20)))
        tid[0] += 2 * n + 2
        return rows

    def jobs(n):
        rows = pending_rows(rng, regime, n, U, jid[0], CODES)
        jid[0] += 2 * n + 2
        return keyed(rows)

    try:
        t = _table(rng, U, [])
        check([p], U, t)                                            # empty: zeros, no device work
        p.apply(run_up=runs(700), up=jobs(900))
        for b in range(5):
            t = _table(rng, U, list(p.run.values()))
            check([p], U, t)
            fin = [k for k in p.run if rng.random() < 0.05]
            p.apply(run_up=runs(200), up=jobs(300), run_rm=fin, rm=list(rng.choice(sorted(p.pend), 40, replace=False)))
            check([p], U, t)
            launch = list(rng.choice(sorted(p.pend), 150, replace=False))
            tids = [tid[0] + 2 * i for i in range(len(launch))]
            tid[0] += 2 * len(launch) + 2
            p.launch(launch, tids, np.full(len(launch), START, np.int64))
        got = check([p], U, t)
        if regime == "mixed":   # user 0 passes 2^43 in both folds: the serial chain beside exact ones
            assert got["mem"][abi.STATS_WAITING][0] > 2.0 ** 43
        p.apply(rm=list(p.pend))
        check([p], U, t)                                            # running only: everybody satisfied
        p.apply(run_rm=list(p.run))
        check([p], U, t)
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("trace", ["c2", "c3"])
def test_churn_traces(trace):
    t0 = c2(31) if trace == "c2" else c3(32)
    rng = np.random.default_rng(33)
    pend, run = pool_rows(t0)
    U = t0["users"].n_users
    items = sorted(pend.items())
    reserve, start = items[len(items) // 2:], items[:len(items) // 2]
    p = Pool.of_trace(t0, name="monitor")
    try:
        p.apply(up=start, run_up=list(run.values()))
        t_next = [10 ** 9]
        for b in range(4):
            t = _table(rng, U, list(p.run.values()))
            check([p], U, t)
            launched = [int(j) for j in rng.choice(sorted(p.pend), 60, replace=False)]
            up, rm, run_up, run_rm = churn(p, rng, reserve, t_next, launched)
            p.apply(up=up, rm=rm, run_up=run_up, run_rm=run_rm)
        check([p], U, t)
    finally:
        p.close()


@pytest.mark.gpu
def test_quota_group_of_three_handles():
    """The union of three handles' rows; a job id two handles hold folds in the order of the handle list."""
    rng = np.random.default_rng(41)
    U = 25
    pools = [stats_pool(f"g{i}") for i in range(3)]
    try:
        for i, p in enumerate(pools):
            p.apply(run_up=random_rows(rng, "off", 300 + 50 * i, U, 10 + 7_000 * i, [-1]),
                    up=keyed(pending_rows(rng, "off", 500, U, 1_000_000 + 9_000 * i, CODES)))
        shared = keyed(pending_rows(rng, "off", 80, U, 5_000_000, CODES))   # the same job ids in g0 and g2
        pools[0].apply(up=shared)
        pools[2].apply(up=[(j, dict(r, cpus=r["cpus"] * 3.0)) for j, r in shared])
        t = _table(rng, U, [r for p in pools for r in p.run.values()])
        check(pools, U, t)
        check(pools, U, t, rest=False)                             # NULL quota_rest_ok: every flag 1, 40 B per user up
        check(pools[::-1], U, t)                                    # the shared ids now fold g2's row first
        check([pools[1], pools[0]], U, t)
    finally:
        for p in pools:
            p.close()


@pytest.mark.gpu
def test_running_part_is_the_usage_fold():
    rng = np.random.default_rng(51)
    U = 30
    p = stats_pool("usage")
    try:
        p.apply(run_up=random_rows(rng, "off", 2500, U, 10, [-1]), up=keyed(pending_rows(rng, "off", 3000, U, 10 ** 6, CODES)))
        t = _table(rng, U, list(p.run.values()))
        got = engine.state_user_stats([p.gpu], users_of(t, U), t["rest_ok"])
        usage = p.gpu.state_usage(U)["user"]
        running = (got["member"] & 1).astype(bool)
        assert np.array_equal(running, usage["count"] > 0)
        assert np.array_equal(got["jobs"][abi.STATS_RUNNING], usage["count"].astype(np.int64))
        assert F.same_bits(got["cpus"][abi.STATS_RUNNING], usage["cpus"])
        assert F.same_bits(got["mem"][abi.STATS_RUNNING], usage["mem"])
        live = np.bincount([r["user"] for r in p.pend.values()], minlength=U)
        assert np.array_equal(got["jobs"][abi.STATS_WAITING], live)
    finally:
        p.close()


@pytest.mark.gpu
def test_golden_replay():
    """test-set-stats-counters! through resident handles pool1 and pool2: submissions as pending upserts, run-job as
    cook_state_launch, kill-job as a removal; a quota-group call over both for "accum"."""
    names = golden_users()
    code = {n: u for u, n in enumerate(names)}
    U = len(names)
    jobs = GOLDEN["monitor"]["jobs"]
    handles = {n: stats_pool(n) for n in ("pool1", "pool2")}
    try:
        for s in GOLDEN["monitor"]["steps"]:
            for n, p in handles.items():
                want_p = {int(j[3:]) for j, q in s["pending"].items() if q == n}
                want_r = {int(j[3:]) for j, q in s["running"].items() if q == n}
                run_jobs = {r["job_id"]: k for k, r in p.run.items()}
                launch = sorted(j for j in want_r if j in p.pend)
                if launch:
                    p.launch(launch, [100 + j for j in launch], np.full(len(launch), START, np.int64))
                rm = [j for j in p.pend if j not in want_p]
                run_rm = [k for j, k in run_jobs.items() if j not in want_r]
                up = [(j, dict(user=code[jobs[f"job{j}"]["user"]], cpus=jobs[f"job{j}"]["cpus"], mem=jobs[f"job{j}"]["mem"]))
                      for j in sorted(want_p - set(p.pend))]
                if rm or run_rm or up:
                    p.apply(rm=rm, run_rm=run_rm, up=up)
            share, quota = golden_tables(s)
            t = dict(div_cpus=np.full(U, float(share["cpus"])), div_mem=np.full(U, float(share["mem"])),
                     quota_count=np.full(U, float(quota["count"])), quota_cpus=np.full(U, float(quota["cpus"])),
                     quota_mem=np.full(U, float(quota["mem"])))
            rest = {k: v for k, v in quota.items() if k not in ("count", "cpus", "mem")}
            ok = np.full(U, int(all(v > 0 for v in rest.values())), np.uint8)
            for call in s["calls"]:
                hs = [handles["pool1"], handles["pool2"]] if call["pool"] == "accum" else [handles[call["pool"]]]
                raw = engine.state_user_stats([h.gpu for h in hs], users_of(dict(t, rest_ok=ok), U), ok)
                got = cycle.monitor_stats(raw, names, [rest] * U)
                check_counters(got, call)
                check(hs, U, dict(t, rest_ok=ok))
    finally:
        for p in handles.values():
            p.close()


@pytest.mark.gpu
def test_nothing_resident_changes():
    t0 = c2(61)
    rng = np.random.default_rng(62)
    pend, run = pool_rows(t0)
    U = t0["users"].n_users
    p = Pool.of_trace(t0, name="monitor")
    try:
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.rank()
        m = p.gpu.state_match(p.offers, p.users, p.params, max_ports=p.max_ports)
        k = np.arange(min(len(m["considerable"]), 32), dtype=np.int32)
        prm = abi.ConsiderableParams(500, 0, 1, abi.USAGE_LAST_MATCH, 0)
        p.gpu.state_usage(U)                                       # the usage slot holds a call check() must not touch

        def seen():
            return (p.gpu.state_digest(16), p.gpu.state_queue(), p.gpu.match_failures(k),
                    p.gpu.state_considerable(p.users, prm))
        before = seen()
        assert len(before[3]) > 0
        t = _table(rng, U, list(p.run.values()))
        check([p], U, t)
        after = seen()
        for a, b in zip(before[0].values(), after[0].values()):
            assert np.array_equal(np.asarray(a), np.asarray(b))
        assert np.array_equal(before[1], after[1]) and before[2] == after[2]
        assert np.array_equal(before[3], after[3])                 # the LAST_MATCH selection reads the same usage
    finally:
        p.close()


@pytest.mark.gpu
def test_errors():
    rng = np.random.default_rng(71)
    a, b = stats_pool("a"), stats_pool("b")
    try:
        a.apply(run_up=random_rows(rng, "grid", 100, 6, 10, [-1]), up=keyed(pending_rows(rng, "grid", 100, 8, 10 ** 6, CODES)))
        U = 8
        t = _table(rng, U, list(a.run.values()))
        users = users_of(t, U)
        lib = a.gpu.lib
        outs = [np.zeros(4 * U, np.int64), np.zeros(4 * U), np.zeros(4 * U), np.zeros(U, np.uint8), np.zeros(4, np.int64),
                np.zeros(4), np.zeros(4), np.zeros(abi.USERS_N, np.int64)]
        types = [abi.P_I64, abi.P_F64, abi.P_F64, abi.P_U8, abi.P_I64, abi.P_F64, abi.P_F64, abi.P_I64]
        ptrs = [abi.ptr(o, ty) for o, ty in zip(outs, types)]
        H = lambda *ps: (C.c_void_p * len(ps))(*ps)
        small = abi.make_users(7)
        no_div = abi.make_users(U)
        no_div.div_cpus = abi.P_F64()
        cases = [(H(a.gpu.pool), 0, users, ptrs), (H(a.gpu.pool), -1, users, ptrs),
                 (H(a.gpu.pool, a.gpu.pool), 2, users, ptrs), (H(a.gpu.pool, None), 2, users, ptrs),
                 (H(a.gpu.pool), 1, None, ptrs), (H(a.gpu.pool), 1, small, ptrs), (H(a.gpu.pool), 1, no_div, ptrs)]
        cases += [(H(a.gpu.pool, b.gpu.pool), 2, users, ptrs[:i] + [None] + ptrs[i + 1:]) for i in range(len(ptrs))]
        for hs, n, us, ps in cases:
            for o in outs:
                o[...] = 7
            rc = lib.cook_state_user_stats(hs, n, C.byref(us) if us is not None else None, None, *ps, None)
            assert rc == abi.COOK_E_BADARG
            assert all(np.all(o == 7) for o in outs)                        # nothing written
        assert lib.cook_state_user_stats(None, 1, C.byref(users), None, *ptrs, None) == abi.COOK_E_BADARG
        # out_stats is optional
        assert lib.cook_state_user_stats(H(a.gpu.pool), 1, C.byref(users), None, *ptrs, None) == abi.COOK_OK
        # no live row in any handle: zeros without device work
        check([a], U, t)
        c = stats_pool("c")
        try:
            got = check([c, b], U, t)
            assert not got["member"].any() and got["users"] == dict.fromkeys(engine.USER_COUNTS, 0)
            assert got["stats"] == abi.PhaseStats().as_dict()
        finally:
            c.close()
    finally:
        a.close()
        b.close()
