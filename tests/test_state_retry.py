"""Retries on a resident handle (cook_state_retry_config, cook_state_retry_facts, cook_state_status): the golden
decisions replayed, a churn past one sort tile checked bit for bit against a twin handle fed
cook_state_finish_history plus the host-built upserts, the handle without facts unchanged, every way a parked copy
is freed, the BADARGs and the transfer formulas."""
import json
import os

import numpy as np
import pytest

import resident_model as M
import retry_ref as RR
from cook_b200 import abi, traces
from cook_b200.engine import CookError, GpuEngine

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "retry_golden.json")))
REASONS = GOLDEN["reasons"]
CODE = {k: v["code"] for k, v in REASONS.items()}
REASON_OF = {v["code"]: v for v in REASONS.values()}
OUTCOME = {abi.JOB_COMPLETED: "completed", abi.JOB_RUNNING: "running", abi.JOB_WAITING: "waiting",
           abi.JOB_WAITING_UNRETAINED: "waiting"}
START = M.START


def handle(name="retry"):
    e = GpuEngine(pool_name=name)
    e.state_retry_config(GOLDEN["mea_culpa_limit"],
                         [(v["code"], v["mea_culpa"], -2 if v["failure_limit"] is None else v["failure_limit"])
                          for v in REASONS.values()])
    return e


def prow(user=0, cpus=1.0, novel=(), groups=(), reserved=-1):
    r = dict(M.DEFAULTS, user=user, priority=50, cpus=cpus, mem=1024.0, novel=list(novel), attr=[], groups=list(groups))
    r["reserved_host"] = reserved
    return r


def run_row(jid, tid, host=-1):
    return dict(user=0, priority=50, start_time=START, task_id=tid, job_id=jid, cpus=1.0, mem=1024.0, gpus=0.0,
                host=host, groups=[])


def bad(fn, *a, **k):
    with pytest.raises(CookError) as ei:
        fn(*a, **k)
    assert ei.value.code == abi.COOK_E_BADARG


def snapshot(e, users=None, offers=None, params=None, probe=()):
    """Digest, export and, with users, the next rank and the queue; with offers, the derived match over that queue;
    with probe (job ids), cook_state_unscheduled's answer for them."""
    d = e.state_digest()
    out = {k: d[k] for k in ("pending", "running", "entries", "consistent")}
    out["export"] = export(e)
    if users is not None:
        out["rank"] = e.state_rank(users).tolist()
        out["queue"] = e.state_queue().tolist()
    if offers is not None:
        m = e.state_match(offers, users, params, derived=True)
        out["match"] = {k: m[k].tolist() for k in ("considerable", "assign", "ports", "fail")}
    if len(probe):
        u = e.state_unscheduled(probe)
        out["unscheduled"] = {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in u.items() if k != "stats"}
    return out


def export(e):
    """cook_state_export's rows as plain lists, column by column."""
    out = {}
    for k, v in e.state_export().items():
        if isinstance(v, np.ndarray):
            out[k] = v.tolist()
            continue
        for n, t in v._fields_:
            c = v.col(n) if t in abi._NP else getattr(v, n)
            out[f"{k}.{n}"] = c.tolist() if isinstance(c, np.ndarray) else c
    return out


# ---- the golden decisions ------------------------------------------------------------------------------------
def _replayable(case):
    ups = [(k, st, r) for k, (st, r) in enumerate(case["updates"]) if st is not None]
    return (len(ups) == 1 and ups[0][1] in RR.DONE and case["instances"][ups[0][0]][0] in ("running", "unknown"))


@pytest.mark.parametrize("case", [c for c in GOLDEN["transitions"] if _replayable(c)], ids=lambda c: c["name"])
def test_golden_transition(case):
    (k, st, r), = [(k, st, r) for k, (st, r) in enumerate(case["updates"]) if st is not None]
    e = handle()
    try:
        e.state_apply(M.delta(up=[(1, prow())]))
        others = [j for j in range(len(case["instances"])) if j != k]
        live = [j for j in others if case["instances"][j][0] in ("running", "unknown")]
        if live:
            e.state_apply(M.delta(run_up=[run_row(1, 100 + j) for j in live]))
        done = [CODE[rr] if rr else -1 for s, rr in (case["instances"][j] for j in others) if s in RR.DONE]
        flags = (abi.RF_DISABLE_MEA_CULPA if case["disable"] else 0) | (
            abi.RF_COMPLETED if case["old_job_state"] == "completed" else 0)
        e.state_retry_facts([1], [case["retry_count"]], [flags], [done])
        e.state_launch([1], [1], [START], [7])
        oc, att = e.state_status([1], [st == "success"], [START + 1000], [CODE[r]])
        assert OUTCOME[int(oc[0])] == case["new_job_state"]
        want = RR.reasons_attempts_consumed(5, case["disable"], [REASON_OF.get(c) for c in done + [CODE[r]]])
        assert int(att[0]) == want
        assert e.state_digest()["pending"][2] == (1 if case["new_job_state"] == "waiting" else 0)
    finally:
        e.close()


@pytest.mark.parametrize("case", GOLDEN["batch"], ids=lambda c: c["name"])
def test_golden_batch(case):
    """Two instances of one job fail in one call: decided one status at a time, in batch order."""
    e = handle()
    try:
        e.state_apply(M.delta(up=[(1, prow())]))
        e.state_retry_facts([1], [case["retry_count"]], [0], [[]])
        e.state_launch([1], [10], [START], [3])
        e.state_apply(M.delta(run_up=[run_row(1, 11, 4)], hosts=True))
        tids = [10 + k for k, _, _ in case["order"]]
        oc, att = e.state_status(tids, [s == "success" for _, s, _ in case["order"]], [START + 5] * 2,
                                 [CODE[r] for _, _, r in case["order"]])
        assert [OUTCOME[int(o)] for o in oc] == case["outcomes"]
        assert att.tolist() == case["attempts"]
    finally:
        e.close()


# ---- a churn against the twin --------------------------------------------------------------------------------
def test_churn_matches_twin():
    rng = np.random.default_rng(7)
    t = M.c2(11)
    pend, _ = M.pool_rows(t)
    users = t["users"]
    jids = sorted(pend)
    for j in jids:   # some lists in the arena, some reservations
        if rng.random() < 0.3:
            pend[j] = dict(pend[j], novel=sorted(set(rng.integers(0, 200, 2).tolist())))
        if rng.random() < 0.1:
            pend[j] = dict(pend[j], groups=[int(rng.integers(0, 5))])
        if rng.random() < 0.1:
            pend[j] = dict(pend[j], reserved_host=int(rng.integers(0, 200)))
    a, b = handle("a"), GpuEngine(pool_name="b")
    try:
        init = M.delta(up=[(j, pend[j]) for j in jids], lists=True)
        a.state_apply(init)
        b.state_apply(M.delta(up=[(j, pend[j]) for j in jids], lists=True))
        facts = {j: dict(max_retries=int(rng.integers(1, 4)), disable=bool(rng.random() < 0.2), completed=False,
                         done=[]) for j in jids}
        a.state_retry_facts(jids, [facts[j]["max_retries"] for j in jids],
                            [abi.RF_DISABLE_MEA_CULPA if facts[j]["disable"] else 0 for j in jids], [[] for _ in jids])
        live_pend, running, parked = set(jids), {}, set()
        tid = [1_000_000]
        codes = [CODE["unknown"], CODE["preempted-by-rebalancer"], CODE["mesos-executor-terminated"], -1]
        offers, params = t["offers"], traces.match_params(1000)
        probe = np.array(jids[::37], np.int64)
        assert snapshot(a, users, offers, params, probe) == snapshot(b, users, offers, params, probe)
        for cycle in range(5):
            # launches
            lj = sorted(rng.choice(sorted(live_pend), size=min(900, len(live_pend)), replace=False).tolist())
            tids = list(range(tid[0], tid[0] + len(lj)))
            tid[0] += len(lj)
            hosts = rng.integers(0, 200, len(lj)).astype(np.int32)
            starts = [START + cycle * 1000] * len(lj)
            a.state_launch(lj, tids, starts, hosts)
            sa = a.last_stats(abi.PHASE_STATE)
            b.state_launch(lj, tids, starts, hosts)
            sb = b.last_stats(abi.PHASE_STATE)
            assert sa["h2d_bytes"] == sb["h2d_bytes"] + 4 * len(lj)   # the parked and freed slots
            for j, tk, h in zip(lj, tids, hosts.tolist()):
                live_pend.discard(j)
                parked.add(j)
                running[tk] = (j, h)
            # terminal statuses of most running tasks
            fin = [tk for tk in sorted(running) if rng.random() < 0.7]
            rng.shuffle(fin)
            ok = (rng.random(len(fin)) < 0.3).astype(np.uint8)
            reason = rng.choice(codes, len(fin)).astype(np.int32)
            pre = (rng.random(len(fin)) < 0.2).astype(np.uint8)
            end = [START + cycle * 1000 + 500] * len(fin)
            oc, att = a.state_status(fin, ok, end, reason, pre)
            sa = a.last_stats(abi.PHASE_STATE)
            b.state_finish_history(fin, end, ok, reason)
            sb = b.last_stats(abi.PHASE_STATE)
            ups, nrq, nap, nfree = [], 0, 0, 0
            for i, tk in enumerate(fin):
                j, h = running.pop(tk)
                other = any(jj == j for jj, _ in running.values())
                want, want_att, facts[j] = RR.decide(facts[j], REASON_OF, bool(ok[i]), int(reason[i]), other)
                got = OUTCOME[int(oc[i])]
                assert (got, int(att[i])) == (want, want_att), (cycle, i)
                if want == "waiting":
                    row = RR.requeued_row(pend[j], h, bool(pre[i]))
                    nap += len(row["novel"]) != len(pend[j]["novel"])
                    pend[j] = row
                    ups.append((j, row))
                    parked.discard(j)
                    live_pend.add(j)
                    nrq += 1
                elif want == "completed" and j in parked:
                    parked.discard(j)
                    nfree += 1
            assert sa["h2d_bytes"] == sb["h2d_bytes"] + 4 * nrq + 8 * nap + 4 * nfree
            if ups:
                b.state_apply(M.delta(up=ups, lists=True))
            assert nrq > 0
            assert snapshot(a, users, offers, params, probe) == snapshot(b, users, offers, params, probe), cycle
            assert a.state_digest()["consistent"]
    finally:
        a.close()
        b.close()


def test_without_facts_unchanged():
    """A handle without retry facts: cook_state_status is cook_state_finish_history (digest, export, transfers and
    launches), every outcome COOK_JOB_NO_FACTS, and its launches free the pending slots."""
    rng = np.random.default_rng(3)
    t = M.c2(5)
    pend, _ = M.pool_rows(t)
    jids = sorted(pend)
    a, b = handle("a"), GpuEngine(pool_name="b")
    try:
        for e in (a, b):
            e.state_apply(M.delta(up=[(j, pend[j]) for j in jids]))
        lj = jids[:1200]
        hosts = rng.integers(0, 50, len(lj)).astype(np.int32)
        for e in (a, b):
            e.state_launch(lj, range(1, len(lj) + 1), [START] * len(lj), hosts)
        la, lb = a.last_stats(abi.PHASE_STATE), b.last_stats(abi.PHASE_STATE)
        assert (la["h2d_bytes"], la["n_launches"]) == (lb["h2d_bytes"], lb["n_launches"])
        assert la["h2d_bytes"] == len(lj) * (4 + 4 + 8 + 8 + 4)   # cook_state_launch's formula, hosts given
        fin = list(range(1, 801))
        ok = (rng.random(800) < 0.5).astype(np.uint8)
        oc, att = a.state_status(fin, ok, [START + 9] * 800, None)
        b.state_finish_history(fin, [START + 9] * 800, ok, None)
        la, lb = a.last_stats(abi.PHASE_STATE), b.last_stats(abi.PHASE_STATE)
        assert (la["h2d_bytes"], la["n_launches"], la["d2h_bytes"]) == (lb["h2d_bytes"], lb["n_launches"], lb["d2h_bytes"])
        assert la["h2d_bytes"] == 13 * 800 and la["d2h_bytes"] == 0   # cook_state_finish_history's, history off
        assert set(oc.tolist()) == {abi.JOB_NO_FACTS} and set(att.tolist()) == {-1}
        assert snapshot(a, t["users"]) == snapshot(b, t["users"])
    finally:
        a.close()
        b.close()


# ---- freeing a parked copy -----------------------------------------------------------------------------------
def _parked(e, jid=1, tids=(1,), novel=(2,)):
    e.state_apply(M.delta(up=[(jid, prow(novel=novel))], lists=True))
    e.state_retry_facts([jid], [3], [0], [[]])
    e.state_launch([jid], [tids[0]], [START], [5])
    for k, t in enumerate(tids[1:]):
        e.state_apply(M.delta(run_up=[run_row(jid, t)]))


def _held(e, jid):
    try:
        e.state_retry_facts([jid], [3], [0], [[]])
        return True
    except CookError as err:
        assert err.code == abi.COOK_E_BADARG
        return False


def test_free_paths():
    e = handle()
    try:
        _parked(e)                                  # a completed decision
        oc, _ = e.state_status([1], [1], [START + 1], [-1])
        assert oc.tolist() == [abi.JOB_COMPLETED] and not _held(e, 1)
        _parked(e, 2, (2,))                         # facts with COMPLETED, no live instance left
        e.state_apply(M.delta(run_rm=[2]))          # the instance leaves without a status
        e.state_retry_facts([2], [3], [abi.RF_COMPLETED], [[]])
        assert not _held(e, 2)
        _parked(e, 3, (3,))                         # a pending upsert of its id: the caller's row wins
        e.state_apply(M.delta(up=[(3, prow(cpus=2.0))], lists=True))
        oc, _ = e.state_status([3], [0], [START + 1], [-1])
        assert oc.tolist() == [abi.JOB_NO_FACTS]
        assert e.state_digest()["pending"][2] == 1
        _parked(e, 4, (4, 5))                       # the finish of the job's last live instance
        e.state_finish([4])
        assert _held(e, 4)
        e.state_finish_history([5], [START + 1], [0], [-1])
        assert not _held(e, 4)
        _parked(e, 6, (6,))                         # a reset
        e.state_apply(M.delta(reset=True))
        assert not _held(e, 6)
        d = e.state_digest()
        assert d["consistent"] and d["pending"][2] == 0 and d["entries"][0] == 0
    finally:
        e.close()


def test_unretained_and_compaction():
    """A job whose task came in through a running upsert has no parked copy; parked lists survive compactions."""
    e = handle()
    try:
        e.state_apply(M.delta(run_up=[run_row(9, 90)]))
        e.state_retry_facts([9], [3], [0], [[]])
        oc, att = e.state_status([90], [0], [START + 1], [-1])
        assert oc.tolist() == [abi.JOB_WAITING_UNRETAINED] and att.tolist() == [1]
        # parked lists, then churn the novel arena until it compacts several times
        for j in range(100, 140):
            _parked(e, j, (j,), novel=(j % 7, 50 + j))
        for k in range(40):
            e.state_apply(M.delta(up=[(1000 + k, prow(novel=list(range(30))))], lists=True))
            e.state_apply(M.delta(rm=[1000 + k]))
        oc, _ = e.state_status(list(range(100, 140)), [0] * 40, [START + 1] * 40, [-1] * 40, None)
        assert set(oc.tolist()) == {abi.JOB_WAITING}
        x = e.state_export()
        rows = {j: i for i, j in enumerate(x["pending_job_id"].tolist())}
        off, hosts = x["pending"].col("novel_off"), x["pending"].col("novel_host")
        for j in range(100, 140):
            i = rows[j]
            assert hosts[off[i]:off[i + 1]].tolist() == [j % 7, 50 + j] + ([5] if j % 7 != 5 else [])
        assert e.state_digest()["consistent"]
    finally:
        e.close()


def test_badargs():
    e = handle()
    try:
        _parked(e, 1, (1, 2))
        bad(e.state_retry_config, -2, [])
        bad(e.state_retry_config, 5, [(1, True, -3)])
        bad(e.state_retry_config, 5, [(1, True, 1), (1, False, 1)])
        bad(e.state_retry_config, 5, [(-1, True, 1)])
        bad(e.state_retry_facts, [77], [3], [0], [[]])                 # not held
        bad(e.state_retry_facts, [1, 1], [3, 3], [0, 0], [[], []])     # twice
        bad(e.state_retry_facts, [1], [-1], [0], [[]])
        bad(e.state_retry_facts, [1], [3], [4], [[]])
        bad(e.state_retry_facts, [1], [3], [0], [[-2]])
        bad(e.state_status, [3], [0], [START], [-1])                   # unknown task
        bad(e.state_status, [1], [0], [START - 1], [-1])               # ends before its start
        bad(e.state_status, [1], [0], [START + 1], [-2])
        rc = e.lib.cook_state_status(e.pool, 1, abi.ptr(np.array([1], np.int64), abi.P_I64),
                                     abi.ptr(np.array([0], np.uint8), abi.P_U8),
                                     abi.ptr(np.array([START + 1], np.int64), abi.P_I64), None, None, None, None)
        assert rc == abi.COOK_E_BADARG
        oc, _ = e.state_status([1, 2], [0, 0], [START + 1] * 2, [-1, -1])   # still live: nothing changed
        assert oc.tolist() == [abi.JOB_RUNNING, abi.JOB_WAITING]
    finally:
        e.close()


# ---- the novel host reaches the matcher ----------------------------------------------------------------------
def test_match_avoids_failed_host(oracle):
    """A job placed on a host, launched there and failed, is requeued with that host on its novel-host list: the next
    resident match does not place it there although the host still offers, and equals cook_match and the oracle on
    the model's rows."""
    t = M.c2(21)
    p = M.Pool.of_trace(t, name="retry")
    p.gpu.state_retry_config(5, [])
    try:
        items = sorted(M.pool_rows(t)[0].items())
        p.apply(up=items, lists=True)
        p.gpu.state_retry_facts([j for j, _ in items], [5] * len(items), [0] * len(items), [[] for _ in items])
        p.rank()
        got = p.check_match()
        hn = t["offers"].col("hostname_id")
        placed = [(int(j), int(hn[a])) for j, a in zip(got["considerable"], got["assign"]) if a >= 0][:200]
        assert placed
        jobs = [j for j, _ in placed]
        tids = list(range(1, len(jobs) + 1))
        p.launch(jobs, tids, [START] * len(jobs), [h for _, h in placed])
        oc, _ = p.gpu.state_status(tids, [0] * len(jobs), [START + 1] * len(jobs), [-1] * len(jobs))
        assert set(oc.tolist()) == {abi.JOB_WAITING}
        rows = dict(items)
        p.mirror(run_rm=tids, up=[(j, RR.requeued_row(rows[j], h, False)) for j, h in placed])
        p.rank()
        got = p.check_match()
        jobs_t, jid, ranked = p.ranked(p.live_queue())
        want = oracle.match(ranked, jobs_t, t["offers"], p.users, p.params, groups=p.groups, max_ports=p.max_ports)
        for k in ("assign", "fail"):
            assert np.array_equal(got[k], want[k]), k
        where = {int(j): int(a) for j, a in zip(got["considerable"], got["assign"])}
        again = [j for j, h in placed if where.get(j, -1) >= 0]
        assert again, "some requeued job is placed again"
        for j, h in placed:
            assert where.get(j, -1) < 0 or int(hn[where[j]]) != h, j
    finally:
        p.close()


# ---- preemptions from a config-#4 rebalance ----------------------------------------------------------------------
def test_rebalance_preemptions_match_twin(oracle):
    """The victims of a config-#4 cook_state_rebalance reported as preempted failures: a launched job with facts is
    requeued without the host it was preempted on; the handle stays bit-identical to the twin."""
    r, codes = M.rebalance_trace(29, True)
    rp, rr = M.rows_of(r, codes)
    rng = np.random.default_rng(5)
    a, b = handle("a"), GpuEngine(pool_name="b")
    try:
        items = sorted(rp.items())
        for e in (a, b):
            e.state_apply(M.delta(up=items, run_up=[dict(x, groups=[]) for x in rr.values()], hosts=True, lists=True))
        launched = [j for j, _ in items[::2]]
        a.state_retry_facts(launched, [5] * len(launched), [0] * len(launched), [[] for _ in launched])
        tids = list(range(10 ** 9, 10 ** 9 + len(launched)))
        hosts = [int(codes[k]) for k in rng.integers(0, len(codes), len(launched))]
        for e in (a, b):
            e.state_launch(launched, tids, [START] * len(launched), hosts)
        host_of = dict(zip(tids, hosts))
        job_of = dict(zip(tids, launched))
        assert a.state_rank(r["users"]).tolist() == b.state_rank(r["users"]).tolist()
        ra = a.state_rebalance(r["hosts"], r["users"], r["params"], groups=r["groups"])
        rb = b.state_rebalance(r["hosts"], r["users"], r["params"], groups=r["groups"])
        assert ra == rb
        victims = sorted({v for d in ra for v in d["victims"] if v >= 0})
        assert any(v in job_of for v in victims)
        n = len(victims)
        oc, _ = a.state_status(victims, [0] * n, [START + 1] * n, [CODE["preempted-by-rebalancer"]] * n, [1] * n)
        b.state_finish_history(victims, [START + 1] * n, [0] * n, [CODE["preempted-by-rebalancer"]] * n)
        ups = []
        for v, o in zip(victims, oc.tolist()):
            if v in job_of:
                assert o == abi.JOB_WAITING
                j = job_of[v]
                ups.append((j, RR.requeued_row(rp[j], host_of[v], True)))
                assert ups[-1][1]["novel"] == rp[j]["novel"]
            else:
                assert o == abi.JOB_NO_FACTS
        b.state_apply(M.delta(up=ups, lists=True))
        assert snapshot(a, r["users"]) == snapshot(b, r["users"])
        assert a.state_rebalance(r["hosts"], r["users"], r["params"], groups=r["groups"]) == \
            b.state_rebalance(r["hosts"], r["users"], r["params"], groups=r["groups"])
    finally:
        a.close()
        b.close()
