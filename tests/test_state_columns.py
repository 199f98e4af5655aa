"""-m gpu: a resident handle's growing device stores across their capacity boundaries, each checked against its
restatement: the history and the completed-job log past 4096 rows, then an advance (a compaction into new columns of
the same capacity), then past that capacity; the match-metrics unmatched counters growing while the round's current
half is the second one; and the park flags growing when the pending table doubles with jobs parked.  The record
table's growth and the compaction after it are crossed by test_state_sweeps.py's churn."""
import numpy as np
import pytest

import completed_ref as CR
import list_ref as L
import match_metrics_ref as MR
import resident_model as M
from cook_b200 import traces
from cook_b200.engine import GpuEngine
from test_state_fact_lifecycle import Twin, prow
from test_state_history_stats import Pools, seed as hist_seed
from test_state_list_completed import ask, record, seed as cj_seed
from test_state_match_metrics import _check, _jobs

pytestmark = pytest.mark.gpu

START = M.START


def test_history_past_capacity_advance_and_past_again():
    import history_ref as Hr
    rng = np.random.default_rng(41)
    ps = Pools(["cols"])
    tid = [10 ** 6]

    def running(n, t0):
        rows = []
        for _ in range(n):
            tid[0] += 1
            rows.append(dict(task_id=tid[0], job_id=tid[0] + 10 ** 7, user=int(rng.integers(0, 5)), priority=50,
                             start_time=t0 + int(rng.integers(0, 10 ** 6)), cpus=float(rng.integers(1, 8)),
                             mem=128.0 * int(rng.integers(1, 64)), gpus=0.0, groups=[]))
        return rows

    def finish(rows):
        ids = [r["task_id"] for r in rows]
        ends = [r["start_time"] + int(rng.integers(0, 10 ** 6)) for r in rows]
        ps.finish(0, ids, ends, [int(x) for x in rng.integers(0, 2, len(ids))],
                  [int(c) for c in rng.choice([-1, 1001, 3001], len(ids))])

    def check():
        for status in (Hr.SUCCESS, Hr.FAILED):
            ps.check(status, ps.h[0].since, START + 10 ** 8)

    try:
        since = START - 10 ** 6
        seeded = [dict(task_id=i, user=i % 5, start=since + 37 * i, end=since + 37 * i + 5000, cpus=1.0 + i % 3,
                       mem=512.0, success=bool(i % 2), reason=-1 if i % 3 else 1001) for i in range(4000)]
        hist_seed(ps.e[0], ps.h[0], since, seeded)
        run = running(600, START)
        ps.apply(0, run_up=run)
        finish(run)                                   # 4600 rows: past 4096
        assert len(ps.h[0].rows) > 4096
        check()
        ps.advance(0, since + 37 * 3000)              # the first 3000 seeded rows leave
        assert len(ps.h[0].rows) == 1600
        check()
        for _ in range(2):
            run = running(3500, START)
            ps.apply(0, run_up=run)
            finish(run)
        assert len(ps.h[0].rows) > 8192               # past the capacity the advance kept
        check()
    finally:
        ps.close()


def test_completed_past_capacity_advance_and_past_again():
    rng = np.random.default_rng(43)
    e, lg = GpuEngine(pool_name="cols-cj"), {}
    jid = [1]

    def batch(n, lo):
        rows = []
        for _ in range(n):
            rows.append((jid[0], 7, int(rng.integers(0, 2)), int(lo + rng.integers(0, 40_000)), int(rng.integers(-1, 3)),
                         int(rng.integers(-1, 2)), int(rng.choice([CR.SUCCESS, CR.FAILED, CR.REOPENED]))))
            jid[0] += 1
        return rows

    def check():
        for u in (0, 1):
            for limit in (150, (1 << 31) - 1):
                q = L.query(u, 0, lg["since"], START + 10 ** 6, limit=limit, include_custom_executor=True)
                for s in (CR.L_SUCCESS, CR.L_FAILED, CR.L_COMPLETED):
                    assert ask([e], q, s)[0] == CR.list_completed([lg], q, s), (u, limit, s)

    try:
        cj_seed(e, lg, START, batch(4000, START))
        record(e, lg, batch(600, START))              # 4600 rows: past 4096
        assert len(lg["rows"]) > 4096
        check()
        e.state_completed_advance(START + 30_000)     # about three quarters leave
        CR.advance(lg, START + 30_000)
        assert len(lg["rows"]) < 4096
        check()
        for _ in range(3):
            record(e, lg, batch(2500, START + 30_000))
        assert len(lg["rows"]) > 8192                 # past the capacity the advance kept
        check()
    finally:
        e.close()


def test_unmatched_counters_grow_in_the_second_half():
    """Round 1 counts a few considerable jobs into half 0 and makes half 1 current; round 2 counts more jobs than
    the counters hold, so they grow while half 1 is current, keeping round 1's pairs."""
    t = M.c2(29)
    p = M.Pool.of_trace(t, name="cols-mm")
    U = p.users.n_users
    try:
        pend, run = M.pool_rows(t)
        p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
        prev, sizes, first = {}, [], set()
        for limit in (64, 3000):
            p.params = traces.match_params(limit)
            p.rank()
            m = p.gpu.state_match(p.offers, p.users, p.params, max_ports=p.max_ports)
            ids = [int(j) for j in m["considerable"]]
            sizes.append(len(ids))
            assigned = [k for k, a in enumerate(m["assign"]) if a >= 0]
            # every job of round 1 unmatched in both rounds: 64 pairs in the counters, then read back by round 2
            dropped = [k for k in assigned if limit == 64 or ids[k] in first]
            got = p.gpu.state_match_metrics(U, dropped, unmatched_warn_cycles=1)
            jobs = _jobs(p, {}, ids)
            want = MR.answer(jobs, set(assigned) - set(dropped), prev, 1, U)
            _check(got, want, jobs)
            prev = want["cycles"]
            if limit == 64:
                assert len(prev) == len(ids) == 64
                first = set(ids)
        assert sizes[1] > 64 and first <= set(ids)
        assert got["too_long"] == 64   # round 1's pairs survived the growth
    finally:
        p.close()


def test_park_flags_grow_with_the_pending_table():
    """100 jobs parked while the pending table holds 1024 slots; the table doubles and another job parks, so the flags
    grow; most other rows leave, and the novel-host arena's compaction keeps the parked entries by those flags; the
    parked jobs are then requeued with their lists."""
    tw = Twin()
    try:
        jobs = list(range(2, 1002, 2))
        tw.apply(0, up=[(j, prow(novel=[j % 40, (j + 1) % 40])) for j in jobs])
        park = jobs[:100]
        tw.retry_facts(0, park, [3] * 100, [0] * 100, [[] for _ in park])
        tw.launch(0, park, [10 ** 6 + j for j in park], [START] * 100, [7] * 100)
        more = list(range(2000, 5000, 2))             # 2000 slots: the table doubles
        tw.apply(0, up=[(j, prow(novel=[j % 40])) for j in more])
        tw.retry_facts(0, [more[0]], [3], [0], [[]])
        tw.launch(0, [more[0]], [10 ** 7], [START], [8])
        tw.check()
        tw.apply(0, rm=sorted(set(jobs[100:] + more[1:])))   # the dead novel entries pass the kept ones
        tw.check()
        tw.status(0, [10 ** 6 + j for j in park], [0] * 100, [START + 1000] * 100)
        tw.check()
    finally:
        tw.close()
