"""The rank's pool quota on the last bit of its running fold, whatever slot order the resident rows sit in.

The pool quota filter starts from the pool's running usage, a left fold over the running tasks in ascending task id
(DESIGN §2), the fold cook_state_usage reports as the pool total.  Each case (rank_quota_cases.py) puts the quota
exactly on the fold of the first k queued jobs continued from that start, and one ulp under it, so a start one ulp
off moves the cut by one job.  CPU: the cases cut where they claim to on the oracle, a running table given in another
order moves the cut (so a fold in slot order cannot pass the GPU tests), and the quota group's given usage leaves no
room for the order.  GPU: a fresh handle loaded in each layout's order ranks as the oracle does on task-id tables,
with the pool quota alone, with the group quota too, with the offensive filter, and hands that queue to the match.
"""
import numpy as np
import pytest

import considerable_ref as CR
import fold_ref as F
import rank_quota_cases as Q
import resident_model as M
from cook_b200 import abi, traces

_CASES = {}


def case(regime):
    if regime not in _CASES:
        c = Q.build(regime)
        c["running"] = Q.running_table(c)
        c["pending"], c["jid"] = Q.pending_table(c)
        _CASES[regime] = c
    return _CASES[regime]


def base_queue(oracle, c):
    """The oracle's rank without a quota: pending indices in queue order."""
    if "base" not in c:
        c["base"] = oracle.rank(c["running"], c["pending"], c["users"])["ranked"]
    return c["base"]


def boundaries(c, base):
    """(column, k, cut position, q*) of every column and boundary."""
    out = []
    for col in Q.COLS:
        for k in Q.KS:
            kk = Q.cut(c, base, col, k)
            out.append((col, k, kk, Q.quota_at(c, base, col, kk)))
    return out


def below(q):
    return float(np.nextafter(q, -np.inf))


# ---- CPU: the cases and the witness ------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", Q.REGIMES)
def test_case_shape(regime):
    """The recorded seeds still give layouts above and below the task-id fold; the mixed case is on the grid but
    fails the rank's grid rule, and the off case's every column depends on the order."""
    c = case(regime)
    cols = Q.sensitive_cols(c)
    assert cols == (["cpus", "mem", "gpus"] if regime == "off" else ["cpus", "mem"])
    assert Q.side(c, Q.layout(c, "above"), cols) == 1
    assert Q.side(c, Q.layout(c, "below"), cols) == -1
    p = c["pending"]
    run = [np.array(Q.run_col(c, col)) for col in Q.COLS]
    amt = [np.concatenate([r, p.col(col)]) for r, col in zip(run, Q.COLS)]
    flag = F.grid_flag(*amt)
    if regime == "mixed":
        assert c["big"] >= 256 and flag[0] == 0
        assert not F.grid_exact(flag, len(amt[0]))
        assert all(Q.running_total(c, col) > F.LIMIT for col in ("cpus", "mem"))
    else:
        assert flag[0] == 1


@pytest.mark.parametrize("regime", Q.REGIMES)
def test_boundary_on_task_id_order(oracle, regime):
    """On running rows in task-id order the oracle keeps exactly the first k queued jobs at q* and k - 1 one ulp
    under it."""
    c = case(regime)
    base = base_queue(oracle, c)
    assert len(base) > F.QF_CH + 2
    for col, k, kk, q in boundaries(c, base):
        for quota, n in ((q, kk), (below(q), kk - 1)):
            got = oracle.rank(c["running"], c["pending"], c["users"], pool_quota=Q.pool_quota(col, quota))["ranked"]
            assert np.array_equal(got, base[:n]), (col, k, quota)


@pytest.mark.parametrize("layout", ["above", "below"])
@pytest.mark.parametrize("regime", Q.REGIMES)
def test_layout_moves_the_cut(oracle, regime, layout):
    """Given the running table in the layout's order, the oracle (a fold in input order) cuts elsewhere at one of the
    two quotas of every boundary: the witness that a fold in slot order cannot rank as the task-id fold does."""
    c = case(regime)
    base = base_queue(oracle, c)
    permuted = Q.running_table(c, Q.layout(c, layout))
    cols = Q.sensitive_cols(c)
    for col, k, kk, q in boundaries(c, base):
        if col not in cols:
            continue
        moved = False
        for quota in (q, below(q)):
            pq = Q.pool_quota(col, quota)
            a = oracle.rank(c["running"], c["pending"], c["users"], pool_quota=pq)["ranked"]
            b = oracle.rank(permuted, c["pending"], c["users"], pool_quota=pq)["ranked"]
            if not np.array_equal(a, b):
                moved = True
                assert abs(len(a) - len(b)) == 1 and np.array_equal(a[:min(len(a), len(b))], b[:min(len(a), len(b))])
        assert moved, (col, k)


@pytest.mark.parametrize("regime", Q.REGIMES)
def test_group_quota_is_layout_free(oracle, regime):
    """The quota group's usage is given, so the running order cannot matter: the same cut for every layout."""
    c = case(regime)
    base = base_queue(oracle, c)
    gu = Q.group_usage(c)
    tables = [Q.running_table(c, Q.layout(c, name)) for name in Q.LAYOUTS]
    for col, k, kk, q in boundaries(c, base):
        for quota, n in ((q, kk), (below(q), kk - 1)):
            for running in tables:
                got = oracle.rank(running, c["pending"], c["users"], group_quota=Q.pool_quota(col, quota),
                                  group_usage=gu)["ranked"]
                assert np.array_equal(got, base[:n]), (col, k, quota)


# ---- GPU: the resident rank in every layout ----------------------------------------------------------------------
def _pool(c, layout, name):
    p = M.Pool(name, drop=M.drop_all_but("gpus"), users=c["users"], offers=Q.offers(),
               params=traces.match_params(300))
    p.apply(up=c["pend"], run_up=[c["run"][i] for i in Q.layout(c, layout)])
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("layout", Q.LAYOUTS)
@pytest.mark.parametrize("regime", Q.REGIMES)
def test_state_rank_pool_quota(oracle, regime, layout):
    """state_rank with a pool quota on the last bit equals the oracle and cook_rank on task-id tables; with the
    group quota too; with the offensive filter (queue and offensive list); the start value is state_usage's pool
    total bit for bit; and the match over the cut queue equals cook_match's."""
    c = case(regime)
    base = base_queue(oracle, c)
    p = _pool(c, layout, f"rank-quota-{regime}-{layout}")
    try:
        running, pending, jobs, jid = p.tables()
        assert np.array_equal(jid, c["jid"])
        users = c["users"]
        gu = Q.group_usage(c)
        pool = p.gpu.state_usage(users.n_users)["pool"]
        assert F.same_bits(pool, gu), "state_usage's pool total != the task-id fold"
        cpus, mem = jobs.col("cpus"), jobs.col("mem")
        caps = (float(np.quantile(mem, 0.8)), float(np.quantile(cpus, 0.9)))
        prm_off = abi.RankParams(100, 1, caps[0], caps[1])
        for col, k, kk, q in boundaries(c, base):
            ci = 1 + Q.COLS.index(col)
            assert F.bits(Q.quota_at(c, base, col, kk, start=pool[ci])) == F.bits(q)
            for quota, n in ((q, kk), (below(q), kk - 1)):
                where = (col, k, quota)
                pq = Q.pool_quota(col, quota)
                gq_slack = Q.pool_quota(col, Q.quota_at(c, base, col, Q.cut(c, base, col, kk + 1)))
                for kw in (dict(pool_quota=pq), dict(pool_quota=pq, group_quota=gq_slack, group_usage=gu),
                           dict(group_quota=pq, group_usage=gu)):
                    want = oracle.rank(running, pending, users, **kw)["ranked"]
                    assert len(want) == n, where
                    got = p.rank(**kw)
                    assert np.array_equal(got, jid[want]), (where, sorted(kw), len(got), n)
                    host = p.ref.rank(running, pending, users, **kw)["ranked"]
                    assert np.array_equal(host, want), (where, sorted(kw))
                want = oracle.rank(running, pending, users, pool_quota=pq, params=prm_off)["ranked"]
                got, off = p.gpu.state_rank(users, pool_quota=pq, params=prm_off, offensive=True)
                assert np.array_equal(got, jid[want]), (where, "offensive")
                wo = CR.offensive(base[:n].tolist(), cpus, mem, caps[0], caps[1])
                assert off.tolist() == [int(jid[i]) for i in wo], (where, "offensive list")
            if k == F.QF_CH:     # the match downstream of a cut queue
                p.rank(pool_quota=Q.pool_quota(col, q))
                assert len(p.queue) == kk
                p.check_match()
    finally:
        p.close()
