"""-m gpu: the switches between the exact-grid and the serial paths of the f64 running sums, reached
through the C ABI and compared with the CPU oracle.

Every trace has exact per-user task counts at the chunk and tile edges (fold_ref.edge_counts) and runs
under three amount regimes:
  grid   on the grid: the order-wide scan and the parallel per-user scans;
  off    off the grid: the serial chain everywhere;
  mixed  on the grid, but one long user's amounts near 2^32: the order-wide total passes 2^43, so the
         same launch takes the parallel scan for the short users and the chain for the long one.
"""
import numpy as np
import pytest

import fold_ref as R
from cook_b200 import abi, sharding, traces

pytestmark = pytest.mark.gpu

REGIMES = ["grid", "off", "mixed"]
_POOLS = {}


def _pool(regime):
    if regime not in _POOLS:
        _POOLS[regime] = R.fold_pool(regime, 7)
    return _POOLS[regime]


def _same_dru(a, b):
    return R.same_bits(np.nan_to_num(a, nan=-1.0), np.nan_to_num(b, nan=-1.0))


def _user_quota(t, frac):
    """Per-user quotas at a fraction of each user's own pending + running totals (left folds), so they
    bind inside the users' segments; off the grid in the 'off' regime."""
    U = t["n_users"]
    c = t["cols"]
    tot = {k: np.zeros(U) for k in ("count", "cpus", "mem")}
    for part in (c["run"], c["pend"]):
        for i in range(len(part["user"])):
            u = part["user"][i]
            tot["count"][u] += 1.0
            tot["cpus"][u] = tot["cpus"][u] + part["cpus"][i]
            tot["mem"][u] = tot["mem"][u] + part["mem"][i]
    return {"count": np.floor(tot["count"] * frac) + 1.0, "cpus": tot["cpus"] * frac,
            "mem": tot["mem"] * (frac + 0.1), "gpus": np.full(U, 1e9)}


def _queue_cut(ranked, t, k):
    """cpus of the ranked queue folded up to position k: a quota that binds right there."""
    return R.left_total(t["cols"]["pend"]["cpus"][ranked[:k]])


def test_the_traces_reach_the_path_switches():
    """The regimes do what their names say (host-side restatement of grid_check + grid_exact)."""
    for regime in REGIMES:
        t = _pool(regime)
        c = t["cols"]
        cpus = np.concatenate([c["run"]["cpus"], c["pend"]["cpus"]])
        mem = np.concatenate([c["run"]["mem"], c["pend"]["mem"]])
        flag = R.grid_flag(cpus, mem, None)
        n = len(cpus)
        counts = c["counts"]
        per_user = [R.grid_exact(flag, k) for k in counts]
        if regime == "grid":
            assert R.grid_exact(flag, n) and all(per_user)
        elif regime == "off":
            assert flag[0] == 1
        else:
            assert not R.grid_exact(flag, n) and any(per_user) and not all(per_user)


@pytest.mark.parametrize("regime", REGIMES)
def test_rank_paths(gpu, oracle, regime):
    """DRU fold, pool and group quota filters (cutting at and around the 1024-entry chunk edge of the
    quota kernel) and max_over_quota cutting inside a user's chunk: ranked, order and DRU bits."""
    t = _pool(regime)
    users = R.build_pool(t["cols"], user_quota=_user_quota(t, 0.45))["users"]
    prm = abi.RankParams(5, 1, 30000.0 if regime != "mixed" else 2.0 ** 33, 6.0)   # the long user stays
    base = oracle.rank(t["running"], t["pending"], users, params=prm)
    assert len(base["ranked"]) > R.QF_CH + 40
    run_cpus = R.left_total(t["cols"]["run"]["cpus"])   # the pool quota counts the running tasks
    gu = np.array([3.0, 0.7, 11.0 / 7.0, 0.0]) if regime == "off" else np.array([3.0, 0.5, 1024.0, 0.0])
    for k in (R.QF_CH - 1, R.QF_CH, R.QF_CH + 1):
        pool_cut = run_cpus + _queue_cut(base["ranked"], t, k)
        pq = abi.make_pool_quota({"count": 1e12, "cpus": pool_cut, "mem": 1e18, "gpus": 1e12})
        group_cut = R.left_total(t["cols"]["pend"]["cpus"][base["ranked"][:k + 30]], gu[1])
        gq = abi.make_pool_quota({"count": 1e12, "cpus": group_cut, "mem": 1e18, "gpus": 1e12})
        for kw in (dict(pool_quota=pq), dict(group_quota=gq, group_usage=gu),
                   dict(pool_quota=pq, group_quota=gq, group_usage=gu)):
            rg = gpu.rank(t["running"], t["pending"], users, params=prm, **kw)
            ro = oracle.rank(t["running"], t["pending"], users, params=prm, **kw)
            assert np.array_equal(rg["ranked"], ro["ranked"]), (k, list(kw))
            assert np.array_equal(rg["order"], ro["order"]), (k, list(kw))
            assert _same_dru(rg["dru"], ro["dru"]), (k, list(kw))
            assert 0 < len(ro["ranked"]) < len(base["ranked"])


@pytest.mark.parametrize("regime", REGIMES)
def test_rank_group_usage_off_the_grid(gpu, oracle, regime):
    """An off-grid group usage (the start value of the group filter) with on- or off-grid addends."""
    t = _pool(regime)
    base = oracle.rank(t["running"], t["pending"], t["users"])
    gu = np.array([1.0 / 3.0, 0.1, 1.0 / 7.0, 0.0])
    for k in (R.QF_CH - 1, R.QF_CH + 1, 3 * R.QF_CH):
        group_cut = R.left_total(t["cols"]["pend"]["cpus"][base["ranked"][:k]], gu[1])
        gq = abi.make_pool_quota({"count": 1e12, "cpus": group_cut, "mem": 1e18, "gpus": 1e12})
        rg = gpu.rank(t["running"], t["pending"], t["users"], group_quota=gq, group_usage=gu)
        ro = oracle.rank(t["running"], t["pending"], t["users"], group_quota=gq, group_usage=gu)
        assert np.array_equal(rg["ranked"], ro["ranked"]) and _same_dru(rg["dru"], ro["dru"]), k
        assert 0 < len(ro["ranked"]) < len(base["ranked"])


def _match_both(gpu, oracle, t, users, ranked, prm, pq=None):
    mg = gpu.match(ranked, t["jobs"], t["offers"], users, prm, pool_quota=pq)
    mo = oracle.match(ranked, t["jobs"], t["offers"], users, prm, pool_quota=pq)
    assert np.array_equal(mg["considerable"], mo["considerable"])
    assert mg["stats"]["n_considerable"] == mo["stats"]["n_considerable"]
    assert np.array_equal(mg["assign"], mo["assign"])
    return mg, mo


@pytest.mark.parametrize("regime", REGIMES)
def test_considerable_paths(gpu, oracle, regime):
    """User quotas (the users' running usage is the start of their folds), the launch-rate limit, with
    and without a pool quota, and a cap below the survivor count: considerable set, count and
    assignments equal the oracle's."""
    t = _pool(regime)
    rng = np.random.default_rng(3)
    U = t["n_users"]
    tokens = rng.integers(0, 200, U).astype(np.int32)
    users = R.build_pool(t["cols"], user_quota=_user_quota(t, 0.6), tokens=tokens)["users"]
    ranked = oracle.rank(t["running"], t["pending"], users)["ranked"]
    J = len(ranked)
    usage = t["usage"]
    pq = abi.make_pool_quota({"count": 1e12, "cpus": R.left_total(usage["cpus"]) + _queue_cut(ranked, t, 1500),
                              "mem": 1e18, "gpus": 1e12})
    for enforce in (0, 1):
        survivors = oracle.match(ranked, t["jobs"], t["offers"], users, traces.match_params(J, enforce))
        n_surv = survivors["stats"]["n_considerable"]
        assert 0 < n_surv < J
        for cap in (n_surv, n_surv - 1, R.CP_BLOCK + 1, R.CP_BLOCK, 600):
            mg, _ = _match_both(gpu, oracle, t, users, ranked, traces.match_params(cap, enforce))
            assert mg["stats"]["n_considerable"] == min(cap, n_surv)
        for cap in (J, 700):
            _match_both(gpu, oracle, t, users, ranked, traces.match_params(cap, enforce), pq)


@pytest.mark.parametrize("regime", REGIMES)
def test_considerable_user_usage_off_the_grid(gpu, oracle, regime):
    """Off-grid running usage of every user (the start value of the per-user quota fold) with the
    regime's addends."""
    t = _pool(regime)
    U = t["n_users"]
    usage = {"count": np.arange(U, dtype=float), "cpus": np.full(U, 0.1) * np.arange(1, U + 1),
             "mem": np.arange(1, U + 1) / 7.0, "gpus": np.zeros(U)}
    users = R.build_pool(t["cols"], user_quota=_user_quota(t, 0.5), user_usage=usage)["users"]
    ranked = oracle.rank(t["running"], t["pending"], users)["ranked"]
    for cap in (len(ranked), 900):
        mg, _ = _match_both(gpu, oracle, t, users, ranked, traces.match_params(cap))
        assert 0 < mg["stats"]["n_considerable"] <= cap


@pytest.mark.parametrize("regime", REGIMES)
def test_usage_exchange_paths(gpu, oracle, regime):
    """cook_exchange_usage after a match round equals the host's np.add.at left fold in queue order:
    the exact kernel on the grid, the serial form off it and past 2^43.  Only the 'off' amounts make the
    order of the additions show in the bits (checked below); in 'mixed' the long user's jobs fit no
    offer, so the serial form runs over small on-grid amounts."""
    t = _pool(regime)
    ranked = oracle.rank(t["running"], t["pending"], t["users"])["ranked"]
    m = gpu.match(ranked, t["jobs"], t["offers"], t["users"], traces.match_params(len(ranked)))
    U = t["n_users"]
    got = gpu.exchange_usage(U + 5)[0]
    j = t["jobs"]
    want = sharding.usage_delta(m["considerable"], m["assign"], j.col("user"), j.col("cpus"), j.col("mem"),
                                j.col("gpus"), U)
    assert m["stats"]["n_matched"] > 0
    assert R.same_bits(got[:U], want) and not got[U:].any()
    if regime == "off":
        placed = m["considerable"][m["assign"] >= 0]
        assert R.segments_sensitive(j.col("mem")[placed], j.col("user")[placed])


def _reb_args(r, users=None):
    return (r["running"], r["pending"], r["pending_job_id"], r["pending_priority"], r["hosts"], users or r["users"],
            r["params"])


@pytest.mark.parametrize("regime", REGIMES)
def test_rebalance_paths(gpu, oracle, regime):
    """The rebalancer's DRU fold and next-state re-folds in a full search (no quotas: job-below-quota is
    skipped, test_job_below_quota_fold runs it)."""
    r = R.fold_rebalance(regime, 11)
    do = oracle.rebalance(*_reb_args(r))
    dg = gpu.rebalance(*_reb_args(r))
    assert len(do) > 0 and dg == do
    tg = gpu.rebalance_trace(*_reb_args(r), forced=None, forced_only=False)
    to = oracle.rebalance_trace(*_reb_args(r), forced=None, forced_only=False)
    assert R.same_bits(np.nan_to_num(tg["pending_dru"]), np.nan_to_num(to["pending_dru"]))
    assert tg["below_quota"] == to["below_quota"]


@pytest.mark.parametrize("regime,lead_mem_offset", [("grid", 0.0), ("off", 0.0), ("mixed", 0.0), ("grid", 1 / 3),
                                                   ("mixed", 1 / 3)])
def test_job_below_quota_fold(gpu, oracle, regime, lead_mem_offset):
    """job-below-quota folds (pending mem, then the user's running tasks) for users of 0, 126, 127, 128,
    129 and 700 tasks, against mem quotas placed exactly on the left fold and one ulp under it, so the
    fold's last bit decides every answer.  lead_mem_offset 1/3 puts the pending request off the grid on
    top of on-grid running tasks (the pending columns feed the same grid flag, so the whole call then
    takes the serial chain).  below_quota, pending DRU bits and a full search's decisions equal the
    oracle's."""
    r = R.fold_rebalance(regime, 11, lead_mem_offset=lead_mem_offset)
    lead = r["lead"]
    forced = [(p, 0, [], 0.0, 0.0, 0.0) for p in range(len(lead))]   # distinct users: each fold sees the inputs
    for below in (True, False):
        users = R.quota_at_fold(r, below)
        tg = gpu.rebalance_trace(*_reb_args(r, users), forced=forced)
        to = oracle.rebalance_trace(*_reb_args(r, users), forced=forced)
        assert to["below_quota"][:len(lead)] == [below] * len(lead)
        assert tg["below_quota"] == to["below_quota"]
        assert R.same_bits(np.nan_to_num(tg["pending_dru"]), np.nan_to_num(to["pending_dru"]))
        do = oracle.rebalance(*_reb_args(r, users))
        assert gpu.rebalance(*_reb_args(r, users)) == do


def _forced(r):
    """Forced decisions: victims of several users on one host each; the new task's user has no running
    task (pending 0), or its task lands before (priority 90), inside (50) or after (10) the user's
    running tasks (pendings 1-3 of users with 129, 127 and 700 tasks)."""
    run, host = r["run"], r["host"]
    out = []
    for i, pidx in enumerate((0, 1, 2, 3)):
        h = int(np.bincount(host).argsort()[-1 - i])
        on_h = np.flatnonzero(host == h)
        vs, seen = [], set()
        for v in on_h:
            if run["user"][v] not in seen or len(vs) < 2:
                vs.append(int(v))
                seen.add(run["user"][v])
            if len(vs) == 4:
                break
        mem = R.left_total(run["mem"][vs]) * r["mem_scale"]
        cpus = R.left_total(run["cpus"][vs])
        out.append((pidx, h, vs, mem, cpus, 0.0))
    return out


@pytest.mark.parametrize("regime", REGIMES)
def test_next_state_refold(gpu, oracle, regime):
    """rebalance_trace with forced decisions: task DRU bits and the order after each next-state step
    equal the oracle's, the element-wise update on the grid and the warp re-fold elsewhere."""
    r = R.fold_rebalance(regime, 12)
    prio = np.array(r["pending_priority"]).copy()
    prio[1], prio[2], prio[3] = 90, 50, 10
    r["pending_priority"] = prio
    forced = _forced(r)
    users_of_victims = {int(r["run"]["user"][v]) for f in forced for v in f[2]}
    assert len(users_of_victims) >= 3
    for k in range(1, len(forced) + 1):
        tg = gpu.rebalance_trace(*_reb_args(r), forced=forced[:k])
        to = oracle.rebalance_trace(*_reb_args(r), forced=forced[:k])
        assert tg["order"] == to["order"], k
        assert R.same_bits(tg["order_dru"], to["order_dru"]), k
        assert tg["spare"] == to["spare"], k


def test_next_state_refold_after_an_element_wise_step(gpu, oracle):
    """A user of 126 tasks is updated element-wise (on the grid rule) when one of its tasks is a victim;
    a later step inserts a task of the same user right after that victim, which makes the segment too
    long for the rule, so the warp re-fold starts from the value the first step left in the victim's
    slot.  The new task's DRU shows whether the victim's own amount left that running sum."""
    r = R.fold_rebalance("mixed", 12)
    run, host = r["run"], r["host"]
    A = 9
    assert r["counts"][A] == 126 and int(np.asarray(r["pending"].col("user"))[4]) == A
    last = int(R.user_task_order(r, A)[-1])   # the last task of A's segment
    h = int(host[last])
    other = [int(i) for i in np.flatnonzero((host == h) & (run["user"] != A))[:2]]
    prio = np.array(r["pending_priority"]).copy()
    prio[4] = run["priority"][last]          # sorts after every running task of A: right after `last`
    r["pending_priority"] = prio
    vs = [last] + other
    forced = [(1, h, vs, R.left_total(run["mem"][vs]), R.left_total(run["cpus"][vs]), 0.0),
              (4, h, [], 0.0, 0.0, 0.0)]
    for k in (1, 2):
        tg = gpu.rebalance_trace(*_reb_args(r), forced=forced[:k])
        to = oracle.rebalance_trace(*_reb_args(r), forced=forced[:k])
        assert tg["order"] == to["order"], k
        assert R.same_bits(tg["order_dru"], to["order_dru"]), k


def _scaled_run(gpu, t, users, rank_kw, prm_m, pq):
    rg = gpu.rank(t["running"], t["pending"], users, **rank_kw)
    mg = gpu.match(rg["ranked"], t["jobs"], t["offers"], users, prm_m, pool_quota=pq)
    return rg, mg


def test_mem_scaled_by_2_pow_20(gpu):
    """Metamorphic: every mem quantity times 2^20 (task and pending mem, offers and their running mem,
    div_mem, mem quotas, usage, the offensive threshold).  The totals pass 2^43, so the kernels leave
    the order-wide scan, yet every partial sum stays exact: rank order, DRU bits, the considerable set,
    the assignments and the rebalancer's decisions equal the unscaled run, decision mem times 2^20."""
    S = 2.0 ** 20
    out = []
    for s in (1.0, S):
        t = R.fold_pool("grid", 7)
        t = R.build_pool(t["cols"], mem_scale=s, user_quota=_user_quota(t, 0.6))
        quota_mem = (R.left_total(t["cols"]["run"]["mem"]) + 0.25 * R.left_total(t["cols"]["pend"]["mem"])) * s
        pq = abi.make_pool_quota({"count": 1e12, "cpus": 1e12, "mem": quota_mem, "gpus": 1e12})
        rank_kw = dict(params=abi.RankParams(5, 1, 30000.0 * s, 6.0), pool_quota=pq)
        out.append(_scaled_run(gpu, t, t["users"], rank_kw, traces.match_params(5000), pq))
        if s == S:
            c = t["cols"]
            cpus = np.concatenate([c["run"]["cpus"], c["pend"]["cpus"]])
            mem = np.concatenate([c["run"]["mem"], c["pend"]["mem"]]) * s
            assert not R.grid_exact(R.grid_flag(cpus, mem, None), len(cpus))
    (r1, m1), (r2, m2) = out
    assert np.array_equal(r1["ranked"], r2["ranked"]) and np.array_equal(r1["order"], r2["order"])
    assert _same_dru(r1["dru"], r2["dru"])
    assert 0 < len(r1["ranked"]) < t["jobs"].n
    assert np.array_equal(m1["considerable"], m2["considerable"])
    assert np.array_equal(m1["assign"], m2["assign"])
    dec = []
    for s in (1.0, S):
        r = R.fold_rebalance("grid", 11, mem_scale=s)
        dec.append(gpu.rebalance(*_reb_args(r)))
    assert len(dec[0]) > 0 and len(dec[0]) == len(dec[1])
    for a, b in zip(*dec):
        assert (a["pending_idx"], a["host"], a["victims"], a["dru"], a["cpus"]) == \
               (b["pending_idx"], b["host"], b["victims"], b["dru"], b["cpus"])
        assert b["mem"] == a["mem"] * S
