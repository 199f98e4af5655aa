"""The rebalancer's rare branches against the oracle: wide decisions (more than 32 and 64 victims, 63-65 victim
users), the nearest walk-back over dead slots, hosts whose item count passes 64 during the walk, jobs placed and
preempted in the same cycle, the safe / min-diff thresholds and the sufficiency test at equality, and host and
victim ties under several CTA splits.  The cases are built in rebalance_edge_cases.py.

Without a GPU: every case reaches the condition it names (on the oracle).  With one: cook_rebalance,
cook_rebalance_trace and (cases A, C, D) cook_state_rebalance equal the oracle bit for bit.
"""
import os

import numpy as np
import pytest

import fold_ref as F
import rebalance_edge_cases as E
from cook_b200 import abi

CASES = E.catalogue()
ALL = [(n, rg) for n in CASES for rg in E.REGIMES]
STATE = [(n, rg) for n, rg in ALL if n[0] in "ACD"]
ids = lambda cases: [f"{n}-{rg}" for n, rg in cases]


def _args(r):
    return (r["running"], r["pending"], r["pending_job_id"], r["pending_priority"], r["hosts"], r["users"],
            r["params"])


def _dec_same(got, want):
    keys = ("pending_idx", "host", "victims")
    assert [tuple(d[k] for k in keys) for d in got] == [tuple(d[k] for k in keys) for d in want]
    for k in ("dru", "mem", "cpus", "gpus"):
        assert F.same_bits([d[k] for d in got], [d[k] for d in want]), k


# ---- the cases reach their paths (CPU, oracle) ---------------------------------------------------------------
def test_catalogue_size():
    """Every case stays small (at most about 20k tasks) and every family is there."""
    for name, b in CASES.items():
        for rg in E.REGIMES:
            r, _ = b(rg)
            assert r["running"].t.n <= 20_000, name
    assert {n[0] for n in CASES} == set("ABCDEFG")


@pytest.mark.parametrize("n_users,k", E.WIDE)
@pytest.mark.parametrize("regime", E.REGIMES)
def test_wide_reaches(oracle, regime, n_users, k):
    r, _ = E.wide(regime, n_users, k)
    d = oracle.rebalance(*_args(r))
    rep = E.replay(r, d)
    cl = r["claims"]
    assert [x["pending_idx"] for x in d] == [0, 1, 2]
    assert d[0]["host"] == cl["host"] and len(d[0]["victims"]) == k
    assert len(set(rep[0]["users"])) == min(k, n_users)
    if k > 64:
        assert len(d[0]["victims"]) >= 65
    # the next two jobs are searched against the re-folded users: each takes a task of a victim user
    for x in rep[1:]:
        assert len(x["users"]) == 1 and x["users"][0] in cl["victim_users"]


def test_wide_distinct_user_edges(oracle):
    """Decisions with exactly 63, 64 and 65 distinct victim users, at <= 64 and > 64 victims."""
    seen = set()
    for n_users, k in E.WIDE:
        r, _ = E.wide("grid", n_users, k)
        rep = E.replay(r, oracle.rebalance(*_args(r)))
        seen.add((len(set(rep[0]["users"])), len(rep[0]["users"]) > 64))
    assert {(63, False), (64, False), (65, True), (1, True), (40, True)} <= seen


@pytest.mark.parametrize("k", [45, 70])
@pytest.mark.parametrize("regime", E.REGIMES)
def test_walkback_reaches(oracle, regime, k):
    r, _ = E.walkback(regime, k)
    tr = oracle.rebalance_trace(*_args(r), forced=None, forced_only=False)
    d = tr["decisions"]
    assert d[0]["pending_idx"] == 0 and len(d[0]["victims"]) == k
    assert tr["below_quota"][:2] == [False, False]
    assert E.walkback_dead(r, d) == k > 32
    assert not np.isnan(tr["pending_dru"][1])


@pytest.mark.parametrize("regime", E.REGIMES)
def test_crowded_reaches(oracle, regime):
    r, _ = E.crowded(regime)
    d = oracle.rebalance(*_args(r))
    rep = E.replay(r, d)
    h63, h64, h65 = r["claims"]["hosts"]
    items = np.array([x["items"] for x in rep])
    for h, n in ((h63, 63), (h64, 64), (h65, 65)):
        assert items[0, h] == n
    # searches of the host of 64 tasks see 64 items and later 65; the host of 63 passes 64 as well
    assert 64 in items[:, h64] and 65 in items[:, h64] and 65 in items[:, h63]
    assert (items[:, h65] > 65).any()                       # more than 64 real tasks and a synthetic one
    # a decision on each crowded host after its count passed 64 takes a whole tie group (3 > the 2 needed)
    for h in (h63, h64, h65):
        assert any(x["host"] == h and len(x["victims"]) == 3 and rep[i]["items"][h] > 64 for i, x in enumerate(d))


@pytest.mark.parametrize("crowd", [0, 70])
@pytest.mark.parametrize("regime", E.REGIMES)
def test_same_cycle_reaches(oracle, regime, crowd):
    r, _ = E.same_cycle(regime, crowd)
    d = oracle.rebalance(*_args(r))
    R = r["running"].t.n
    assert [(x["pending_idx"], x["host"]) for x in d] == [(0, r["claims"]["host"]), (2, r["claims"]["host"])]
    assert d[1]["victims"] == [R + 0]                      # the task decision 0 placed
    assert (R + crowd > 64) == (crowd > 0)


def _rank_order(oracle, r):
    run, pend = r["running"].t, r["pending"]
    p = abi.make_tasks(user=pend.col("user"), priority=r["pending_priority"],
                       start_time=np.full(pend.n, abi.INT64_MAX, np.int64), task_id=np.full(pend.n, -1, np.int64),
                       job_id=r["pending_job_id"], cpus=pend.col("cpus"), mem=pend.col("mem"))
    return oracle.rank(run, p, r["users"])["ranked"].tolist()


@pytest.mark.parametrize("name", [n for n in CASES if n[0] in "ACD"])
def test_resident_arm_walks_the_same_order(oracle, name):
    """The resident arm walks the last rank's queue: for cases A, C and D it is the jobs' index order, so
    cook_state_rebalance reaches the same branches."""
    r, _ = CASES[name]("grid")
    assert _rank_order(oracle, r) == list(range(r["pending"].n))


@pytest.mark.parametrize("kind", ["safe", "diff"])
@pytest.mark.parametrize("pad", [0, 70])
@pytest.mark.parametrize("regime", E.REGIMES)
def test_thresholds_flip(oracle, regime, kind, pad):
    """The exact and the one-ulp variant of each threshold disagree on the victim's eligibility."""
    got = {}
    for edge in ("exact", "ulp"):
        r, _ = E.threshold(regime, kind, edge, pad)
        d = oracle.rebalance(*_args(r))
        assert bool(d) == r["claims"]["eligible"]
        if d:
            assert d[0]["victims"] == [r["claims"]["victim"]]
        got[edge] = len(d)
    assert got["exact"] != got["ulp"]
    r, _ = E.threshold(regime, kind, "exact", pad)
    cl = r["claims"]
    assert cl["pend"] * 2.0 >= cl["d"] >= cl["pend"] and F.exact_sum([cl["d"], -cl["pend"]]) == cl["d"] - cl["pend"]


@pytest.mark.parametrize("pad", [0, 70])
@pytest.mark.parametrize("regime", E.REGIMES)
def test_sufficiency_flips(oracle, regime, pad):
    """Request at the left fold of [spare ; k victims]: k victims; one ulp above: k + 1.  Off the grid another
    summation order of the same prefix gives other bits."""
    for edge in ("exact", "ulp"):
        r, _ = E.sufficiency(regime, edge, pad=pad)
        d = oracle.rebalance(*_args(r))
        assert len(d) == 1 and len(d[0]["victims"]) == r["claims"]["n"]
        assert F.same_bits([d[0]["mem"]], [F.left_total(r["claims"]["addends"][:1] + [
            r["case"].tasks[v]["mem"] for v in d[0]["victims"][::-1]])])
    if regime == "off":
        assert F.association_sensitive(r["claims"]["addends"])


@pytest.mark.parametrize("n_hosts", E.TIE_HOSTS)
@pytest.mark.parametrize("regime", E.REGIMES)
def test_ties_reach(oracle, regime, n_hosts):
    r, _ = E.ties(regime, n_hosts)
    d = oracle.rebalance(*_args(r))
    top = r["claims"]["top"]
    assert [x["host"] for x in d] == top
    assert all(0 < h < n_hosts - 1 for h in top)
    c = r["case"]
    dru = c.initial()[0]
    for x in d:                                             # every victim of the walk has the same DRU
        assert len({dru[v] for v in x["victims"]}) == 1
    # decision 0: (user name, later position first) -> ascending-DRU list is the reverse
    sel = d[0]["victims"][::-1]
    us = [c.tasks[v]["user"] for v in sel]
    w = r["claims"]["w"]
    assert us == sorted(us) and us.count(w) == 2 and len(set(us)) == 4
    iw = [v for v in sel if c.tasks[v]["user"] == w]
    assert iw[0] > iw[1]


# ---- GPU: the kernel against the oracle ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,regime", ALL, ids=ids(ALL))
def test_rebalance_equals_oracle(gpu, oracle, name, regime):
    r, _ = CASES[name](regime)
    _dec_same(gpu.rebalance(*_args(r)), oracle.rebalance(*_args(r)))


@pytest.mark.gpu
@pytest.mark.parametrize("name,regime", ALL, ids=ids(ALL))
def test_rebalance_trace_equals_oracle(gpu, oracle, name, regime):
    """The walk's state: the final priority-map order and its DRU bits (a wrong re-fold shows here even where the
    decisions agree), spare resources, pending DRU bits and job-below-quota."""
    r, _ = CASES[name](regime)
    tg = gpu.rebalance_trace(*_args(r), forced=None, forced_only=False)
    to = oracle.rebalance_trace(*_args(r), forced=None, forced_only=False)
    _dec_same(tg["decisions"], to["decisions"])
    assert tg["order"] == to["order"]
    assert F.same_bits(tg["order_dru"], to["order_dru"])
    assert sorted(tg["spare"]) == sorted(to["spare"])
    for h in to["spare"]:
        assert F.same_bits(tg["spare"][h], to["spare"][h]), h
    assert F.same_bits(np.nan_to_num(tg["pending_dru"], nan=-1.0), np.nan_to_num(to["pending_dru"], nan=-1.0))
    assert tg["below_quota"] == to["below_quota"]


@pytest.mark.gpu
@pytest.mark.parametrize("name,regime", STATE, ids=ids(STATE))
def test_state_rebalance_equals_oracle(oracle, name, regime):
    """The same rows through the resident state: victims as task ids, a synthetic one as -1 - e."""
    from test_state_rebalance import RPool, rows_of
    r, codes = CASES[name](regime)
    pend, run = rows_of(r, codes)
    p = RPool(r, codes)
    try:
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        assert p.rank() == [int(j) for j in r["pending_job_id"]]
        got = p.check(oracle)
        want = oracle.rebalance(*_args(r))
        tid = [t["task_id"] for t in r["case"].tasks]
        R = len(tid)
        assert [[int(tid[v]) if v < R else -1 - (v - R) for v in x["victims"]] for x in want] == \
               [x["victims"] for x in got]
        if name.startswith("D"):
            assert got[1]["victims"] == [-1]
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_hosts", E.TIE_HOSTS)
@pytest.mark.parametrize("regime", E.REGIMES)
def test_ties_under_cta_splits(gpu, oracle, regime, n_hosts):
    """Host ties across warps and CTAs: the same decisions whatever the CTAs per SM."""
    r, _ = E.ties(regime, n_hosts)
    want = oracle.rebalance(*_args(r))
    saved = os.environ.get("COOK_REB_CTAS_PER_SM")
    try:
        for v in (None, "1", "2", "3"):
            os.environ.pop("COOK_REB_CTAS_PER_SM", None)
            if v is not None:
                os.environ["COOK_REB_CTAS_PER_SM"] = v
            _dec_same(gpu.rebalance(*_args(r)), want)
    finally:
        os.environ.pop("COOK_REB_CTAS_PER_SM", None)
        if saved is not None:
            os.environ["COOK_REB_CTAS_PER_SM"] = saved


@pytest.mark.gpu
@pytest.mark.parametrize("regime", E.REGIMES)
def test_padding_moves_a_host_to_the_slow_path(gpu, regime):
    """Metamorphic: ineligible tasks padded onto case C's host of 63 tasks (slow path from the start) leave every
    decision as it was; a synthetic victim's index moves by the padding."""
    pad = 3
    (r0, _), (r1, _) = E.crowded(regime), E.crowded(regime, pad=pad)
    R = r0["running"].t.n
    assert r1["running"].t.n == R + pad
    d0, d1 = gpu.rebalance(*_args(r0)), gpu.rebalance(*_args(r1))
    assert len(d0) == 12
    for x in d0:
        x["victims"] = [v if v < R else v + pad for v in x["victims"]]
    _dec_same(d1, d0)
