"""-m gpu: the resident pool state (cook_state_apply / cook_state_rank / cook_state_match).

A Python model keeps the same rows as the handle; after every batch the resident rank and match must
equal cook_rank / cook_match run on host tables built from the model (and rank the oracle), whatever the
slot layout, across capacity doublings and arena compactions.  Plus the upload accounting and the
all-or-nothing errors.
"""
import numpy as np
import pytest

from cook_b200 import abi, traces
from cook_b200.engine import CookError
import fold_ref as F
import rank_quota_cases as Q
from resident_model import START, Pool, c2, c3, churn, delta, drop_all_but, nb, pool_rows

pytestmark = pytest.mark.gpu

@pytest.mark.parametrize("kind", ["c2", "c3"])
def test_equivalence_random_deltas(kind, oracle):
    t = c2(11) if kind == "c2" else c3(13)
    p = Pool.of_trace(t, t.get("groups"))
    try:
        pend, run = pool_rows(t)
        items = sorted(pend.items())
        rng = np.random.default_rng(5)
        cut = int(len(items) * 0.85)
        reserve = items[cut:]
        p.apply(up=items[:cut], run_up=list(run.values()), reset=True)
        t_next = [10 ** 9]
        for cycle in range(5):
            p.check_rank(oracle if cycle % 2 == 0 else None)
            launched = []
            for rnd in range(2):                     # two match rounds per rank, a kill between rank and match
                live_q = [j for j in p.queue if j not in p.gone]
                if live_q:
                    p.apply(rm=[live_q[int(rng.integers(len(live_q)))]])
                got = p.check_match()
                launched = [int(j) for j, a in zip(got["considerable"], got["assign"]) if a >= 0][:40]
                up, rm, run_up, run_rm = churn(p, rng, reserve, t_next, launched)
                p.apply(up, rm, run_up, run_rm)
            if cycle == 3:                            # new leadership
                pend_now = sorted(p.pend.items())
                run_now = list(p.run.values())
                p.apply(up=pend_now, run_up=run_now, reset=True)
                with pytest.raises(CookError):       # nothing survives a reset: old ids are unknown to removals
                    p.gpu.state_apply(delta(rm=[10 ** 12]))
        p.check_rank(oracle)
        p.check_match()
    finally:
        p.close()


def test_layout_independence(oracle):
    t = c2(21, cpus=(0.1, 0.5, 1.0, 2.0))           # off the binary grid: the serial folds run
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    a, b = Pool.of_trace(t), Pool.of_trace(t)
    try:
        a.apply(up=items, run_up=list(run.values()))
        rng = np.random.default_rng(3)
        perm = rng.permutation(len(items))
        junk = [(10 ** 11 + i, items[i][1]) for i in range(500)]
        b.apply(up=junk)                              # churn that frees slots the real rows then reuse
        b.apply(rm=[j for j, _ in junk])
        b.apply(up=[items[i] for i in perm[: len(perm) // 2]])
        rr = list(run.values())
        b.apply(up=[items[i] for i in perm[len(perm) // 2:]], run_up=[rr[i] for i in rng.permutation(len(rr))])
        qa, qb = a.check_rank(), b.check_rank()
        assert np.array_equal(qa, qb)
        ma, mb = a.check_match(), b.check_match()
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
        # a pool quota on the last bit of the running fold: the same cut on both layouts, the oracle's
        q = qa.tolist()
        for k in (37, F.QF_CH + 1):
            at = a.quota_at(q, "cpus", k)
            for quota, n in ((at, k), (np.nextafter(at, -np.inf), k - 1)):
                pq = Q.pool_quota("cpus", quota)
                ra, rb = a.check_rank(oracle, pool_quota=pq), b.check_rank(oracle, pool_quota=pq)
                assert len(ra) == n and np.array_equal(ra, rb), (k, quota)
        ma, mb = a.check_match(), b.check_match()
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
    finally:
        a.close()
        b.close()


def test_pool_quota_through_churn(oracle):
    """Slot orders that churn leaves: running rows removed and upserted again (they refill the freed slots last in,
    first out), growth past a capacity doubling, launches into freed running slots.  After every step the rank with
    a pool quota on the last bit of the model's running fold (off the grid) equals cook_rank's and the oracle's on
    task-id tables, and the match over that queue equals cook_match's."""
    c = Q.build("off")
    run = c["run"]
    rng = np.random.default_rng(17)
    order = rng.permutation(len(run))
    first, later = order[:700], order[700:]          # 700 rows fit the first 1024 slots; 1200 do not
    p = Pool("quota-churn", drop=drop_all_but("gpus"), users=c["users"], offers=Q.offers(),
             params=traces.match_params(300))
    try:
        def check(k):
            q = p.check_rank(oracle).tolist()
            for col in ("cpus", "mem"):
                at = p.quota_at(q, col, k)
                for quota, n in ((at, k), (np.nextafter(at, -np.inf), k - 1)):
                    assert len(p.check_rank(oracle, pool_quota=Q.pool_quota(col, quota))) == n, (col, k, quota)
            p.check_match()

        def reinsert(n):
            tids = [int(t) for t in rng.choice(sorted(p.run), n, replace=False)]
            rows = [p.run[t] for t in tids]
            p.apply(run_rm=tids)
            p.apply(run_up=[rows[i] for i in rng.permutation(n)])

        def launch(n, tid0):
            p.apply(run_rm=[int(t) for t in rng.choice(sorted(p.run), n, replace=False)])
            jobs = [int(j) for j in rng.choice(sorted(p.pend), n, replace=False)]
            tids = tid0 + 4 * rng.permutation(n)      # even: the case's task ids are odd
            p.launch(jobs, tids, START + rng.integers(0, 10 ** 6, n))

        p.apply(up=c["pend"], run_up=[run[i] for i in first])
        check(37)
        reinsert(200)
        check(F.QF_CH)
        p.apply(run_up=[run[i] for i in later])
        check(F.QF_CH + 1)
        launch(150, 2 * 10 ** 7)
        check(37)
        reinsert(300)
        launch(100, 10 ** 8)
        check(F.QF_CH)
    finally:
        p.close()


def test_growth_and_compaction():
    t = c3(31)
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    p = Pool.of_trace(t, t.get("groups"))
    try:
        hosts = t["offers"].col("hostname_id")
        for i in range(0, len(items), 300):           # from empty past several capacity doublings
            p.apply(up=items[i:i + 300])
            if i % 900 == 0:
                p.check_rank()
                p.check_match()
        p.apply(run_up=list(run.values()))
        p.check_rank()
        p.check_match()
        long_rows = []
        for k, (j, r) in enumerate(items[:400]):      # long novel-host lists, upserted then removed
            r = dict(r)
            r["novel"] = hosts[(np.arange(60) * 7 + k) % len(hosts)].tolist()
            long_rows.append((j, r))
        p.apply(up=long_rows)
        p.check_rank()
        p.check_match()
        p.apply(rm=[j for j, _ in long_rows[:300]])   # dead entries now outnumber the live ones
        p.apply(up=[items[k] for k in range(300, 400)])
        p.check_rank()
        p.check_match()
    finally:
        p.close()


@pytest.mark.parametrize("scale", [1, 2])
def test_accounting(scale):
    t = traces.gen_pool(41, 2000 * scale, 150, 20, 400 * scale)
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    p = Pool.of_trace(t)
    try:
        d = delta(up=items, run_up=list(run.values()))
        p.gpu.state_apply(d)
        p.mirror(items, (), list(run.values()))
        pj, rt = d.col("pending"), d.col("running")
        lists = {"novel_host": "novel_off", "attr_col": "attr_off", "attr_val": "attr_off", "group_idx": "group_off"}
        want = sum(4 * int(pj.col(lists[n])[-1]) if n in lists else pj.col(n).nbytes
                   for n, _ in pj._fields_ if isinstance(pj.col(n), np.ndarray))   # a list uploads its entries
        want += nb(d.col("pending_priority"), d.col("pending_job_id"), *[rt.col(n) for n, _ in rt._fields_])
        want += 4 * (pj.n + rt.n)                      # one slot per row
        st = p.gpu.last_stats(abi.PHASE_STATE)
        assert st["h2d_bytes"] == want and st["n_launches"] >= 2
        p.check_rank()
        u = t["users"]
        rk = p.gpu.last_stats(abi.PHASE_RANK)
        assert rk["h2d_bytes"] == nb(*[u.col(n) for n in ("name_rank", "div_mem", "div_cpus", "div_gpus",
                                                            "quota_count", "quota_cpus", "quota_mem", "quota_gpus")])
        assert rk["n_launches"] > 0
        got = p.check_match()
        o = t["offers"]
        # name_rank stays on the host; the offer order it gives (O int32) is uploaded instead
        want = nb(*[o.col(n) for n, _ in o._fields_]) + nb(*[u.col(n) for n in (
            "quota_count", "quota_cpus", "quota_mem", "quota_gpus", "usage_count", "usage_cpus", "usage_mem",
            "usage_gpus", "tokens")])
        assert got["stats"]["h2d_bytes"] == want      # the same at scale 1 and 2: nothing per resident job
        assert got["stats"]["n_launches"] > 0
        # a launch batch uploads its own rows only
        j = int(got["considerable"][0])
        r = p.pend[j]
        task = dict(user=r["user"], priority=r["priority"], start_time=1, task_id=7, job_id=j, cpus=r["cpus"],
                    mem=r["mem"], gpus=r["gpus"])
        d = delta(rm=[j], run_up=[task])
        p.gpu.state_apply(d)
        assert p.gpu.last_stats(abi.PHASE_STATE)["h2d_bytes"] == nb(*[d.col("running").col(n) for n, _ in
                                                                         abi.TasksSoA._fields_]) + 4 + 4
    finally:
        p.close()


def test_errors():
    t = c3(51)
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    p = Pool.of_trace(t, t["groups"])
    try:
        with pytest.raises(CookError) as e:           # match before any rank
            p.gpu.state_match(p.offers, p.users, p.params, groups=p.groups)
        assert e.value.code == abi.COOK_E_BADARG
        p.apply(up=items, run_up=list(run.values()))
        q0 = p.check_rank()

        def fails(fn, code=abi.COOK_E_BADARG):
            with pytest.raises(CookError) as e:
                fn()
            assert e.value.code == code
            assert np.array_equal(p.gpu.state_rank(p.users), q0)

        fails(lambda: p.gpu.state_apply(delta(rm=[items[0][0], 10 ** 12])))          # unknown id
        fails(lambda: p.gpu.state_apply(delta(up=[items[1]], rm=[items[1][0]])))      # an id twice
        fails(lambda: p.gpu.state_apply(delta(up=[items[2], items[2]])))
        bad = delta(up=items[3:5])
        bad.col("pending").col("novel_off")[1] = -1                                   # malformed CSR
        fails(lambda: p.gpu.state_apply(bad))
        nu = p.users.n_users
        r = dict(items[5][1]); r["user"] = nu
        p.apply(up=[(10 ** 12, r)])                    # a user code the user table does not cover
        with pytest.raises(CookError) as e:
            p.gpu.state_rank(p.users)
        assert e.value.code == abi.COOK_E_BADARG
        p.apply(rm=[10 ** 12])
        assert np.array_equal(p.gpu.state_rank(p.users), q0)
        G = p.groups.n_groups
        r = dict(items[6][1]); r["groups"] = [G]       # a group code the groups table does not cover
        p.apply(up=[(10 ** 12 + 1, r)])
        with pytest.raises(CookError) as e:
            p.gpu.state_match(p.offers, p.users, p.params, groups=p.groups)
        assert e.value.code == abi.COOK_E_BADARG
        p.apply(rm=[10 ** 12 + 1])
        prm = traces.match_params(100, reuse_resident=1)
        fails(lambda: p.gpu.state_match(p.offers, p.users, prm, groups=p.groups))
        p.check_rank()
        p.check_match()
    finally:
        p.close()
