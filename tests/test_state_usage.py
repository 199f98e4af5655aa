"""cook_state_usage: the running usage per user, of the pool and per host, folded on the device from the
resident running rows, each sum a left fold in ascending task id.

CPU: the restatement in usage_ref.py against plain folds, the order sensitivity of the off-grid tables, the
known answer of aggregate-quota-groups, the export and the phase code.
GPU (-m gpu): bit equality with the restatement after every batch of a churn (apply, launch with and without
hosts, finishes, a reset, capacity doubling, arena compaction) on and off the grid and on a table that mixes
both paths; independence from the slot layout; the host edges; a resident match fed from the derived columns
against cook_match and the oracle on host tables; the errors and the upload accounting.
"""
import numpy as np
import pytest

import fold_ref as F
from cook_b200 import abi, engine
from resident_model import START, Pool, amounts, drop_all_but, keyed, pending_rows, random_rows, tasks_soa
from usage_ref import KEYS, aggregate_quota_groups, running_usage

def plain_fold(rows, key, order):
    """The sum of `key` over rows in `order` (a list of rows), one float addition each."""
    return F.left_total([r[key] for r in order])


# ---- CPU -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["grid", "off", "mixed"])
@pytest.mark.parametrize("seed", [1, 2])
def test_restatement_is_the_ascending_task_id_fold(regime, seed):
    rng = np.random.default_rng(seed)
    U, codes = 9, list(range(12))
    rows = random_rows(rng, regime, 700, U, 1000, codes + [-1, 40, 41])
    listed = rng.permutation(codes + [90, 91])[:11]
    got = running_usage(rows, U, listed)
    by_tid = sorted(rows, key=lambda r: r["task_id"])
    for u in range(U):
        mine = [r for r in by_tid if r["user"] == u]
        assert got["user"]["count"][u] == float(len(mine))
        for k in ("cpus", "mem", "gpus"):
            assert F.bits(got["user"][k][u]) == F.bits(plain_fold(rows, k, mine)), (u, k)
    for j, k in enumerate(KEYS[1:], 1):
        assert F.bits(got["pool"][j]) == F.bits(plain_fold(rows, k, by_tid))
    assert got["pool"][0] == float(len(rows))
    for h, c in enumerate(listed):
        mine = [r for r in by_tid if r["host"] == c]
        assert got["run_count"][h] == len(mine)
        assert F.bits(got["run_cpus"][h]) == F.bits(plain_fold(rows, "cpus", mine))
        assert F.bits(got["run_mem"][h]) == F.bits(plain_fold(rows, "mem", mine))


@pytest.mark.parametrize("regime", ["off", "mixed"])
def test_off_grid_tables_see_the_order(regime):
    """The tables the GPU tests use off the grid would catch another order: the fold in slot (input) order or a
    pairwise sum gives other bits for some user, the pool or some host."""
    rng = np.random.default_rng(7)
    rows = random_rows(rng, regime, 1000, 9, 1000, list(range(12)))   # mixed: user 0 passes 2^43
    by_tid = sorted(rows, key=lambda r: r["task_id"])
    slot, pair = False, False
    groups = [by_tid] + [[r for r in by_tid if r["user"] == u] for u in range(9)] + \
        [[r for r in by_tid if r["host"] == c] for c in range(12)]
    for g in groups:
        ids = {id(r) for r in g}
        in_input = [r for r in rows if id(r) in ids]
        for k in ("cpus", "mem"):
            want = F.bits(plain_fold(rows, k, g))
            slot |= F.bits(plain_fold(rows, k, in_input)) != want
            pair |= F.bits(F.pairwise_sum([r[k] for r in g])) != want
    assert slot and pair


def test_aggregate_quota_groups_known_answer():
    """test-aggregate-quota-groups (reference test/cook/test/scheduler/scheduler.clj:222-230): pools a-d whose
    running rows add up to the given usages, grouped {"a" "s", "b" "s"}, give {"s" {:count 300 :cpus 30 :mem 3}}."""
    want = {"a": (100, 10, 1), "b": (200, 20, 2), "c": (400, 40, 4), "d": (800, 80, 8)}
    totals = {}
    for p, (n, c, m) in want.items():
        rows = [dict(user=0, task_id=7 * i + 3, cpus=1.0 if i < c else 0.0, mem=1.0 if i < m else 0.0, host=-1)
                for i in range(n)]
        totals[p] = running_usage(rows, 1)["pool"]
        assert totals[p].tolist() == [float(n), float(c), float(m), 0.0]
    got = aggregate_quota_groups({"a": "s", "b": "s"}, totals)
    assert list(got) == ["s"]
    assert got["s"].tolist() == [300.0, 30.0, 3.0, 0.0]


# ---- GPU -------------------------------------------------------------------------------------------------
def new_handle(name="usage"):
    """A resident handle whose pending upserts carry user, amounts and novel hosts only, and its model."""
    return Pool(name, drop=drop_all_but("gpus", "novel"), send_hosts=True)


def check(h, U, listed):
    got = h.gpu.state_usage(U, listed)
    want = running_usage(h.run.values(), U, listed)
    for k in KEYS:
        assert F.same_bits(got["user"][k], want["user"][k]), k
    assert F.same_bits(got["pool"], want["pool"])
    assert F.same_bits(got["run_cpus"], want["run_cpus"]) and F.same_bits(got["run_mem"], want["run_mem"])
    assert np.array_equal(got["run_count"], want["run_count"])
    st = h.gpu.last_stats(abi.PHASE_USAGE)
    assert st["h2d_bytes"] == (4 * len(listed) if h.run else 0)
    assert st["d2h_bytes"] == (32 * U + 32 + 20 * len(listed) if h.run else 0)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["grid", "off", "mixed"])
def test_churn_matches_the_fold(regime):
    rng = np.random.default_rng({"grid": 11, "off": 12, "mixed": 13}[regime])
    U, codes = 40, list(range(60))
    listed = np.array(rng.permutation(list(range(50)) + [200, 201, 202]), np.int32)   # 50..59 unlisted, 200.. empty
    hosts = codes + [7] * 30 + [-1] * 5   # host 7 carries more than 64 rows
    h = new_handle()
    tid, jid = [1_000], [5_000_000]

    def fresh_rows(n):
        rows = random_rows(rng, regime, n, U, tid[0], hosts)
        tid[0] += 2 * n + 2
        return rows

    def fresh_jobs(n):
        rows = pending_rows(rng, regime, n, U, jid[0], codes)
        jid[0] += 2 * n + 2
        return keyed(rows)

    try:
        check(h, U, listed)                                        # an empty handle: zeros
        h.apply(run_up=fresh_rows(700), up=fresh_jobs(600))
        check(h, U, listed)
        for b in range(6):
            fin = [t for t in h.run if rng.random() < 0.05]
            h.apply(run_up=fresh_rows(250), up=fresh_jobs(150), run_rm=fin, hosts=b % 2 == 0)   # past 1024, then 2048
            check(h, U, listed)
            launch = list(rng.choice(sorted(h.pend), 120, replace=False))
            tids = [tid[0] + 2 * i for i in range(len(launch))]
            tid[0] += 2 * len(launch) + 2
            hn = np.array(rng.choice(hosts, len(launch)), np.int32) if b % 2 else None
            h.launch(launch, tids, np.full(len(launch), START, np.int64), hn)                           # lists leave with the rows: arena compaction
            check(h, U, listed)
        h.apply(reset=True, run_up=fresh_rows(900), up=fresh_jobs(50))
        got = check(h, U, listed)
        if regime == "mixed":   # both paths in one call: user 0 passes 2^43, the others stay exact
            assert got["user"]["mem"][0] > 2.0 ** 43 and got["user"]["mem"][1:].max() < 2.0 ** 30
            mine = [r["mem"] for r in sorted(h.run.values(), key=lambda r: r["task_id"]) if r["user"] == 0]
            assert F.association_sensitive(mine)
        h.apply(run_rm=list(h.run)[:300])
        check(h, U, listed)
        h.apply(run_rm=list(h.run))
        check(h, U, listed)                                        # no live row: zeros again
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["off", "mixed"])
def test_layout_independence(regime):
    """The same rows reached by two histories: one batch in task id order, or after junk rows whose freed slots
    the real rows reuse in a permuted order.  Every output is identical to the bit."""
    rng = np.random.default_rng(21)
    U, hosts = 30, list(range(40)) + [-1]
    rows = random_rows(rng, regime, 1500, U, 10, hosts)
    listed = np.array(rng.permutation(40), np.int32)
    a, b = new_handle("a"), new_handle("b")
    try:
        a.apply(run_up=sorted(rows, key=lambda r: r["task_id"]))
        junk = random_rows(rng, regime, 800, U, 10_000_000, hosts)
        b.apply(run_up=junk)
        perm = [rows[i] for i in rng.permutation(len(rows))]
        b.apply(run_up=perm[:600], run_rm=[r["task_id"] for r in junk[:500]])
        b.apply(run_up=perm[600:], run_rm=[r["task_id"] for r in junk[500:]])
        ga, gb = check(a, U, listed), check(b, U, listed)
        for k in KEYS:
            assert F.same_bits(ga["user"][k], gb["user"][k])
        for k in ("pool", "run_cpus", "run_mem"):
            assert F.same_bits(ga[k], gb[k])
        assert np.array_equal(ga["run_count"], gb["run_count"])
        # the permuted insertion order folds to other bits somewhere: a slot-order fold would fail above
        alt = running_usage([dict(r, task_id=i) for i, r in enumerate(perm)], U, listed)
        assert any(not F.same_bits(alt["user"][k], ga["user"][k]) for k in ("cpus", "mem")) or \
            not F.same_bits(alt["run_mem"], ga["run_mem"])
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_host_edges():
    rng = np.random.default_rng(31)
    U = 5
    h = new_handle()
    try:
        assert np.all(check(h, U, np.array([3, 9], np.int32))["run_count"] == 0)
        # host 3: 3000 rows (past two sort tiles); host 4: 65; rows with -1 and with codes 8, 1000 not listed
        hosts = [3] * 3000 + [4] * 65 + [-1] * 40 + [8] * 30 + [1000] * 10 + [5]
        rows = random_rows(rng, "off", len(hosts), U, 100, [0])
        for r, c in zip(rows, hosts):
            r["host"] = c
        h.apply(run_up=rows)
        got = check(h, U, np.array([4, 3, 77, 5, 2], np.int32))   # 77 and 2: listed, no rows
        assert got["run_count"].tolist() == [65, 3000, 0, 1, 0]
        assert got["run_cpus"][2] == 0.0 and got["run_mem"][4] == 0.0
        assert got["pool"][0] == float(len(rows))
        check(h, U, np.zeros(0, np.int32))                         # no host list
        check(h, U, np.array([1000], np.int32))
    finally:
        h.close()


@pytest.mark.gpu
def test_errors_leave_the_handle_unchanged():
    rng = np.random.default_rng(41)
    h = new_handle()
    try:
        h.apply(run_up=random_rows(rng, "off", 300, 6, 100, list(range(10))))
        listed = np.arange(10, dtype=np.int32)
        before = check(h, 6, listed)
        lib, pool = h.gpu.lib, h.gpu.pool
        out = np.zeros(64)
        codes = np.array([1, 2, 1], np.int32)
        neg = np.array([1, -2], np.int32)
        P = abi.P_F64
        cases = [
            (5, abi.ptr(out, P), None, 0, None),                 # n_users <= the largest user code
            (6, abi.ptr(out, P), None, -1, None),                # n_hosts < 0
            (6, None, None, 3, None),                            # NULL hostname_id
            (6, None, abi.ptr(out, P), 3, abi.ptr(codes, abi.P_I32)),   # a code twice
            (6, None, None, 2, abi.ptr(neg, abi.P_I32)),         # a negative code
        ]
        for nu, uo, po, nh, hn in cases:
            rc = lib.cook_state_usage(pool, nu, uo, po, nh, hn, abi.ptr(out, P), None, None)
            assert rc == abi.COOK_E_BADARG
        assert lib.cook_state_usage(pool, 0, None, abi.ptr(out, P), 0, None, None, None, None) == abi.COOK_OK
        assert F.same_bits(out[:4], before["pool"])               # n_users is not read without out_user_usage
        after = check(h, 6, listed)
        for k in KEYS:
            assert F.same_bits(after["user"][k], before["user"][k])
        assert F.same_bits(after["run_mem"], before["run_mem"])
    finally:
        h.close()


@pytest.mark.gpu
def test_resident_match_fed_from_state_usage(oracle):
    """Several cycles: the resident pool is ranked and matched with users' usage and offers' run columns from
    cook_state_usage, and equals cook_match on host tables whose columns are Python folds in ascending task id,
    and the oracle's considerable set.  Quotas bind at the derived usage, and launches move it between cycles:
    a match with the first cycle's usage would choose another considerable set in some cycle."""
    rng = np.random.default_rng(51)
    U, O, J = 10, 40, 500
    codes = (100 + np.arange(O)).astype(np.int32)
    h, ref = new_handle("resident"), engine.GpuEngine(pool_name="host")
    pend = pending_rows(rng, "grid", J, U, 1_000_000, codes.tolist())
    for p in pend:
        p["gpus"] = 0.0
        p["novel"] = []
    run = random_rows(rng, "grid", 300, U, 10, codes.tolist() + [-1])
    for r in run:
        r["gpus"] = 0.0
    h.apply(up=keyed(pend), run_up=run)
    cnt0 = np.bincount([r["user"] for r in run], minlength=U).astype(float)
    quota = {"count": cnt0 + 30.0, "cpus": np.full(U, 1e9), "mem": np.full(U, 1e12), "gpus": np.full(U, 1e9)}
    lease_c, lease_m = np.full(O, 12.0), np.full(O, 32768.0)
    rank = rng.permutation(O).astype(np.int32)
    params = abi.MatchParams(num_considerable=1000, enforce_rate_limit=0, host_lifetime_mins=0, fitness_kind=0,
                             good_enough_fitness=1.0, reuse_resident=0, max_ctas=0)
    div = dict(div_cpus=np.full(U, 40.0), div_mem=np.full(U, 81920.0), div_gpus=np.ones(U))

    def tables(usage):
        users = abi.make_users(U, quota=quota, usage=usage["user"], **div)
        offers = abi.OffersSoA(n=O, hostname_id=codes, name_rank=rank, cpus=lease_c, mem=lease_m,
                               run_cpus=usage["run_cpus"], run_mem=usage["run_mem"], run_count=usage["run_count"],
                               n_attr_cols=0)
        return users, offers

    first, differs = None, False
    next_tid = 10_000_000
    try:
        for cycle in range(4):
            got = h.gpu.state_usage(U, codes)
            want = running_usage(h.run.values(), U, codes)
            users, offers = tables(got)
            users_h, offers_h = tables(want)
            q = h.gpu.state_rank(users)
            m = h.gpu.state_match(offers, users, params)
            # host arm: the same rows as host tables, sorted by id
            jids = np.array(sorted(h.pend), np.int64)
            pr = [h.pend[j] for j in jids]
            jobs = abi.JobsSoA(n=len(pr), user=np.array([p["user"] for p in pr], np.int32),
                               cpus=np.array([p["cpus"] for p in pr]), mem=np.array([p["mem"] for p in pr]),
                               gpus=np.zeros(len(pr)))
            pt = abi.make_tasks(user=jobs.col("user"), priority=np.full(len(pr), 50, np.int32),
                                start_time=np.full(len(pr), abi.INT64_MAX), task_id=np.full(len(pr), -1, np.int64),
                                job_id=jids, cpus=jobs.col("cpus"), mem=jobs.col("mem"))
            rr = sorted(h.run.values(), key=lambda r: r["task_id"])
            rt = tasks_soa(rr)
            hr = ref.rank(rt, pt, users_h)
            assert np.array_equal(q, jids[hr["ranked"]])
            hm = ref.match(hr["ranked"], jobs, offers_h, users_h, params)
            assert np.array_equal(m["considerable"], jids[hm["considerable"]])
            assert np.array_equal(m["assign"], hm["assign"])
            om = oracle.match(hr["ranked"], jobs, offers_h, users_h, params)
            assert np.array_equal(om["considerable"], hm["considerable"])
            # the quotas bind: fewer considerable jobs than queued ones
            assert 0 < len(m["considerable"]) < min(len(q), params.num_considerable)
            if first is None:
                first = got
            else:
                stale_users, stale_offers = tables(first)
                st = oracle.match(hr["ranked"], jobs, stale_offers, stale_users, params)
                differs |= not np.array_equal(st["considerable"], hm["considerable"])
            placed = m["assign"] >= 0
            jl = m["considerable"][placed]
            assert len(jl) > 0
            tids = next_tid + 2 * np.arange(len(jl), dtype=np.int64)
            next_tid += 2 * len(jl) + 2
            h.launch(jl.tolist(), tids.tolist(), np.full(len(jl), START, np.int64), codes[m["assign"][placed]])
        assert differs
    finally:
        h.close()
        ref.close()
