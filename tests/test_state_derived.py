"""cook_state_match_derived / cook_state_rebalance_derived: a resident match or rebalance whose running-side
inputs (the users' usage, the offers' run columns, the groups' cotask lists) are derived on the device from the
live running rows, without the round trip through cook_state_usage and cook_state_cotasks.

CPU: the exports, the prototypes (each derived call takes exactly its plain call's arguments, checked by the C
compiler) and the ctypes signatures against the header.
GPU (-m gpu): after every batch of a churn, the derived match against the three-call sequence on the same handle
(bit equality of considerable, assign, ports and fail; failure counts and the usage exchange; the upload and
download formula) and against the oracle on host tables built from a model; config-#3 cycles with groups and K13's
group cases; a config-#4 rebalance; freshness after launches; slot-layout independence; errors and edges.
"""
import ctypes as C

import numpy as np
import pytest

import fold_ref as F
from cook_b200 import abi, traces
from cook_b200.engine import CookError, GpuEngine
from cotask_ref import cotasks
from resident_model import (COT_FIELDS, K13, RUN_FIELDS, START, USAGE_FIELDS, Pool, decisions_eq, drop_all_but, fed_tables,
                            host_inputs, jobs_soa, keyed, pending_rows, pool_rows, random_rows, rebalance_trace, rows_of,
                            tasks_soa, with_fields)
from usage_ref import KEYS, running_usage



# ---- GPU helpers -------------------------------------------------------------------------------------------
def derived_inputs(offers, users, groups):
    """The tables of a derived call: the fields it derives are NULL."""
    users = with_fields(users, **{f: None for f in USAGE_FIELDS})
    offers = with_fields(offers, **{f: None for f in RUN_FIELDS})
    groups = with_fields(groups, **{f: None for f in COT_FIELDS}) if groups is not None else None
    return offers, users, groups


def sequenced_inputs(e, offers, users, groups):
    """cook_state_usage and cook_state_cotasks downloaded, then the tables a cook_state_match takes."""
    usage = e.state_usage(users.n_users, offers.col("hostname_id") if offers.n else None)
    cot = None
    if groups is not None and groups.n_groups:
        cot = e.state_cotasks(groups.n_groups, groups.col("attr_col"), offers)
    return fed_tables(offers, users, groups, usage, cot), usage, cot


def saved_up(G, O, U, n_cot, grouped):
    return 32 * U + 20 * O + ((4 * (G + 1) + 8 * max(1, n_cot)) if grouped else 0)


def compare(e, offers, users, prm, groups=None, max_ports=0, grouped=False):
    """The derived match against the three-call sequence on handle e (both only read the state).  Returns the
    derived result and the sequenced tables."""
    (so, su, sg), usage, cot = sequenced_inputs(e, offers, users, groups)
    ps_u, ps_c = e.last_stats(abi.PHASE_USAGE), e.last_stats(abi.PHASE_COTASKS)
    want = e.state_match(so, su, prm, groups=sg, max_ports=max_ports)
    n = len(want["considerable"])
    k = np.arange(n, dtype=np.int32)
    fw = e.match_failures(k) if n else []
    xw = e.exchange_usage(users.n_users)
    do, du, dg = derived_inputs(offers, users, groups)
    got = e.state_match(do, du, prm, groups=dg, max_ports=max_ports, derived=True)
    for key in ("considerable", "assign", "ports", "fail"):
        assert np.array_equal(got[key], want[key]), key
    if n:
        assert e.match_failures(k) == fw
    assert np.array_equal(e.exchange_usage(users.n_users), xw)
    # the phases of the standalone calls are untouched by the derived one
    assert e.last_stats(abi.PHASE_USAGE) == ps_u and e.last_stats(abi.PHASE_COTASKS) == ps_c
    sw, sd = want["stats"], got["stats"]
    if n:
        G = groups.n_groups if groups is not None else 0
        n_cot = len(cot[1]) if cot is not None else 0
        assert sd["h2d_bytes"] == sw["h2d_bytes"] - saved_up(G, offers.n, users.n_users, n_cot, grouped and G > 0)
        assert sd["d2h_bytes"] == sw["d2h_bytes"]
    return got, (so, su, sg)


def oracle_check(oracle, got, run_rows, jobs, jid, ranked_, offers, users, prm, groups=None, max_ports=0):
    ho, hu, hg = host_inputs(run_rows, offers, users, groups)
    om = oracle.match(ranked_, jobs, ho, hu, prm, groups=hg, max_ports=max_ports)
    assert np.array_equal(got["considerable"], jid[om["considerable"]])
    assert np.array_equal(got["assign"], om["assign"])


def new_pool(name):
    """A resident handle whose running upserts carry hosts and group lists, and the model of its rows."""
    return Pool(name, send_hosts=True, send_lists=True)


def grouped(p):
    return any(r["groups"] for r in p.pend.values())


def live_positions(p, q):
    return p.ranked([j for j in q.tolist() if j in p.pend])


def _hosts_for(rng, run, codes, unlisted=(), none=0.05):
    for r in run.values():
        x = rng.random()
        r["host"] = -1 if x < none else int(rng.choice(unlisted)) if unlisted and x < 2 * none else int(rng.choice(codes))


# ---- GPU: a C2 pool under churn, on and off the grid ----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["grid", "off"])
def test_c2_churn(regime, oracle):
    cpus = (0.5, 1, 2, 4, 8) if regime == "grid" else (0.1, 0.5, 1.0, 2.0)
    t = traces.gen_pool(41 if regime == "grid" else 43, 3000, 200, 30, 600, cpus_choices=cpus)
    rng = np.random.default_rng(7)
    offers, users = t["offers"], t["users"]
    codes = offers.col("hostname_id")
    U = users.n_users
    pend, run = pool_rows(t)
    if regime == "off":                                  # the serial folds: tenths and thirds
        for r in run.values():
            r["cpus"] = r["cpus"] + 0.1
            r["mem"] = r["mem"] / 3.0
    _hosts_for(rng, run, codes, unlisted=(5000, 5001, 5002))
    idle = {int(u) for u in rng.choice(U, 4, replace=False)}   # users without running rows, now or later
    run = {k: r for k, r in run.items() if r["user"] not in idle}
    items = sorted((j, r) for j, r in pend.items() if r["user"] not in idle)
    cut = int(len(items) * 0.6)
    reserve = items[cut:]
    prm = traces.match_params(1000)
    p = new_pool("c2")
    tid = [10 ** 9]

    def tids(n):
        out = [tid[0] + 3 * i for i in range(n)]
        tid[0] += 3 * n + 3
        return out

    try:
        p.apply(up=items[:cut], run_up=list(run.values()), reset=True)
        for cycle in range(7):
            q = p.gpu.state_rank(users)
            got, _ = compare(p.gpu, offers, users, prm)
            jobs, jid, ranked_ = live_positions(p, q)
            if cycle % 2 == 0:
                oracle_check(oracle, got, p.run.values(), jobs, jid, ranked_, offers, users, prm)
            cnt = running_usage(p.run.values(), U)["user"]["count"]
            assert (cnt == 0).any()
            placed = got["assign"] >= 0
            jl = got["considerable"][placed].tolist()[:60]
            assert jl
            hn = codes[got["assign"][placed][:len(jl)]].astype(np.int32) if cycle % 3 != 1 else None
            p.launch(jl, tids(len(jl)), np.full(len(jl), START, np.int64), hn)                    # launches with and without hosts
            fin = [x for x in p.run if rng.random() < 0.04]
            new = [reserve.pop() for _ in range(min(len(reserve), 80))]
            p.apply(up=new, run_rm=fin)                          # finishes and submissions
            live = sorted(p.pend)
            flip = [int(j) for j in rng.choice(live, 30, replace=False)]
            p.patch(flip, allowed=np.zeros(30, np.uint8))        # patches keep the queue
            if cycle == 2:                                       # growth: past the running table's capacity
                more = [dict(r, task_id=r["task_id"] + 5 * 10 ** 8, job_id=r["job_id"] + 5 * 10 ** 8)
                        for r in list(p.run.values())[:700]]
                p.apply(run_up=more)
            if cycle == 4:                                       # a reset with the same rows, then compaction
                p.apply(up=sorted(p.pend.items()), run_up=list(p.run.values()), reset=True)
                p.apply(run_rm=[x for x in p.run if rng.random() < 0.7])
        q = p.gpu.state_rank(users)
        got, _ = compare(p.gpu, offers, users, prm)
        jobs, jid, ranked_ = live_positions(p, q)
        oracle_check(oracle, got, p.run.values(), jobs, jid, ranked_, offers, users, prm)
    finally:
        p.close()


# ---- GPU: config-#3 cycles with groups, K13 --------------------------------------------------------------------
@pytest.mark.gpu
def test_c3_cycles_with_groups(oracle):
    t = traces.gen_c3_pool(17, n_jobs=2500, n_offers=160, n_users=24, n_running=500)
    rng = np.random.default_rng(19)
    g0, offers, users = t["groups"], t["offers"], t["users"]
    G = g0.n_groups
    hn = offers.col("hostname_id")
    pend, run = pool_rows(t)
    _hosts_for(rng, run, hn, unlisted=(9000, 9001))
    for r in run.values():
        r["groups"] = [int(rng.integers(G))] if rng.random() < 0.2 else []
    items = sorted(pend.items())
    cut = int(len(items) * 0.7)
    reserve = items[cut:]
    prm = traces.match_params(1000, host_lifetime_mins=t.get("host_lifetime_mins", 0))
    max_ports = int(t["jobs"].col("ports").max())
    p = new_pool("c3")
    tid = 10 ** 9
    try:
        p.apply(up=items[:cut], run_up=list(run.values()), reset=True)
        n_cot = 0
        for cycle in range(5):
            q = p.gpu.state_rank(users)
            got, (so, su, sg) = compare(p.gpu, offers, users, prm, groups=g0, max_ports=max_ports, grouped=grouped(p))
            n_cot = max(n_cot, int(sg.col("cot_off")[-1]))
            jobs, jid, ranked_ = live_positions(p, q)
            oracle_check(oracle, got, p.run.values(), jobs, jid, ranked_, offers, users, prm, g0, max_ports)
            placed = got["assign"] >= 0
            jl = got["considerable"][placed].tolist()
            assert jl
            p.launch(jl, [tid + 3 * i for i in range(len(jl))], np.full(len(jl), START, np.int64),
                     hn[got["assign"][placed]].astype(np.int32))
            tid += 3 * len(jl) + 3
            fin = [x for x in p.run if rng.random() < 0.03]
            new = [reserve.pop() for _ in range(min(len(reserve), len(fin) + 20))]
            for _, r in new[:10]:
                r["groups"] = sorted({*r["groups"], int(rng.integers(G))})
            p.apply(up=new, run_rm=fin)
        assert n_cot > 50
    finally:
        p.close()


def derived_cycle(k, spec):
    """K13's group cases through the derived call: the cycle's derived match equals the sequenced one and the oracle
    on host-built lists (failure counts included), then its placements are launched."""
    offers = k.offers(spec)
    q = k.e.gpu.state_rank(k.users)
    G = len(k.kind)
    groups = abi.Groups(n_groups=G, kind=k.kind, attr_col=k.col, minimum=k.minimum)
    prm = traces.match_params(len(q))
    m, _ = compare(k.e.gpu, offers, k.users, prm, groups=groups, grouped=True)
    ids, jobs = k.jobs()
    pos = {j: i for i, j in enumerate(ids)}
    ranked = np.array([pos[j] for j in q], np.int32)
    hc = cotasks(k.e.run.values(), G, k.col, offers.col("hostname_id"), offers.col("attr").reshape(1, offers.n))
    hg = fed_tables(offers, k.users, groups, running_usage([], 1), hc)[2]
    om = k.o.match(ranked, jobs, offers, k.users, prm, groups=hg)
    assert np.array_equal(m["considerable"], np.array(ids)[om["considerable"]])
    assert np.array_equal(m["assign"], om["assign"])
    kk = np.arange(len(m["considerable"]), dtype=np.int32)
    fg, fo = k.e.gpu.match_failures(kk), k.o.match_failures(ranked, jobs, offers, k.users, prm, kk, groups=hg)
    grp = slice(abi.FAILC_N - 3, abi.FAILC_N)
    assert [(f["n_vms"], f["counts"][grp]) for f in fg] == [(f["n_vms"], f["counts"][grp]) for f in fo]
    k.launch_placed(m, offers)
    return [spec[a]["host"] if a >= 0 else None for a in m["assign"]]


@pytest.mark.gpu
def test_k13_groups_through_the_derived_call(oracle):
    p = K13(oracle, [dict(kind=abi.GROUP_UNIQUE)])
    try:
        host = [dict(host="test-host", cpus=100.0)]
        p.submit(1)
        assert derived_cycle(p, host) == ["test-host"]
        p.submit(2)                                   # its cotask runs on the only host
        assert derived_cycle(p, host) == [None, None]
    finally:
        p.close()
    p = K13(oracle, [dict(kind=abi.GROUP_BALANCED, col=0, minimum=3)])
    try:
        hosts = [dict(host=h, cpus=100.0, attrs={0: i + 1}) for i, h in enumerate(["straw", "sticks", "bricks"])]
        p.submit(3)
        first = derived_cycle(p, hosts)
        p.submit(6)
        second = derived_cycle(p, hosts)
        assert None not in first + second
        assert sorted(np.unique(first + second, return_counts=True)[1].tolist()) == [3, 3, 3]
    finally:
        p.close()
    p = K13(oracle, [dict(kind=abi.GROUP_ATTR_EQUALS, col=0)])
    try:
        east = dict(host="first-east-host", cpus=1.0, attrs={0: 1})
        p.submit(1)
        assert derived_cycle(p, [east]) == ["first-east-host"]
        offers = [dict(east, cpus=0.5)] + [dict(host=f"west-{i:02d}", cpus=1.0, attrs={0: 2}) for i in range(20)]
        offers.append(dict(host="east-big", cpus=5.0, attrs={0: 1}))
        p.submit(20)
        got = derived_cycle(p, offers)
        assert got.count("east-big") == 5 and got.count(None) == 15
    finally:
        p.close()


# ---- GPU: config-#4 rebalance -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_c4_rebalance_derived(oracle):
    r, codes = rebalance_trace(23, True)
    rng = np.random.default_rng(29)
    G, g0, hosts = r["groups"].n_groups, r["groups"], r["hosts"]
    pend, run = rows_of(r, codes)
    for row in run.values():
        row["groups"] = [int(rng.integers(G))] if rng.random() < 0.2 else []
    p = Pool.of_rebalance(r, codes)
    try:
        run_up = list(run.values())
        pj, pp, jid = jobs_soa(sorted(pend.items()))
        off, idx = abi.csr([x["groups"] for x in run_up])
        p.gpu.state_apply(abi.make_delta(reset=True, pending=pj, pending_priority=pp, pending_job_id=jid,
                                         running=tasks_soa(run_up), running_hostname_id=np.array([x["host"] for x in run_up], np.int32),
                                         running_group_off=off, running_group_idx=idx))
        p.pend, p.run = dict(pend), dict(run)
        acol = g0.col("attr_col")
        for step in range(3):
            p.rank()
            cot = p.gpu.state_cotasks(G, acol, hosts)
            assert len(cot[1]) > 300
            p.groups = with_fields(g0, cot_off=cot[0], cot_hostname_id=cot[1], cot_attr_val=cot[2])
            want = p.gpu.state_rebalance(hosts, p.users, p.rparams, groups=p.groups)
            sw = p.gpu.last_stats(abi.PHASE_REBALANCE)
            got = p.gpu.state_rebalance(hosts, p.users, p.rparams, groups=with_fields(g0, **{f: None for f in COT_FIELDS}),
                                        derived=True)
            sd = p.gpu.last_stats(abi.PHASE_REBALANCE)
            decisions_eq(got, want)
            assert got
            decisions_eq(got, p.want_rebalance(oracle))
            assert sd["h2d_bytes"] == sw["h2d_bytes"] - (4 * (G + 1) + 8 * len(cot[1]))
            assert sd["d2h_bytes"] == sw["d2h_bytes"]
            fin = [t for t in p.run if rng.random() < 0.1]       # finishes move the lists between steps
            p.apply(run_rm=fin)
    finally:
        p.close()


# ---- GPU: freshness, layout, accounting ----------------------------------------------------------------------
@pytest.mark.gpu
def test_freshness_after_launches(oracle):
    """After each cycle's launches the derived match sees the launched tasks: it equals a sequenced match fed with
    freshly derived inputs, while a match fed with the previous cycle's arrays differs on the same inputs."""
    rng = np.random.default_rng(51)
    U, O, J = 10, 40, 500
    codes = (100 + np.arange(O)).astype(np.int32)
    h = Pool("fresh", drop=drop_all_but("gpus", "novel"), send_hosts=True)
    pend = pending_rows(rng, "grid", J, U, 1_000_000, codes.tolist())
    for x in pend:
        x["gpus"], x["novel"] = 0.0, []
    run = random_rows(rng, "grid", 300, U, 10, codes.tolist() + [-1])
    for x in run:
        x["gpus"] = 0.0
    h.apply(up=keyed(pend), run_up=run)
    cnt0 = np.bincount([x["user"] for x in run], minlength=U).astype(float)
    quota = {"count": cnt0 + 30.0, "cpus": np.full(U, 1e9), "mem": np.full(U, 1e12), "gpus": np.full(U, 1e9)}
    users = abi.make_users(U, quota=quota, div_cpus=np.full(U, 40.0), div_mem=np.full(U, 81920.0), div_gpus=np.ones(U))
    offers = abi.OffersSoA(n=O, hostname_id=codes, name_rank=rng.permutation(O).astype(np.int32), cpus=np.full(O, 12.0),
                           mem=np.full(O, 32768.0), n_attr_cols=0)
    prm = traces.match_params(1000)
    stale, differs = None, False
    tid = 10_000_000
    try:
        for cycle in range(4):
            h.gpu.state_rank(users)
            got, (so, su, _) = compare(h.gpu, offers, users, prm)
            want = running_usage(h.run.values(), U, codes)
            for f, k in zip(USAGE_FIELDS, KEYS):
                assert F.same_bits(su.col(f), want["user"][k])
            assert 0 < len(got["considerable"]) < len(h.pend)
            if stale is not None:
                old = h.gpu.state_match(stale[0], stale[1], prm)
                differs |= not np.array_equal(old["considerable"], got["considerable"])
            stale = (so, su)
            placed = got["assign"] >= 0
            jl = got["considerable"][placed]
            tids = tid + 2 * np.arange(len(jl), dtype=np.int64)
            tid += 2 * len(jl) + 2
            h.launch(jl.tolist(), tids.tolist(), np.full(len(jl), START, np.int64), codes[got["assign"][placed]])
        assert differs
    finally:
        h.close()


@pytest.mark.gpu
def test_layout_independence():
    t = traces.gen_c3_pool(31, n_jobs=1500, n_offers=120, n_users=20, n_running=600)
    rng = np.random.default_rng(33)
    g0, offers, users = t["groups"], t["offers"], t["users"]
    pend, run = pool_rows(t)
    _hosts_for(rng, run, offers.col("hostname_id"))
    for r in run.values():
        r["groups"] = [int(rng.integers(g0.n_groups))] if rng.random() < 0.3 else []
        r["cpus"] = r["cpus"] + 0.1                          # off the grid
    items, rr = sorted(pend.items()), list(run.values())
    prm = traces.match_params(1000)
    max_ports = int(t["jobs"].col("ports").max())
    a, b = new_pool("a"), new_pool("b")
    try:
        a.apply(up=items, run_up=sorted(rr, key=lambda r: r["task_id"]))
        junk = [dict(r, task_id=r["task_id"] + 10 ** 10, job_id=r["job_id"] + 10 ** 10) for r in rr[:400]]
        b.apply(run_up=junk)
        b.apply(run_rm=[r["task_id"] for r in junk])
        perm = [rr[i] for i in rng.permutation(len(rr))]
        b.apply(up=items[::-1], run_up=perm[:300])
        b.apply(run_up=perm[300:])
        out = []
        for p in (a, b):
            p.gpu.state_rank(users)
            do, du, dg = derived_inputs(offers, users, g0)
            out.append(p.gpu.state_match(do, du, prm, groups=dg, max_ports=max_ports, derived=True))
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(out[0][k], out[1][k]), k
        assert (out[0]["assign"] >= 0).sum() > 0
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1, 6])
def test_transfer_accounting(scale):
    """h2d = the sequenced match's minus exactly 32 U + 20 O + 4 (G + 1) + 8 max(1, N); d2h equal (compare())."""
    t = traces.gen_c3_pool(61 + scale, n_jobs=500 * scale, n_offers=40 * scale, n_users=8 * scale, n_running=200 * scale)
    rng = np.random.default_rng(scale)
    g0, offers, users = t["groups"], t["offers"], t["users"]
    pend, run = pool_rows(t)
    _hosts_for(rng, run, offers.col("hostname_id"))
    for r in run.values():
        r["groups"] = [int(rng.integers(g0.n_groups))] if rng.random() < 0.3 else []
    p = new_pool("acct")
    try:
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.gpu.state_rank(users)
        got, (_, _, sg) = compare(p.gpu, offers, users, traces.match_params(1000), groups=g0,
                                  max_ports=int(t["jobs"].col("ports").max()), grouped=grouped(p))
        assert grouped(p) and int(sg.col("cot_off")[-1]) > 0 and len(got["considerable"]) > 0
        assert got["stats"]["ms_h2d"] > 0.0 and got["stats"]["n_launches"] > 0
    finally:
        p.close()


# ---- GPU: errors and edges -------------------------------------------------------------------------------------
def _small(rng, n_run=120, G=4):
    t = traces.gen_c3_pool(71, n_jobs=300, n_offers=30, n_users=6, n_running=n_run)
    pend, run = pool_rows(t)
    _hosts_for(rng, run, t["offers"].col("hostname_id"))
    for r in run.values():
        r["groups"] = [int(rng.integers(G))] if rng.random() < 0.5 else []
    groups = abi.Groups(n_groups=G, kind=np.array([0, 1, 2, 0][:G], np.int32), attr_col=np.array([-1, 0, 1, -1][:G], np.int32),
                        minimum=np.zeros(G, np.int32))
    return t, pend, run, groups


@pytest.mark.gpu
def test_errors_write_nothing():
    rng = np.random.default_rng(81)
    t, pend, run, groups = _small(rng)
    offers, users = t["offers"], t["users"]
    prm = traces.match_params(1000)
    p = new_pool("errors")
    try:
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.gpu.state_rank(users)
        before, _ = compare(p.gpu, offers, users, prm, groups=groups, grouped=grouped(p))
        lib, pool = p.gpu.lib, p.gpu.pool
        do, du, dg = derived_inputs(offers, users, groups)
        O = offers.n
        hn = offers.col("hostname_id")
        dup = with_fields(do, hostname_id=np.concatenate([hn[:-1], hn[:1]]).astype(np.int32))
        neg = with_fields(do, hostname_id=np.concatenate([hn[:-1], [-3]]).astype(np.int32))
        no_hn = with_fields(do, hostname_id=None)
        no_attr = with_fields(do, attr=None)
        few_users = with_fields(du, n_users=int(max(r["user"] for r in run.values())))
        few_groups = with_fields(dg, n_groups=1, kind=dg.col("kind")[:1], attr_col=dg.col("attr_col")[:1],
                                 minimum=dg.col("minimum")[:1])
        col_hi = with_fields(dg, attr_col=np.array([-1, offers.n_attr_cols, 1, -1], np.int32))
        col_lo = with_fields(dg, attr_col=np.array([-2, 0, 1, -1], np.int32))
        no_kind = with_fields(dg, kind=None)
        bad_prm = traces.match_params(1000)
        bad_prm.reuse_resident = 1
        k = max(prm.num_considerable, 1)
        cons, assign = np.full(k, -7, np.int64), np.full(k, -7, np.int32)
        ports, fail = np.full(k, -7, np.int32), np.full(k, 7, np.uint8)

        def call(o=do, u=du, g=dg, pr=prm):
            return lib.cook_state_match_derived(pool, C.byref(o), C.byref(g) if g is not None else None, C.byref(u),
                                                C.byref(abi.make_pool_quota(None)), C.byref(pr),
                                                abi.ptr(cons, abi.P_I64), abi.ptr(assign, abi.P_I32),
                                                abi.ptr(ports, abi.P_I32), 1, abi.ptr(fail, abi.P_U8), None)
        cases = [call(o=dup), call(o=neg), call(o=no_hn), call(o=no_attr), call(u=few_users), call(g=few_groups),
                 call(g=col_hi), call(g=col_lo), call(g=no_kind), call(pr=bad_prm)]
        assert cases == [abi.COOK_E_BADARG] * len(cases)
        assert (cons == -7).all() and (assign == -7).all() and (ports == -7).all() and (fail == 7).all()
        assert lib.cook_state_match_derived(pool, None, None, None, None, None, None, None, None, 0, None, None) == \
            abi.COOK_E_BADARG
        after, _ = compare(p.gpu, offers, users, prm, groups=groups, grouped=grouped(p))   # unaffected
        for key in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(after[key], before[key])
        # the rebalance's own cases; GPU DRU mode is unsupported
        hosts = abi.HostTable(n=O, hostname_id=hn, name_rank=offers.col("name_rank"), n_attr_cols=offers.n_attr_cols,
                              attr=offers.col("attr"))
        rp = abi.RebalanceParams(max_preemption=8, min_dru_diff=0.5, safe_dru_threshold=1.0, host_lifetime_mins=0)
        dec, jid = (abi.Decision * 8)(), np.zeros(8, np.int64)
        vict, n = np.zeros(len(run) + 8, np.int64), C.c_int32(-7)

        def rcall(h=hosts, g=dg):
            return lib.cook_state_rebalance_derived(pool, C.byref(h), C.byref(g), C.byref(du), C.byref(rp), dec,
                                                    abi.ptr(jid, abi.P_I64), abi.ptr(vict, abi.P_I64), len(vict), C.byref(n))
        rcases = [rcall(g=few_groups), rcall(g=col_hi), rcall(g=col_lo), rcall(h=with_fields(hosts, attr=None))]
        assert rcases == [abi.COOK_E_BADARG] * len(rcases)
        assert n.value in (-7, 0) and (jid == 0).all()
        dru = GpuEngine(pool_name="dru", dru_mode=1)
        try:
            with pytest.raises(CookError) as ex:
                dru.state_rebalance(hosts, users, rp, groups=groups, derived=True)
            assert ex.value.code == abi.COOK_E_UNSUPPORTED_CONSTRAINT
        finally:
            dru.close()
    finally:
        p.close()


@pytest.mark.gpu
def test_edges(oracle):
    rng = np.random.default_rng(91)
    t, pend, run, groups = _small(rng)
    offers, users = t["offers"], t["users"]
    prm = traces.match_params(1000)
    p = new_pool("edges")
    try:
        items = sorted(pend.items())
        p.apply(up=items)                                  # no live running row
        p.gpu.state_rank(users)
        got, (so, su, sg) = compare(p.gpu, offers, users, prm, groups=groups, grouped=grouped(p))
        assert all((su.col(f) == 0).all() for f in USAGE_FIELDS) and (sg.col("cot_off") == 0).all()
        n0 = p.gpu.last_stats(abi.PHASE_MATCH)["n_launches"]
        zo, zu, zg = fed_tables(offers, users, groups, running_usage([], users.n_users, offers.col("hostname_id")),
                                ([0] * (groups.n_groups + 1), [], []))
        plain = p.gpu.state_match(zo, zu, prm, groups=zg)
        assert p.gpu.last_stats(abi.PHASE_MATCH)["n_launches"] == n0   # no derivation kernel: the same launches
        assert np.array_equal(plain["assign"], got["assign"])
        # no groups; groups without a running row that has both a host and a group
        rows = list(run.values())
        p.apply(run_up=[dict(r, groups=[]) for r in rows[:40]] + [dict(r, host=-1) for r in rows[40:80]])
        p.gpu.state_rank(users)
        compare(p.gpu, offers, users, prm, grouped=grouped(p))
        _, (_, _, sg) = compare(p.gpu, offers, users, prm, groups=groups, grouped=grouped(p))
        assert (sg.col("cot_off") == 0).all()
        # running rows on hosts without an offer this cycle, and with host -1
        p.apply(run_up=[dict(r, host=7777) for r in rows[80:]])
        p.gpu.state_rank(users)
        got, _ = compare(p.gpu, offers, users, prm, groups=groups, grouped=grouped(p))
        jobs, jid, ranked_ = live_positions(p, p.gpu.state_rank(users))
        oracle_check(oracle, got, p.run.values(), jobs, jid, ranked_, offers, users, prm, groups)
        # offers->n == 0: as cook_state_match
        empty = abi.OffersSoA(n=0, hostname_id=np.zeros(1, np.int32), name_rank=np.zeros(1, np.int32),
                              cpus=np.zeros(1), mem=np.zeros(1), run_cpus=np.zeros(1), run_mem=np.zeros(1),
                              run_count=np.zeros(1, np.int32), n_attr_cols=offers.n_attr_cols, attr=np.zeros(4, np.int32))
        got, _ = compare(p.gpu, empty, users, prm, groups=groups, grouped=grouped(p))
        assert (got["fail"] == abi.FAIL_NO_OFFERS).all() and len(got["fail"]) > 0
        # no live queue row: returns before any device work, as cook_state_match does
        p.apply(rm=sorted(p.pend))
        got, _ = compare(p.gpu, offers, users, prm, groups=groups, grouped=grouped(p))
        assert len(got["considerable"]) == 0
        q = new_pool("fresh")
        try:
            do, du, dg = derived_inputs(offers, users, groups)
            with pytest.raises(CookError):                 # no rank on a fresh handle
                q.gpu.state_match(do, du, prm, groups=dg, derived=True)
        finally:
            q.close()
    finally:
        p.close()
