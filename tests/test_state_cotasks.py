"""cook_state_cotasks: each group's running cotasks, derived on the device from the resident running rows and the
group lists they carry (running upserts' running_group_off / running_group_idx, or the job's list moved by a launch).

CPU: the StateDelta layout against the C compiler with the new fields, the export and the phase code, and the
restatement in cotask_ref.py on hand-built cases.
GPU (-m gpu): equality with the restatement after every batch of a churn (upserts with and without lists,
replacements, removals, launches with and without hosts, a reset, growth, slot reuse, arena compaction) and
between two handles that reach the same rows by different histories; a launch twin against a delta twin; the edges,
errors and transfer accounting; K13's group answers through the resident path; and multi-cycle config-#3 matches
and a config-#4 rebalance fed from the derived lists against the oracle and the host-table calls.
"""
import ctypes as C

import numpy as np
import pytest

from cook_b200 import abi, engine, traces
from cotask_ref import cotasks
from resident_model import (K13, START, Pool, group_pool, group_row, jobs_soa, keyed, pool_rows, rebalance_trace, rows_of,
                            task_of, tasks_soa)



# ---- CPU -------------------------------------------------------------------------------------------------
def test_restatement_hand_built():
    rows = [dict(task_id=9, host=7, groups=[1]), dict(task_id=3, host=5, groups=[1, 0]),
            dict(task_id=4, host=-1, groups=[0, 1]), dict(task_id=6, host=8, groups=[1]),
            dict(task_id=1, host=5, groups=[])]
    hn = [5, 7]                                    # host 8 is not listed
    attr = [[10, 20], [30, 40]]                    # [column][host index]
    off, host, val = cotasks(rows, 3, [1, 0, -1], hn, attr)
    assert off == [0, 1, 4, 4]                     # group 2 has no entry
    assert host == [5, 5, 8, 7]                    # group 0: task 3; group 1: tasks 3, 6, 9 (task 4 has no host)
    assert val == [30, 10, 0, 20]                  # column 1 for group 0, column 0 for group 1; host 8 -> 0
    assert cotasks(rows, 3, None, hn, attr)[2] == [0, 0, 0, 0]
    assert cotasks(rows, 3, [1, 0, -1])[1:] == (host, [0, 0, 0, 0])
    assert cotasks([], 2) == ([0, 0, 0], [], [])


# ---- GPU helpers -------------------------------------------------------------------------------------------
def host_table(codes, attr):
    """A host table of hostname codes with attribute columns attr[c][h] (only what cook_state_cotasks reads)."""
    attr = np.asarray(attr, np.int32).reshape(-1, len(codes)) if len(codes) else np.zeros((0, 0), np.int32)
    return abi.HostTable(n=len(codes), hostname_id=np.asarray(codes, np.int32), n_attr_cols=attr.shape[0],
                         attr=attr.reshape(-1) if attr.size else None)


def ref_of(rows, G, attr_col, hosts):
    if hosts is None:
        return cotasks(rows, G, attr_col)
    hn = hosts.col("hostname_id")
    at = hosts.col("attr")
    return cotasks(rows, G, attr_col, hn if hn is not None else [], at.reshape(hosts.n_attr_cols, hosts.n) if at is not None else None)


def expected_bytes(G, attr_col, hosts, n):
    """The header's transfer formula; nothing moves without an entry."""
    if n == 0:
        return 0, 0
    H = hosts.n if hosts is not None else 0
    D = len({int(c) for c in attr_col if c >= 0}) if hosts is not None and attr_col is not None and H else 0
    return 4 * H * (1 + D) + 4 * G, 4 * (G + 1) + 8 * n


def check(h, G, attr_col=None, hosts=None):
    got = h.gpu.state_cotasks(G, attr_col, hosts)
    want = ref_of(h.run.values(), G, attr_col, hosts)
    assert got[0].tolist() == want[0] and got[1].tolist() == want[1] and got[2].tolist() == want[2]
    st = h.gpu.last_stats(abi.PHASE_COTASKS)
    assert (st["h2d_bytes"], st["d2h_bytes"]) == expected_bytes(G, attr_col, hosts, len(want[1]))
    return got


def random_running(rng, n, tid0, codes, G, U=8):
    return [group_row(user=int(rng.integers(U)), task_id=tid0 + 3 * i, job_id=10 ** 9 + tid0 + 3 * i,
                 host=int(rng.choice(codes)),
                 groups=[int(g) for g in rng.choice(G, int(rng.choice([0, 0, 1, 1, 1, 2, 3])), replace=False)])
            for i in range(n)]


def random_pending(rng, n, jid0, G, U=8):
    return [group_row(user=int(rng.integers(U)), job_id=jid0 + 2 * i,
                 groups=[int(g) for g in rng.choice(G, int(rng.choice([0, 0, 1, 1, 2])), replace=False)])
            for i in range(n)]


# ---- GPU: churn, layout, launch twin -------------------------------------------------------------------------
@pytest.mark.gpu
def test_churn_matches_the_restatement():
    rng = np.random.default_rng(3)
    G = 60
    listed = rng.permutation(45).astype(np.int32)               # 45..54 are hosts no table lists
    hosts = host_table(listed, rng.integers(0, 6, (3, len(listed))))
    attr_col = rng.integers(-1, 3, G).astype(np.int32)
    codes = list(range(55)) + [-1] * 6
    h = group_pool("cotasks")
    nxt = {"t": 1_000, "j": 5_000_000}

    def fresh_run(n):
        rows = random_running(rng, n, nxt["t"], codes, G)
        nxt["t"] += 3 * n + 3
        return rows

    def fresh_pend(n):
        rows = random_pending(rng, n, nxt["j"], G)
        nxt["j"] += 2 * n + 2
        return rows

    def check_all():
        check(h, G, attr_col, hosts)
        check(h, G)                                               # no table: every value 0
        check(h, G, None, hosts)

    try:
        check_all()                                              # no state yet
        h.apply(run_up=fresh_run(700), up=keyed(fresh_pend(600)))
        check_all()
        for b in range(6):
            fin = [t for t in h.run if rng.random() < 0.05]
            again = [dict(r, host=int(rng.choice(codes)), groups=[int(rng.integers(G))])
                     for r in rng.choice(list(h.run.values()), 25, replace=False) if r["task_id"] not in fin]
            h.apply(run_up=fresh_run(250) + again, up=keyed(fresh_pend(150)), run_rm=fin, lists=b % 3 != 1,
                    hosts=b % 2 == 0)
            check_all()                                          # past 1024, then 2048 running slots
            launch = [int(j) for j in rng.choice(sorted(h.pend), 120, replace=False)]
            tids = [nxt["t"] + 3 * i for i in range(len(launch))]
            nxt["t"] += 3 * len(launch) + 3
            hn = np.array(rng.choice(codes, len(launch)), np.int32) if b % 2 else None
            h.launch(launch, tids, np.full(len(launch), START, np.int64), hn)
            check_all()
        h.apply(run_rm=[t for t in h.run if rng.random() < 0.8])     # dead entries outnumber live: compaction
        check_all()
        h.apply(run_up=fresh_run(400))                               # the freed slots are taken again
        check_all()
        h.apply(reset=True, run_up=fresh_run(900), up=keyed(fresh_pend(50)))
        check_all()
        h.apply(run_rm=list(h.run))
        check_all()                                              # no live row: empty lists
    finally:
        h.close()


@pytest.mark.gpu
def test_layout_independence():
    """The same live rows reached by one batch in id order, or after junk rows whose freed slots the real rows take
    in a permuted order over two batches: identical lists."""
    rng = np.random.default_rng(5)
    G, codes = 40, list(range(30)) + [-1]
    hosts = host_table(np.arange(25, dtype=np.int32), rng.integers(0, 5, (2, 25)))
    attr_col = rng.integers(-1, 2, G).astype(np.int32)
    rows = random_running(rng, 1500, 10, codes, G)
    a, b = group_pool("a"), group_pool("b")
    try:
        a.apply(run_up=sorted(rows, key=lambda r: r["task_id"]))
        junk = random_running(rng, 900, 10_000_000, codes, G)
        b.apply(run_up=junk)
        perm = [rows[i] for i in rng.permutation(len(rows))]
        b.apply(run_up=perm[:700], run_rm=[r["task_id"] for r in junk[:600]])
        b.apply(run_up=perm[700:], run_rm=[r["task_id"] for r in junk[600:]])
        ga, gb = check(a, G, attr_col, hosts), check(b, G, attr_col, hosts)
        assert all(np.array_equal(x, y) for x, y in zip(ga, gb))
        assert len(ga[1]) > 1000
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_launch_against_delta():
    """A launches by id, B receives the equivalent delta (the jobs' removal plus their tasks with the jobs' group
    lists): identical lists after every step, and the launch uploads what it did before group lists existed."""
    rng = np.random.default_rng(9)
    G, codes = 30, list(range(20)) + [-1]
    hosts = host_table(np.arange(20, dtype=np.int32), rng.integers(0, 4, (2, 20)))
    attr_col = rng.integers(-1, 2, G).astype(np.int32)
    a, b = group_pool("launch"), group_pool("delta")
    try:
        pend, run = random_pending(rng, 800, 1_000_000, G), random_running(rng, 300, 10, codes, G)
        for h in (a, b):
            h.apply(up=keyed(pend), run_up=run)
        tid = 100_000
        for step in range(5):
            jobs = [int(j) for j in rng.choice(sorted(a.pend), 90, replace=False)]
            tids = [tid + 3 * i for i in range(len(jobs))]
            tid += 3 * len(jobs) + 3
            hn = np.array(rng.choice(codes, len(jobs)), np.int32) if step % 2 == 0 else None
            a.launch(jobs, tids, np.full(len(jobs), START, np.int64), hn)
            st = a.gpu.last_stats(abi.PHASE_STATE)
            assert st["h2d_bytes"] == len(jobs) * (4 + 4 + 8 + 8) + (4 * len(jobs) if hn is not None else 0)
            tasks = [task_of(b.pend[j], j, t, START, hn[i] if hn is not None else -1) for i, (j, t) in enumerate(zip(jobs, tids))]
            b.apply(rm=jobs, run_up=tasks, hosts=hn is not None)
            fin = [t for t in a.run if rng.random() < 0.3]       # the running arena compacts on both
            for h in (a, b):
                h.apply(run_rm=fin)
            ga, gb = check(a, G, attr_col, hosts), check(b, G, attr_col, hosts)
            assert all(np.array_equal(x, y) for x, y in zip(ga, gb))
            assert np.array_equal(a.gpu.state_rank(abi.make_users(8)), b.gpu.state_rank(abi.make_users(8)))
    finally:
        a.close()
        b.close()


# ---- GPU: edges, errors --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edges():
    h = group_pool("cotasks")
    try:
        hosts = host_table([5, 7], [[11, 12], [21, 22]])
        rows = [group_row(user=0, task_id=10, job_id=1, host=-1, groups=[0, 1]),     # no host: not a cotask
                group_row(user=0, task_id=30, job_id=2, host=9, groups=[1]),         # unlisted host: kept, attribute 0
                group_row(user=1, task_id=20, job_id=3, host=7, groups=[1, 3]),
                group_row(user=1, task_id=40, job_id=4, host=5, groups=[0])]
        h.apply(run_up=rows)
        off, hn, av = check(h, 5, np.array([1, 0, -1, -1, 0], np.int32), hosts)
        assert off.tolist() == [0, 1, 3, 3, 4, 4]                              # groups 2 and 4: empty
        assert hn.tolist() == [5, 7, 9, 7] and av.tolist() == [21, 12, 0, 0]
        assert check(h, 5, np.array([-1] * 5, np.int32), hosts)[2].tolist() == [0, 0, 0, 0]
        assert check(h, 9)[0].tolist() == [0, 1, 3, 3, 4, 4, 4, 4, 4, 4]       # more groups than codes
        lib, pool = h.gpu.lib, h.gpu.pool
        n = C.c_int32(-7)
        assert lib.cook_state_cotasks(pool, 5, None, None, 0, None, None, None, C.byref(n)) == abi.COOK_OK
        assert n.value == 4                                                    # the size query is exact
        n = C.c_int32(-7)
        assert lib.cook_state_cotasks(pool, 5, None, C.byref(hosts), 0, None, None, None, C.byref(n)) == abi.COOK_OK
        assert n.value == 4 and h.gpu.last_stats(abi.PHASE_COTASKS)["h2d_bytes"] == 0
        h.apply(run_rm=[20, 30, 40])
        assert check(h, 5, np.array([1, 0, -1, -1, 0], np.int32), hosts)[0].tolist() == [0] * 6
        h.apply(run_up=[group_row(user=0, task_id=50, job_id=5, host=-1, groups=[4])], hosts=False)
        assert check(h, 5)[0].tolist() == [0] * 6                               # grouped rows, none with a host
    finally:
        h.close()


@pytest.mark.gpu
def test_errors_write_nothing():
    rng = np.random.default_rng(11)
    h = group_pool("cotasks")
    try:
        h.apply(run_up=random_running(rng, 200, 10, list(range(10)), 6))
        hosts = host_table(np.arange(10, dtype=np.int32), rng.integers(1, 5, (2, 10)))
        ac = np.array([0, 1, -1, 0, 1, -1], np.int32)
        want = check(h, 6, ac, hosts)
        N = len(want[1])
        lib, pool = h.gpu.lib, h.gpu.pool
        P = abi.P_I32
        off, hn, av = np.full(7, -9, np.int32), np.full(N + 4, -9, np.int32), np.full(N + 4, -9, np.int32)
        n = C.c_int32(-9)
        dup = host_table(np.array([1, 2, 1], np.int32), np.ones((2, 3)))
        neg = host_table(np.array([1, -2], np.int32), np.ones((2, 2)))
        bad_hn = abi.HostTable(n=3, n_attr_cols=2, attr=np.ones(6, np.int32))
        bad_attr = abi.HostTable(n=10, hostname_id=np.arange(10, dtype=np.int32), n_attr_cols=2)
        neg_n = abi.HostTable(n=-1, hostname_id=np.arange(10, dtype=np.int32))
        ac_hi, ac_lo = np.array([0, 2, -1, 0, 1, -1], np.int32), np.array([0, -2, -1, 0, 1, -1], np.int32)

        def call(G, a, hs, cap, o=off, x=hn, v=av, out=True):
            return lib.cook_state_cotasks(pool, G, abi.ptr(a, P) if a is not None else None,
                                          C.byref(hs) if hs is not None else None, cap,
                                          abi.ptr(o, P) if o is not None else None, abi.ptr(x, P) if x is not None else None,
                                          abi.ptr(v, P) if v is not None else None, C.byref(n) if out else None)
        cases = [
            call(2, ac[:2], hosts, N + 4),                 # n_groups <= a live row's group code
            call(-1, None, hosts, N + 4),                  # n_groups < 0
            call(6, ac, hosts, N - 1),                     # cap < the size
            call(6, ac_hi, hosts, N + 4),                  # attr_col >= n_attr_cols
            call(6, ac_lo, hosts, N + 4),                  # attr_col < -1
            call(6, ac, dup, N + 4),                       # a hostname code twice
            call(6, ac, neg, N + 4),                       # a negative hostname code
            call(6, ac, bad_hn, N + 4),                    # NULL hostname_id
            call(6, ac, bad_attr, N + 4),                  # NULL attr while a group names a column
            call(6, ac, neg_n, N + 4),                     # hosts->n < 0
            call(6, ac, hosts, N + 4, o=None),             # NULL out_cot_off
            call(6, ac, hosts, N + 4, v=None),             # NULL out_cot_attr_val
            call(6, ac, hosts, N + 4, out=False),          # NULL out_n
            call(6, ac, hosts, 0, o=None, x=None, v=None, out=False),   # a size query without out_n
        ]
        assert cases == [abi.COOK_E_BADARG] * len(cases)
        assert n.value == -9 and (off == -9).all() and (hn == -9).all() and (av == -9).all()
        got = check(h, 6, ac, hosts)                        # the handle is unchanged
        assert all(np.array_equal(x, y) for x, y in zip(got, want))
        bad = dict(running=tasks_soa([group_row(user=0, task_id=1, job_id=1)]))
        for o, i in (([1, 1], [1]), ([0, -1], [1]), ([0, 1], [-1])):   # malformed CSR, negative group code
            with pytest.raises(engine.CookError):
                h.gpu.state_apply(abi.make_delta(running_group_off=np.array(o, np.int32),
                                               running_group_idx=np.array(i, np.int32), **bad))
        got = check(h, 6, ac, hosts)
        assert all(np.array_equal(x, y) for x, y in zip(got, want))
    finally:
        h.close()


# ---- GPU: K13 through the resident path --------------------------------------------------------------------
def k13_cycle(p, spec):
    """Rank, derive, match; the same match by the oracle on host tables with host-built lists.  Launches what was
    placed and returns the assignment as offer host names (None: unplaced)."""
    offers = p.offers(spec)
    q = p.e.gpu.state_rank(p.users)
    G = len(p.kind)
    cot = check(p.e, G, p.col, offers)
    want = ref_of(p.e.run.values(), G, p.col, offers)
    prm = traces.match_params(len(q))
    m = p.e.gpu.state_match(offers, p.users, prm, groups=p.groups(cot))
    ids, jobs = p.jobs()
    pos = {j: i for i, j in enumerate(ids)}
    ranked = np.array([pos[j] for j in q], np.int32)
    om = p.o.match(ranked, jobs, offers, p.users, prm, groups=p.groups(want))
    assert np.array_equal(m["considerable"], np.array(ids)[om["considerable"]]) and np.array_equal(m["assign"], om["assign"])
    k = np.arange(len(m["considerable"]), dtype=np.int32)
    fg, fo = p.e.gpu.match_failures(k), p.o.match_failures(ranked, jobs, offers, p.users, prm, k, groups=p.groups(want))
    grp = slice(abi.FAILC_N - 3, abi.FAILC_N)   # unique, balanced, attribute-equals
    assert [(f["n_vms"], f["counts"][grp]) for f in fg] == [(f["n_vms"], f["counts"][grp]) for f in fo]
    p.launch_placed(m, offers)
    return [spec[a]["host"] if a >= 0 else None for a in m["assign"]]


@pytest.mark.gpu
def test_k13_unique_across_cycles(oracle):
    p = K13(oracle, [dict(kind=abi.GROUP_UNIQUE)])
    try:
        host = [dict(host="test-host", cpus=100.0)]
        p.submit(1)
        assert k13_cycle(p, host) == ["test-host"]
        p.submit(1)                                        # its cotask now runs on the only host: 0 placed
        assert k13_cycle(p, host) == [None]
        assert p.e.gpu.state_cotasks(1)[1].tolist() == [0]
    finally:
        p.close()


@pytest.mark.gpu
def test_k13_unique_same_cycle(oracle):
    p = K13(oracle, [dict(kind=abi.GROUP_UNIQUE)])
    try:
        p.submit(2)
        assert k13_cycle(p, [dict(host="test-host", cpus=100.0)]) == ["test-host", None]
    finally:
        p.close()


@pytest.mark.gpu
def test_k13_balanced(oracle):
    p = K13(oracle, [dict(kind=abi.GROUP_BALANCED, col=0, minimum=3)])
    try:
        hosts = [dict(host=h, cpus=100.0, attrs={0: i + 1}) for i, h in enumerate(["straw", "sticks", "bricks"])]
        p.submit(3)
        first = k13_cycle(p, hosts)
        p.submit(6)
        second = k13_cycle(p, hosts)
        assert None not in first + second
        assert sorted(np.unique(first + second, return_counts=True)[1].tolist()) == [3, 3, 3]
    finally:
        p.close()


@pytest.mark.gpu
def test_k13_attribute_equals(oracle):
    EAST, WEST = 1, 2
    p = K13(oracle, [dict(kind=abi.GROUP_ATTR_EQUALS, col=0)])
    try:
        east = dict(host="first-east-host", cpus=1.0, attrs={0: EAST})
        p.submit(1)
        assert k13_cycle(p, [east]) == ["first-east-host"]
        # the cotask's host stays in the offer table, full; 20 one-cpu west offers and a 5-cpu east offer
        offers = [dict(east, cpus=0.5)] + [dict(host=f"west-{i:02d}", cpus=1.0, attrs={0: WEST}) for i in range(20)]
        offers.append(dict(host="east-big", cpus=5.0, attrs={0: EAST}))
        p.submit(20)
        got = k13_cycle(p, offers)
        assert got.count("east-big") == 5 and got.count(None) == 15
    finally:
        p.close()


# ---- GPU: config-#3 match cycles and a config-#4 rebalance -------------------------------------------------------
@pytest.mark.gpu
def test_c3_cycles_against_the_oracle(oracle):
    t = traces.gen_c3_pool(17, n_jobs=2500, n_offers=160, n_users=24, n_running=500)
    rng = np.random.default_rng(19)
    g0, offers, users = t["groups"], t["offers"], t["users"]
    G, kind, acol = g0.n_groups, g0.col("kind"), g0.col("attr_col")
    hn = offers.col("hostname_id")
    pend, run = pool_rows(t)
    for r in run.values():
        r["host"] = int(hn[rng.integers(len(hn))]) if rng.random() < 0.95 else -1
        r["groups"] = [int(rng.integers(G))] if rng.random() < 0.2 else []
    items = sorted(pend.items())
    cut = int(len(items) * 0.7)
    reserve = items[cut:]
    m = Pool("c3", send_hosts=True, send_lists=True)
    e, ref, apply = m.gpu, m.ref, m.apply

    prm = traces.match_params(1000, host_lifetime_mins=t.get("host_lifetime_mins", 0))
    max_ports = int(t["jobs"].col("ports").max())
    hosts_attr = offers.col("attr").reshape(offers.n_attr_cols, offers.n)
    tid = 10 ** 9
    try:
        apply(up=items[:cut], run_up=list(run.values()), reset=True)
        n_cot = 0
        for cycle in range(5):
            q = e.state_rank(users)
            cot = e.state_cotasks(G, acol, offers)
            want = cotasks(m.run.values(), G, acol, hn, hosts_attr)
            assert [x.tolist() for x in cot] == list(want)
            n_cot = max(n_cot, len(want[1]))
            gr = abi.Groups(n_groups=G, kind=kind, attr_col=acol, minimum=g0.col("minimum"), cot_off=cot[0],
                            cot_hostname_id=cot[1] if len(cot[1]) else np.zeros(1, np.int32),
                            cot_attr_val=cot[2] if len(cot[2]) else np.zeros(1, np.int32))
            gh = abi.Groups(n_groups=G, kind=kind, attr_col=acol, minimum=g0.col("minimum"),
                            cot_off=np.array(want[0], np.int32), cot_hostname_id=np.array(want[1] or [0], np.int32),
                            cot_attr_val=np.array(want[2] or [0], np.int32))
            got = e.state_match(offers, users, prm, groups=gr, max_ports=max_ports)
            _, _, jobs, jid = m.tables()
            pos = {j: i for i, j in enumerate(jid.tolist())}
            ranked = np.array([pos[j] for j in q.tolist()], np.int32)
            hm = ref.match(ranked, jobs, offers, users, prm, groups=gh, max_ports=max_ports)
            om = oracle.match(ranked, jobs, offers, users, prm, groups=gh, max_ports=max_ports)
            assert np.array_equal(got["considerable"], jid[hm["considerable"]])
            for k in ("assign", "ports", "fail"):
                assert np.array_equal(got[k], hm[k]), k
            assert np.array_equal(hm["considerable"], om["considerable"]) and np.array_equal(hm["assign"], om["assign"])
            placed = got["assign"] >= 0
            jl = got["considerable"][placed].tolist()
            assert jl
            tids = [tid + 3 * i for i in range(len(jl))]
            tid += 3 * len(jl) + 3
            hosts = hn[got["assign"][placed]].astype(np.int32)
            m.launch(jl, tids, np.full(len(jl), START, np.int64), hosts)
            fin = [x for x in m.run if rng.random() < 0.03]
            new = [reserve.pop() for _ in range(min(len(reserve), len(fin) + 20))]
            for _, r in new[:10]:                           # new members of existing groups
                r["groups"] = sorted({*r["groups"], int(rng.integers(G))})
            apply(up=new, run_rm=fin)
        assert n_cot > 50
    finally:
        m.close()


@pytest.mark.gpu
def test_c4_rebalance_from_derived_lists(oracle):
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
        p.rank()
        acol = g0.col("attr_col")
        cot = p.gpu.state_cotasks(G, acol, hosts)
        want = cotasks(p.run.values(), G, acol, hosts.col("hostname_id"), hosts.col("attr").reshape(hosts.n_attr_cols, hosts.n))
        assert [x.tolist() for x in cot] == list(want) and len(want[1]) > 300
        p.groups = abi.Groups(n_groups=G, kind=g0.col("kind"), attr_col=acol, minimum=g0.col("minimum"),
                              cot_off=cot[0], cot_hostname_id=cot[1], cot_attr_val=cot[2])
        p.check_rebalance(oracle)
    finally:
        p.close()
