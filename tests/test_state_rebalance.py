"""cook_state_rebalance: the rebalancer over the resident pool state.

A Python model keeps the same rows as the handle; the resident rebalance must equal cook_rebalance run on host
tables built from the model (running tasks by task id, each on the table index of its hostname code; pending
jobs the first max_preemption allowed jobs of the last rank's queue that are still live), and the oracle, over a
stream of deltas, whatever the slot layout.  Plus: the state is left as it was, the upload accounting, the
errors.  Host codes are a permuted, non-contiguous set, so a host's index differs from its code.
"""
import ctypes as C

import numpy as np
import pytest

from cook_b200 import abi, traces
from cook_b200.engine import CookError, GpuEngine
from resident_model import Pool, decisions_eq, delta, nb, pool_rows, rebalance_trace, remap_hosts, rows_of


@pytest.mark.gpu
@pytest.mark.parametrize("constraints", [False, True])
def test_equivalence_over_deltas(constraints, oracle):
    r, codes = rebalance_trace(71 if constraints else 73, constraints)
    pend, run = rows_of(r, codes)
    p = Pool.of_rebalance(r, codes)
    rng = np.random.default_rng(9)
    try:
        items = sorted(pend.items())
        reserve = items[-60:]
        p.apply(up=items[:-60], run_up=list(run.values()), reset=True)
        t_next = [10 ** 9]
        many_victims = removed_ahead = 0
        for cycle in range(5):
            p.rank()
            # after the rank: the first job the walk would take is killed, one more allowed flag flips (the
            # upsert replaces the job: it leaves the queue), one priority changes
            live = [j for j in p.queue if p.pend[j]["allowed"]]
            kill = [live[0]] + [int(j) for j in rng.choice(live[1:], 2, replace=False)]
            flip = [j for j in p.queue if j not in kill][5]
            prio = [j for j in p.queue if j not in kill and j != flip][7]
            ups = [(flip, dict(p.pend[flip], allowed=1 - p.pend[flip]["allowed"])),
                   (prio, dict(p.pend[prio], priority=int(rng.choice([10, 50, 90]))))]
            p.apply(up=ups, rm=kill)
            got = p.check_rebalance(oracle if cycle % 2 == 0 else None)
            many_victims = max([many_victims] + [len(d["victims"]) for d in got])
            removed_ahead += len(got) > 0
            # churn: the victims die, some tasks finish, some jobs start on random hosts, new jobs arrive,
            # some jobs are disallowed or change priority before the next rank
            dead = {v for d in got for v in d["victims"] if v >= 0 and v in p.run}
            fin = [t for t in p.run if t not in dead and rng.random() < 0.03]
            starts = [j for j in p.pend if rng.random() < 0.05]
            run_up = []
            for j in starts:
                t_next[0] += 1
                row = p.pend[j]
                run_up.append(dict(user=row["user"], priority=row["priority"], start_time=1_700_000_000_000 + t_next[0],
                                   task_id=t_next[0], job_id=j, cpus=row["cpus"], mem=row["mem"], gpus=0.0,
                                   host=int(codes[rng.integers(len(codes))])))
            up = [reserve.pop() for _ in range(min(10, len(reserve)))]
            for j in [j for j in p.pend if j not in starts][:: 17]:
                up.append((j, dict(p.pend[j], allowed=int(rng.random() < 0.7), priority=int(rng.choice([10, 50, 90])))))
            p.apply(up=up, rm=starts, run_up=run_up, run_rm=sorted(dead) + fin)
            if cycle == 2:                           # new leadership
                p.apply(up=sorted(p.pend.items()), run_up=list(p.run.values()), reset=True)
        assert many_victims >= 2, "no decision with several victims"
        assert removed_ahead >= 1, "no cycle decided after the queue's first allowed job was removed"
    finally:
        p.close()


@pytest.mark.gpu
def test_layout_independence():
    r, codes = rebalance_trace(81, True)
    pend, run = rows_of(r, codes)
    for k, t in enumerate(sorted(run)):              # off the binary grid: the serial folds run
        if k % 3 == 0:
            run[t]["cpus"] += 0.1
    for k, j in enumerate(sorted(pend)):
        if k % 4 == 0:
            pend[j]["cpus"] += 0.1
    items = sorted(pend.items())
    a, b = Pool.of_rebalance(r, codes), Pool.of_rebalance(r, codes)
    rng = np.random.default_rng(4)
    try:
        a.apply(up=items, run_up=[run[t] for t in sorted(run)])
        junk = [(10 ** 11 + i, items[i][1]) for i in range(200)]
        jrun = [dict(row, task_id=10 ** 12 + i) for i, row in enumerate(list(run.values())[:500])]
        b.apply(up=junk, run_up=jrun)                # slots the real rows then reuse
        b.apply(rm=[j for j, _ in junk], run_rm=[row["task_id"] for row in jrun])
        perm = rng.permutation(len(items))
        rr = list(run.values())
        b.apply(up=[items[i] for i in perm[: len(perm) // 2]], run_up=[rr[i] for i in rng.permutation(len(rr))])
        b.apply(up=[items[i] for i in perm[len(perm) // 2:]])
        assert a.rank().tolist() == b.rank().tolist()
        ga, gb = a.check_rebalance(), b.check_rebalance()
        assert len(ga) > 0
        decisions_eq(ga, gb)
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_stated_size_c4_pool3():
    r = traces.gen_config_pool("c4", 3)["rebalance"]
    assert (r["running"].col("t").n, r["params"].max_preemption) == (40_000, 128)
    codes = remap_hosts(r, 5)
    pend, run = rows_of(r, codes)
    p = Pool.of_rebalance(r, codes)
    try:
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.rank()
        got = p.check_rebalance()
        assert len(got) > 0
    finally:
        p.close()


def _c3_with_hosts(seed):
    """A config-#3-like pool with offers, its running tasks on the offers' hosts, and the host table."""
    t = traces.gen_c3_pool(seed, n_jobs=2500, n_offers=160, n_users=24, n_running=500)
    o = t["offers"]
    hn = o.col("hostname_id")
    hosts = abi.HostTable(n=o.n, hostname_id=hn, name_rank=o.col("name_rank"), has_spare=np.zeros(o.n, np.uint8),
                          spare_cpus=np.zeros(o.n), spare_mem=np.zeros(o.n), spare_gpus=np.zeros(o.n),
                          n_attr_cols=o.n_attr_cols, attr=o.col("attr"))
    pend, run = pool_rows(t)
    rng = np.random.default_rng(seed)
    for row in run.values():
        row["host"] = int(hn[rng.integers(o.n)])
    return t, hosts, pend, run


@pytest.mark.gpu
def test_state_untouched():
    t, hosts, pend, run = _c3_with_hosts(91)
    prm = abi.RebalanceParams(32, 0.0, 0.0, 0)
    params = traces.match_params(1000)
    mp = int(t["jobs"].col("ports").max()) if t["jobs"].col("ports") is not None else 0
    a, b = GpuEngine(pool_name="a"), GpuEngine(pool_name="b")
    try:
        d = delta(up=sorted(pend.items()), run_up=list(run.values()), hosts=True)
        for e in (a, b):
            e.state_apply(d)
        qa, qb = a.state_rank(t["users"]), b.state_rank(t["users"])
        assert np.array_equal(qa, qb)
        a.state_rebalance(hosts, t["users"], prm, groups=t["groups"])
        ma = a.state_match(t["offers"], t["users"], params, groups=t["groups"], max_ports=mp)
        mb = b.state_match(t["offers"], t["users"], params, groups=t["groups"], max_ports=mp)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
        assert np.array_equal(a.state_rank(t["users"]), qa)
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_accounting():
    r, codes = rebalance_trace(101, True, n_running=2000, n_pending=200, n_hosts=150, n_users=30, mp=16)
    pend, run = rows_of(r, codes)
    h, u, g = r["hosts"], r["users"], r["groups"]
    want = nb(*[h.col(n) for n, _ in h._fields_])
    want += nb(*[u.col(n) for n in ("name_rank", "div_mem", "div_cpus", "quota_count", "quota_cpus", "quota_mem",
                                      "quota_gpus")])
    want += nb(*[g.col(n) for n, _ in g._fields_])
    got = []
    for scale in (1, 2):                             # the same rows, and as many again under new ids
        p = Pool.of_rebalance(r, codes)
        try:
            up = sorted(pend.items())
            rr = list(run.values())
            if scale == 2:
                up += [(j + 10 ** 10, row) for j, row in up]
                rr += [dict(row, task_id=row["task_id"] + 10 ** 10) for row in rr]
            p.apply(up=up, run_up=rr)
            p.rank()
            p.check_rebalance()
            st = p.gpu.last_stats(abi.PHASE_REBALANCE)
            assert st["n_launches"] > 0
            got.append(st["h2d_bytes"])
        finally:
            p.close()
    assert got == [want, want]


@pytest.mark.gpu
def test_errors():
    r, codes = rebalance_trace(111, True, mp=16)
    pend, run = rows_of(r, codes)
    items = sorted(pend.items())
    p = Pool.of_rebalance(r, codes)
    try:
        p.apply(up=items, run_up=list(run.values()))

        def code_of(fn):
            with pytest.raises(CookError) as e:
                fn()
            return e.value.code

        reb = lambda hosts=p.hosts, groups=p.groups: p.gpu.state_rebalance(hosts, p.users, p.rparams, groups=groups)
        assert code_of(reb) == abi.COOK_E_BADARG                 # no rank yet
        q0 = p.rank().tolist()
        r0 = reb()
        assert len(r0) > 0

        def fails(fn, code=abi.COOK_E_BADARG, undo=None):
            assert code_of(fn) == code
            if undo:
                undo()
            assert reb() == r0
            assert p.rank().tolist() == q0
            assert reb() == r0

        R, MP = len(p.run), p.rparams.max_preemption

        def raw(cap, dec=True):
            out = (abi.Decision * MP)()
            jid, vict, n = np.zeros(MP, np.int64), np.zeros(max(cap, 1), np.int64), C.c_int32(0)
            rc = p.gpu.lib.cook_state_rebalance(p.gpu.pool, C.byref(p.hosts), C.byref(p.groups), C.byref(p.users),
                                                C.byref(p.rparams), out if dec else None, abi.ptr(jid, abi.P_I64),
                                                abi.ptr(vict, abi.P_I64), int(cap), C.byref(n))
            if rc != 0:
                p.gpu._err(rc)

        fails(lambda: raw(R + MP, dec=False))                      # a null required argument
        fails(lambda: raw(R + MP - 1))                             # victim_cap below the bound
        raw(R + MP)
        task = dict(next(iter(p.run.values())), task_id=10 ** 13)
        p.gpu.state_apply(delta(run_up=[task]))  # host unknown (-1)
        fails(reb, undo=lambda: p.gpu.state_apply(delta(run_rm=[10 ** 13])))
        p.gpu.state_apply(delta(run_up=[dict(task, host=int(codes.max()) + 1)], hosts=True))   # a code not in the table
        fails(reb, undo=lambda: p.gpu.state_apply(delta(run_rm=[10 ** 13])))
        hn = p.hosts.col("hostname_id").copy()
        hn[1] = hn[0]
        kw = {n: p.hosts.col(n) for n, _ in p.hosts._fields_ if p.hosts.col(n) is not None}
        kw.update(n=p.hosts.n, n_attr_cols=p.hosts.n_attr_cols, hostname_id=hn)
        fails(lambda: reb(hosts=abi.HostTable(**kw)))             # a hostname code twice
        bad_rows = [dict(items[0][1], user=p.users.n_users),       # user, group, attribute column out of range
                    dict(items[0][1], groups=[p.groups.n_groups]),
                    dict(items[0][1], attr=[(p.hosts.n_attr_cols, 1)])]
        for row in bad_rows:
            p.gpu.state_apply(delta(up=[(10 ** 13, row)]))
            fails(reb, undo=lambda: p.gpu.state_apply(delta(rm=[10 ** 13])))
        g = GpuEngine(pool_name="gpu-dru", dru_mode=1)              # GPU DRU mode
        try:
            with pytest.raises(CookError) as e:
                g.state_rebalance(p.hosts, p.users, p.rparams)
            assert e.value.code == abi.COOK_E_UNSUPPORTED_CONSTRAINT
        finally:
            g.close()
    finally:
        p.close()
