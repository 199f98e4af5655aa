"""cook_state_job_facts and cook_state_match_metrics: the match-cycle metrics of a resident pool's last match round.

GPU (-m gpu): a churn of C2-shaped (on and off the grid) and config-#3-shaped cycles (deltas, rank, match, facts,
metrics with dropped matches, launches), every output checked bit for bit after every cycle against match_metrics_ref
fed the round's downloaded considerable ids, the device counts against PoolCycle.unmatched_cycles, and a twin handle
that never calls the new calls keeping identical outputs; the golden rounds replayed on resident handles, the 500 /
501 boundary included; the facts' reset by an upsert and the count kept across one; the BADARGs with the digest
unchanged; the key_cap retry; the transfer formula.
"""
import numpy as np
import pytest

import match_metrics_ref as MR
from cook_b200 import abi, cycle, traces
from cook_b200.engine import CookError, GpuEngine
from resident_model import Pool, c2, c3, churn, delta, pool_rows

pytestmark = pytest.mark.gpu


def _facts(rng, jids):
    """Random job facts for `jids`: {job id: fact dict}, and the columns cook_state_job_facts takes."""
    out = {}
    for j in jids:
        f = 0
        if rng.random() < 0.3:
            f |= abi.JF_GPUS
        if rng.random() < 0.3:
            f |= abi.JF_DISK | (abi.JF_DISK_REQUEST if rng.random() < 0.8 else 0) | \
                (abi.JF_DISK_LIMIT if rng.random() < 0.6 else 0)
        if rng.random() < 0.0005:
            f |= abi.JF_URIS
        out[j] = dict(facts=f, gpu_model=int(rng.integers(-1, 3)), disk_type=int(rng.integers(-1, 2)),
                      disk_request=float(rng.choice([1024.0, 0.3, 2048.5])),
                      disk_limit=float(rng.choice([4096.0, 0.7])))
    cols = {k: np.array([out[j][k] for j in jids]) for k in ("gpu_model", "disk_type", "disk_request", "disk_limit")}
    return out, np.array([out[j]["facts"] for j in jids], np.uint8), cols


def _jobs(p, facts, ids):
    jobs = []
    for j in ids:
        r = p.pend[j]
        f = facts.get(j, {"facts": 0})
        jobs.append(dict(job_id=j, user=r["user"], cpus=r["cpus"], mem=r["mem"], gpus=r["gpus"], ports=r["ports"],
                         **{k: f.get(k, 0) for k in ("facts", "gpu_model", "disk_type", "disk_request", "disk_limit")}))
    return jobs


def _check(got, want, jobs):
    for k in ("considerable", "matched", "head_job_id", "head_matched", "too_long", "uris", "uris_position"):
        assert got[k] == want[k], k
    assert got["first"] == want["first"]
    assert got["user_considerable"].tolist() == want["user_considerable"]
    assert got["user_matched"].tolist() == want["user_matched"]
    if not want["considerable"]:
        return
    assert got["keys"] == want["keys"]
    assert got["total_cpus"] == want["total_cpus"] and got["total_mem"] == want["total_mem"]
    assert got["pct_cpus"] == want["pct_cpus"] and got["pct_mem"] == want["pct_mem"]
    head, lc, lm = got["rows"]
    assert head["position"] == 0 and head["job_id"] == jobs[0]["job_id"]
    assert lc["position"] == want["largest_cpus"] and lm["position"] == want["largest_mem"]
    for row in (head, lc, lm):
        j = jobs[row["position"]]
        for k in ("job_id", "user", "ports", "facts", "cpus", "mem", "gpus"):
            assert row[k] == j[k], k
        assert row["gpu_model"] == (j["gpu_model"] if j["facts"] & abi.JF_GPUS else -1)
        assert row["disk_type"] == (j["disk_type"] if j["facts"] & abi.JF_DISK else -1)
        assert row["disk_request"] == (j["disk_request"] if j["facts"] & abi.JF_DISK_REQUEST else 0.0)


def _fp(pool):
    return {k: v for k, v in pool.gpu.state_digest().items() if k in ("pending", "running", "queue")}


def _phase(pool, phase):
    st = pool.gpu.last_stats(phase)
    return {k: st[k] for k in ("h2d_bytes", "d2h_bytes", "n_launches")}


@pytest.mark.parametrize("kind", ["c2", "c2_offgrid", "c3"])
def test_churn(kind):
    """Every output against the restatement after every cycle; the device counts against PoolCycle.unmatched_cycles;
    a twin handle fed the same deltas that never calls the new calls keeps identical rank, match, launch and digest
    outputs, transfers and launches."""
    t = {"c2": lambda: c2(21), "c2_offgrid": lambda: c2(22, cpus=(0.1, 0.5, 1.0, 2.7)),
         "c3": lambda: c3(23)}[kind]()
    rng = np.random.default_rng(5)
    groups = t.get("groups")
    p = Pool.of_trace(t, groups=groups, name="metrics")
    twin = Pool.of_trace(t, groups=groups, name="twin")
    for q in (p, twin):
        q.params = traces.match_params(3000, host_lifetime_mins=t.get("host_lifetime_mins", 0))
    U = p.users.n_users
    pc = cycle.PoolCycle(engine=None)
    sizes = []
    try:
        pend, run = pool_rows(t)
        items = sorted(pend.items())
        cut = int(len(items) * 0.85)
        reserve = items[cut:]
        for q in (p, twin):
            q.apply(up=items[:cut], run_up=list(run.values()), reset=True)
        t_next = [10 ** 9]
        prev = {}        # the restated counts
        for cyc in range(6):
            live = sorted(p.pend)
            facts, flags, cols = _facts(rng, live)
            p.gpu.state_job_facts(live, flags, **cols)
            assert np.array_equal(p.rank(), twin.rank())
            assert _phase(p, abi.PHASE_RANK) == _phase(twin, abi.PHASE_RANK)
            m = p.gpu.state_match(p.offers, p.users, p.params, groups=groups, max_ports=p.max_ports)
            mt = twin.gpu.state_match(twin.offers, twin.users, twin.params, groups=groups, max_ports=twin.max_ports)
            for k in ("considerable", "assign", "ports", "fail"):
                assert np.array_equal(m[k], mt[k]), k
            assert _phase(p, abi.PHASE_MATCH) == _phase(twin, abi.PHASE_MATCH)
            ids = [int(j) for j in m["considerable"]]
            sizes.append(len(ids))
            assigned = [k for k, a in enumerate(m["assign"]) if a >= 0]
            dropped = sorted(rng.choice(assigned, size=min(len(assigned), 7), replace=False).tolist()) \
                if assigned else []
            if cyc == 2 and assigned and 0 in assigned:
                dropped = sorted(set(dropped) | {0})   # a dropped head
            thr = 1 if cyc % 2 else 2
            got = p.gpu.state_match_metrics(U, dropped, unmatched_warn_cycles=thr, key_cap=1)
            jobs = _jobs(p, facts, ids)
            matched = set(assigned) - set(dropped)
            want = MR.answer(jobs, matched, prev, thr, U)
            _check(got, want, jobs)
            assert got["stats"]["h2d_bytes"] == 4 * len(dropped)
            assert got["stats"]["d2h_bytes"] == MR.down_bytes(len(ids), U, len(want["keys"]))
            prev = want["cycles"]
            mj = {ids[k] for k in matched}
            pc._finish(np.zeros(0, np.int32), [{"jobs": list(mj)}] if mj else [], mj, set(), True, len(ids), 3000,
                       considerable=ids)
            over = [j for j in ids if pc.unmatched_cycles.get(j, 0) > thr]
            assert got["too_long"] == len(over)
            assert got["first"] == [(j, pc.unmatched_cycles[j]) for j in over[:10]]
            launched = [ids[k] for k in sorted(matched)][:40]
            up, rm, run_up, run_rm = churn(p, rng, reserve, t_next, launched)
            for q in (p, twin):
                q.apply(up, rm, run_up, run_rm)
            assert _phase(p, abi.PHASE_STATE) == _phase(twin, abi.PHASE_STATE)
            assert _fp(p) == _fp(twin)
        assert max(sizes) > 2048   # past one sort tile
    finally:
        p.close()
        twin.close()


def _empty_offers():
    return abi.OffersSoA(n=0, hostname_id=np.zeros(1, np.int32), name_rank=np.zeros(1, np.int32), cpus=np.zeros(1),
                         mem=np.zeros(1), run_cpus=np.zeros(1), run_mem=np.zeros(1), run_count=np.zeros(1, np.int32),
                         n_attr_cols=0)


def test_golden_replay():
    """The golden rounds without matches on a resident handle: the jobs upserted in take order (priorities falling),
    their facts sent, rank, a match against no offer, the metrics.  Rounds keep the handle, so the counts carry over,
    to the 500 / 501 boundary."""
    import test_match_metrics_reference as T
    g = T.GOLDEN
    U = g["n_users"]
    users = abi.make_users(U)
    for name, case in g["rounds"].items():
        if any(r["assigned"] for r in case):
            continue
        e = GpuEngine(pool_name="golden")
        try:
            held = set()
            for r, jobs, a in T.replay(case, g["threshold"], U):
                ids = [j["job_id"] for j in jobs]
                up = [(j["job_id"], dict(user=j["user"], priority=1000 - k, cpus=j["cpus"], mem=j["mem"],
                                         gpus=j["gpus"], ports=j["ports"])) for k, j in enumerate(jobs)]
                e.state_apply(delta(up=up, rm=sorted(held - set(ids)), drop=("novel", "attr", "groups")))
                held = set(ids)
                if jobs:
                    e.state_job_facts(ids, np.array([j["facts"] for j in jobs], np.uint8),
                                      gpu_model=np.array([j["gpu_model"] for j in jobs], np.int32),
                                      disk_request=np.array([j["disk_request"] for j in jobs]),
                                      disk_limit=np.array([j["disk_limit"] for j in jobs]),
                                      disk_type=np.array([j["disk_type"] for j in jobs], np.int32))
                e.state_rank(users)
                m = e.state_match(_empty_offers(), users, traces.match_params(len(jobs)))
                assert [int(x) for x in m["considerable"]] == ids
                got = e.state_match_metrics(U, unmatched_warn_cycles=g["threshold"])
                _check(got, a, jobs)
                if not r.get("repeat"):
                    T.check_want(a, r["want"], jobs)
        finally:
            e.close()


def _small_pool():
    t = c2(31)
    p = Pool.of_trace(t, name="metrics-small")
    p.params = traces.match_params(2000)
    pend, run = pool_rows(t)
    p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
    return p


def test_badargs_and_counts_across_upserts():
    p = _small_pool()
    U = p.users.n_users
    try:
        with pytest.raises(CookError) as e:
            p.gpu.state_match_metrics(U)          # no round yet
        assert e.value.code == abi.COOK_E_BADARG
        p.rank()
        m = p.gpu.state_match(p.offers, p.users, p.params, max_ports=p.max_ports)
        ids = [int(j) for j in m["considerable"]]
        unassigned = [k for k, a in enumerate(m["assign"]) if a < 0]
        assigned = [k for k, a in enumerate(m["assign"]) if a >= 0]
        assert unassigned and assigned
        fp = lambda: {k: v for k, v in p.gpu.state_digest().items() if k in ("pending", "running", "queue")}
        digest = fp()
        bad = [dict(dropped=[len(ids)]), dict(dropped=[assigned[0], assigned[0]]), dict(dropped=[unassigned[0]]),
               dict(dropped=[-1]), dict(unmatched_warn_cycles=-1)]
        for kw in bad:
            with pytest.raises(CookError) as e:
                p.gpu.state_match_metrics(U, **kw)
            assert e.value.code == abi.COOK_E_BADARG, kw
        with pytest.raises(CookError) as e:
            p.gpu.state_match_metrics(0)
        assert e.value.code == abi.COOK_E_BADARG
        assert fp() == digest
        # a considerable row upserted since the match refuses the round; another row does not
        j0 = ids[unassigned[0]]
        other = next(j for j in p.pend if j not in set(ids))
        p.apply(up=[(other, dict(p.pend[other]))])
        got = p.gpu.state_match_metrics(U, key_cap=0)
        assert got["considerable"] == len(ids)
        assert got["stats"]["d2h_bytes"] == MR.down_bytes(len(ids), U, got["keys_n"], changed=True)
        with pytest.raises(CookError) as e:
            p.gpu.state_match_metrics(U)          # already counted
        assert e.value.code == abi.COOK_E_BADARG
        assert got["too_long"] == 0 and got["first"] == []   # nothing passes 500 cycles in one round
        # the count is kept across an upsert of the same id, and the facts are reset by it
        p.gpu.state_job_facts([j0], np.array([abi.JF_GPUS], np.uint8), gpu_model=np.array([1], np.int32))
        p.apply(up=[(j0, dict(p.pend[j0]))])
        p.rank()
        m = p.gpu.state_match(p.offers, p.users, p.params, max_ports=p.max_ports)
        ids2 = [int(j) for j in m["considerable"]]
        k0 = ids2.index(j0)
        assert m["assign"][k0] < 0
        p.apply(up=[(ids2[k0], dict(p.pend[ids2[k0]]))])   # changed since the match: refused, nothing counted
        with pytest.raises(CookError) as e:
            p.gpu.state_match_metrics(U)
        assert e.value.code == abi.COOK_E_BADARG
        p.rank()
        m = p.gpu.state_match(p.offers, p.users, p.params, max_ports=p.max_ports)
        ids3 = [int(j) for j in m["considerable"]]
        got = p.gpu.state_match_metrics(U, unmatched_warn_cycles=1)
        k0 = ids3.index(j0)
        assert m["assign"][k0] < 0
        assert got["too_long"] >= 1 and all(c == 2 for _, c in got["first"])   # unmatched in both counted rounds
        assert got["keys"] == []   # the upsert reset the gpus fact
        # an empty round zeroes the counts
        p.rank()
        m = p.gpu.state_match(p.offers, p.users, traces.match_params(0))
        got = p.gpu.state_match_metrics(U)
        assert got["considerable"] == 0 and got["head_job_id"] == -1 and got["stats"]["d2h_bytes"] == 0
    finally:
        p.close()


def test_key_cap_retry():
    p = _small_pool()
    U = p.users.n_users
    try:
        live = sorted(p.pend)
        flags = np.full(len(live), abi.JF_GPUS | abi.JF_DISK | abi.JF_DISK_REQUEST, np.uint8)
        p.gpu.state_job_facts(live, flags, gpu_model=np.arange(len(live), dtype=np.int32) % 5,
                              disk_type=np.zeros(len(live), np.int32), disk_request=np.full(len(live), 10.0))
        p.rank()
        m = p.gpu.state_match(p.offers, p.users, p.params, max_ports=p.max_ports)
        n = len(m["considerable"])
        k = len({int(x) % 5 for x in np.searchsorted(live, m["considerable"])}) + 1
        counts = np.zeros(abi.MMC_N, np.int64)
        z = lambda n, t: np.zeros(n, t)
        rc = p.gpu.lib.cook_state_match_metrics(
            p.gpu.pool, U, 0, None, 500, 0, abi.ptr(counts, abi.P_I64), abi.ptr(z(abi.MMA_N, np.float64), abi.P_F64),
            abi.ptr(z(21, np.int64), abi.P_I64), abi.ptr(z(15, np.float64), abi.P_F64),
            abi.ptr(z(10, np.int64), abi.P_I64), abi.ptr(z(10, np.int32), abi.P_I32), abi.ptr(z(U, np.int32), abi.P_I32),
            abi.ptr(z(U, np.int32), abi.P_I32), abi.ptr(z(1, np.int32), abi.P_I32), abi.ptr(z(1, np.int32), abi.P_I32),
            abi.ptr(z(1, np.float64), abi.P_F64), None)
        assert rc == abi.COOK_E_TOO_LARGE and counts[abi.MMC_KEYS] == k
        got = p.gpu.state_match_metrics(U, key_cap=0)   # retried with the reported count; the round was not counted
        assert len(got["keys"]) == k and got["considerable"] == n
        assert got["keys"][-1] == (abi.MM_DISK_REQUEST, 0, 10.0 * n)
    finally:
        p.close()


def test_job_facts_badargs():
    p = _small_pool()
    try:
        j = sorted(p.pend)[:2]
        for kw in (dict(flags=np.array([32, 0], np.uint8)), dict(flags=np.array([abi.JF_DISK_REQUEST, 0], np.uint8)),
                   dict(gpu_model=np.array([-2, 0], np.int32)), dict(disk_request=np.array([np.nan, 0.0]))):
            with pytest.raises(CookError) as e:
                p.gpu.state_job_facts(j, **kw)
            assert e.value.code == abi.COOK_E_BADARG
        with pytest.raises(CookError):
            p.gpu.state_job_facts([j[0], j[0]], flags=np.zeros(2, np.uint8))
        p.gpu.state_job_facts(j, flags=np.array([abi.JF_GPUS, 0], np.uint8), gpu_model=np.array([3, 0], np.int32))
        assert p.gpu.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 2 * (4 + 1 + 4)
    finally:
        p.close()
