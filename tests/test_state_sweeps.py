"""-m gpu: cook_state_task_facts, cook_state_finish, cook_state_group_runtimes and cook_state_sweep against sweep_ref.

The golden scenarios replay on resident handles (upserts, facts, finishes) and each check's sweep must give the
reference's answer.  A churn of eight batches keeps a host mirror of the rows and records and compares every list after
every batch, past one sort tile of rows and records and past a growth and a compaction of the record table.  A group
spread over three handles and a task id two handles hold check the pool column and the orders.  Twin handles show that a
finish is a removal for every other reader, that facts leave the digest and export as they are, and every BADARG leaves
the digest unchanged.  Each call's transfers are checked against its formula.
"""
import numpy as np
import pytest

import resident_model as M
import sweep_ref as W
from cook_b200 import abi, engine
from cook_b200.engine import CookError
from test_state_audit import flat, same_arrays

pytestmark = pytest.mark.gpu

KIND = {"none": abi.SWEEP_NONE, "quantile-deviation": abi.SWEEP_QUANTILE_DEVIATION}


def group_cols(groups, G):
    """state_sweep's group columns of {code: group} over codes [0, G); a code without a group is kind none."""
    cols = {"kind": np.zeros(G, np.int32), "quantile": np.zeros(G), "multiplier": np.zeros(G),
            "n_jobs": np.zeros(G, np.int32)}
    for g, p in groups.items():
        if g >= G:
            continue
        cols["kind"][g] = KIND[p["kind"]]
        cols["quantile"][g] = p.get("quantile", 0.0)
        cols["multiplier"][g] = p.get("multiplier", 0.0)
        cols["n_jobs"][g] = p["n_jobs"]
    return cols


class Mirror:
    """A resident handle and what it should hold for the sweeps: running rows {task id: row} and records [(g, s)]."""

    def __init__(self, name="sweeps"):
        self.e = engine.GpuEngine(pool_name=name)
        self.rows, self.records = {}, []
        # the record table's tail, by the arena rule; grew: past 4096 records; compacted: a compaction that kept
        # records after that growth (into a target made again, as the growth freed it)
        self.tail = self.grew = self.compacted = 0

    def _appended(self, n):
        if self.tail + n > 4096 >= self.tail:
            self.grew = 1
        self.tail += n
        if self.tail - len(self.records) > len(self.records):
            self.compacted |= self.grew and len(self.records) > 0
            self.tail = len(self.records)

    def close(self):
        self.e.close()

    def upsert(self, rows):
        self.e.state_apply(M.delta(run_up=[dict(r, start_time=r["start"]) for r in rows], lists=True))
        for r in rows:
            self.rows[r["task_id"]] = dict(r, max_runtime=-1, status="running", cancelled=False)

    def facts(self, tids, max_runtime=None, cancelled=None, unknown=None):
        self.e.state_task_facts(tids, max_runtime, cancelled, unknown)
        for k, t in enumerate(tids):
            r = self.rows[t]
            if max_runtime is not None:
                r["max_runtime"] = int(max_runtime[k])
            if cancelled is not None:
                r["cancelled"] = bool(cancelled[k])
            if unknown is not None:
                r["status"] = "unknown" if unknown[k] else "running"

    def finish(self, tids, end, ok):
        self.e.state_finish(tids, end, ok)
        n = len(self.records)
        for t, e, s in zip(tids, end, ok):
            r = self.rows.pop(t)
            if s:
                self.records += [(g, W.runtime_s(r["start"], int(e))) for g in r["groups"]]
        self._appended(len(self.records) - n)

    def seed(self, group=(), runtime=(), forget=()):
        self.e.state_group_runtimes(group, runtime, forget)
        self.records = [x for x in self.records if x[0] not in set(forget)] + list(zip(group, runtime))
        self._appended(len(group))


def sweep_all(mirrors, now, dflt, mx, groups, G):
    got = engine.state_sweep([m.e for m in mirrors], now, dflt, mx, group_cols(groups, G))
    rows = [dict(r, pool=k) for k, m in enumerate(mirrors) for r in m.rows.values()]
    records = [x for m in mirrors for x in m.records]
    assert got["linger"] == W.lingering(rows, now, dflt, mx)
    assert got["cancel"] == W.cancelled(rows)
    assert got["straggler"] == W.stragglers(rows, records, groups, now)
    return got


# ---- the golden scenarios, replayed ---------------------------------------------------------------------------
@pytest.mark.parametrize("sc", W.load_golden()["scenarios"], ids=lambda s: s["name"])
def test_golden_replay(sc):
    m = Mirror()
    try:
        rows, records, groups = W.scenario_inputs(sc)
        base = dict(user=0, job_id=1, cpus=1.0, mem=64.0)
        # each success: a row of its group, finished successfully
        succ = [dict(base, task_id=10 ** 6 + i, start=s["start"], groups=[s["group"]]) for i, s in enumerate(sc["successes"])]
        if succ:
            m.upsert(succ)
            m.finish([r["task_id"] for r in succ], [s["end"] for s in sc["successes"]], [1] * len(succ))
        m.upsert([dict(base, task_id=t["task_id"], start=t["start"], groups=t["groups"]) for t in sc["tasks"]])
        tids = [t["task_id"] for t in sc["tasks"]]
        m.facts(tids, max_runtime=[r["max_runtime"] for r in rows], cancelled=[t["cancelled"] for t in sc["tasks"]],
                unknown=[t["status"] == "unknown" for t in sc["tasks"]])
        assert sorted(m.records) == sorted(records)
        G = 1 + max([g for t in sc["tasks"] for g in t["groups"]] + list(groups) + [-1])
        for chk in sc["checks"]:
            got = engine.state_sweep([m.e], chk["now"], chk["default_timeout_ms"], chk["max_timeout_ms"],
                                     group_cols(groups, G))
            W.check_answers(chk, [t for t, _ in got["linger"]], [t for t, _ in got["cancel"]],
                            [[g, t] for g, t, _ in got["straggler"]])
    finally:
        m.close()


# ---- churn -----------------------------------------------------------------------------------------------------
NOW = M.START + 40 * 3_600_000


def churn_groups(rng, G):
    return {g: dict(kind="quantile-deviation" if rng.random() < 0.8 else "none", quantile=float(rng.choice([0.0, 0.3, 0.5, 0.9, 1.0])),
                    multiplier=float(rng.choice([1.0, 1.5, 2.5])), n_jobs=int(rng.integers(1, 60))) for g in range(G)}


def random_rows(rng, n, tid0, G):
    starts = NOW - rng.integers(1000, 30 * 3_600_000, n)
    return [dict(user=0, job_id=1, cpus=1.0, mem=64.0, task_id=tid0 + 3 * i, start=int(starts[i]),
                 groups=sorted(set(rng.integers(0, G, int(rng.choice([0, 1, 1, 2, 3]))).tolist()))) for i in range(n)]


def test_churn():
    rng = np.random.default_rng(71)
    G = 40
    groups = churn_groups(rng, G)
    m = Mirror("churn")
    tid = 1000
    seen = {"linger": 0, "cancel": 0, "straggler": 0, "rows": 0, "records": 0}
    try:
        for batch in range(8):
            m.upsert(random_rows(rng, 1500 if batch < 3 else 300, tid, G))
            tid += 3 * 1500
            if batch == 4:   # a launch: pending rows with group lists become running rows
                pend = [(10 ** 7 + 2 * i, M.group_row(user=0, groups=[int(rng.integers(0, G))])) for i in range(50)]
                m.e.state_apply(M.delta(up=pend, drop=M.drop_all_but("groups")))
                tids = [tid + 3 * i for i in range(50)]
                starts = NOW - rng.integers(1000, 10 ** 7, 50)
                m.e.state_launch([j for j, _ in pend], tids, starts)
                for (j, r), t, s in zip(pend, tids, starts):
                    m.rows[t] = dict(task_id=t, start=int(s), groups=r["groups"], max_runtime=-1, status="running",
                                     cancelled=False)
                tid += 200
            live = sorted(m.rows)
            pick = [t for t in live if rng.random() < 0.15]
            m.facts(pick, max_runtime=rng.choice([-1, 3_600_000, 20 * 3_600_000, 2 ** 62], len(pick)),
                    cancelled=rng.random(len(pick)) < 0.3, unknown=rng.random(len(pick)) < 0.2)
            pick = [t for t in live if rng.random() < 0.05]
            m.facts(pick, cancelled=np.zeros(len(pick), np.uint8))    # one column only: the other bit stays
            done = [t for t in live if rng.random() < 0.2]
            end = [m.rows[t]["start"] + int(rng.integers(0, 5 * 3_600_000)) for t in done]
            m.finish(done, end, rng.random(len(done)) < 0.7)
            if batch in (1, 5):
                m.seed(rng.integers(0, G, 3000).tolist(), rng.integers(0, 20000, 3000).tolist())
            if batch in (3, 6):
                m.seed(forget=[g for g in range(G) if g % 3] + [G + 5])
            got = sweep_all([m], NOW, 8 * 3_600_000, 12 * 3_600_000, groups, G)
            for k in ("linger", "cancel", "straggler"):
                seen[k] += len(got[k])
            seen["rows"] = max(seen["rows"], len(m.rows))
            seen["records"] = max(seen["records"], sum(groups[g]["kind"] != "none" for g, _ in m.records))
        assert all(seen.values()) and seen["rows"] > 2048 and seen["records"] > 2048, seen
        assert m.grew and m.compacted
    finally:
        m.close()


def test_three_handles():
    """Group 0 spread over three handles, judged over all of them; task id 77 held by handles 0 and 2."""
    rng = np.random.default_rng(5)
    ms = [Mirror(f"h{k}") for k in range(3)]
    try:
        groups = {0: dict(kind="quantile-deviation", quantile=0.5, multiplier=2.0, n_jobs=20),
                  1: dict(kind="quantile-deviation", quantile=0.0, multiplier=1.0, n_jobs=2)}
        for k, m in enumerate(ms):
            rows = [dict(user=0, job_id=1, cpus=1.0, mem=64.0, task_id=100 * k + i, start=NOW - 1000 * int(rng.integers(1, 9000)),
                         groups=[0] if i % 3 else [0, 1]) for i in range(1, 40)]
            if k != 1:
                rows.append(dict(user=0, job_id=1, cpus=1.0, mem=64.0, task_id=77, start=NOW - 5 * 3_600_000, groups=[0]))
            m.upsert(rows)
            m.facts([77] if k != 1 else [101], max_runtime=[1000], cancelled=[1])
            m.seed([0] * (k + 4) + [1] * (k == 2), rng.integers(100, 3000, k + 4 + (k == 2)).tolist())
        got = sweep_all(ms, NOW, 3_600_000, 3_600_000, groups, 2)
        assert [p for t, p in got["cancel"] if t == 77] == [0, 2]
        assert {p for _, _, p in got["straggler"]} == {0, 1, 2}
    finally:
        for m in ms:
            m.close()


# ---- a finish is a removal ---------------------------------------------------------------------------------------
def digest_eq(da, db):
    for k in ("pending", "running", "queue", "entries", "consistent", "first_mismatch"):
        assert da[k] == db[k], k
    assert da["consistent"]
    for k in ("pending_buckets", "running_buckets"):
        assert da[k].tobytes() == db[k].tobytes(), k


def test_finish_is_removal():
    rng = np.random.default_rng(9)
    t = M.c2(33)
    pend, run = M.pool_rows(t)
    for r in run.values():
        r["host"] = int(rng.choice(t["offers"].col("hostname_id")))
        r["groups"] = sorted(set(rng.integers(0, 6, int(rng.integers(0, 3))).tolist()))
    a, b = M.Pool.of_trace(t, name="finish"), M.Pool.of_trace(t, name="remove")
    try:
        for p in (a, b):
            p.apply(up=list(pend.items()), run_up=list(run.values()), hosts=True, lists=True)
            p.rank()
        ids = [x for x in run if rng.random() < 0.4]
        end = [run[x]["start_time"] + 1000 * int(rng.integers(0, 10 ** 5)) for x in ids]
        a.gpu.state_task_facts(ids[:50], max_runtime_ms=np.full(50, 5000), cancelled=np.ones(50), unknown=np.ones(50))
        digest_eq(a.gpu.state_digest(16), b.gpu.state_digest(16))
        same_arrays(flat(a.gpu.state_export()), flat(b.gpu.state_export()))
        a.gpu.state_finish(ids, end, rng.random(len(ids)) < 0.6)
        b.gpu.state_apply(abi.make_delta(running_rm=ids))
        digest_eq(a.gpu.state_digest(16), b.gpu.state_digest(16))
        same_arrays(flat(a.gpu.state_export()), flat(b.gpu.state_export()))
        assert np.array_equal(a.gpu.state_queue(), b.gpu.state_queue())
        assert np.array_equal(a.gpu.state_rank(a.users), b.gpu.state_rank(b.users))
        ma = a.gpu.state_match(a.offers, a.users, a.params, derived=True, max_ports=a.max_ports)
        mb = b.gpu.state_match(b.offers, b.users, b.params, derived=True, max_ports=b.max_ports)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
    finally:
        a.close()
        b.close()


def test_upsert_resets_facts_and_reset_drops_records():
    m = Mirror("reset")
    try:
        groups = {0: dict(kind="quantile-deviation", quantile=0.0, multiplier=1.0, n_jobs=1)}
        row = dict(user=0, job_id=1, cpus=1.0, mem=64.0, task_id=5, start=NOW - 3_600_000, groups=[0])
        m.upsert([row])
        m.facts([5], max_runtime=[10], cancelled=[1], unknown=[1])
        m.seed([0], [60])
        got = sweep_all([m], NOW, 10 ** 9, 10 ** 9, groups, 1)
        assert got["cancel"] == [(5, 0)] and got["linger"] == [(5, 0)] and got["straggler"] == []
        m.upsert([row])   # the facts go back to absent
        got = sweep_all([m], NOW, 10 ** 9, 10 ** 9, groups, 1)
        assert got["cancel"] == [] and got["linger"] == [] and got["straggler"] == [(0, 5, 0)]
        m.e.state_apply(abi.make_delta(reset=True))
        m.rows, m.records = {}, []
        m.upsert([row])
        assert sweep_all([m], NOW, 10 ** 9, 10 ** 9, groups, 1)["straggler"] == []
    finally:
        m.close()


# ---- errors and transfers --------------------------------------------------------------------------------------
def test_badargs_leave_digest():
    m = Mirror("bad")
    try:
        groups = {0: dict(kind="quantile-deviation", quantile=0.5, multiplier=1.0, n_jobs=3)}
        m.upsert([dict(user=0, job_id=1, cpus=1.0, mem=64.0, task_id=t, start=NOW - 10 ** 6, groups=[0]) for t in (1, 2, 3)])
        m.seed([0, 0], [5, 6])
        before = m.e.state_digest(16)
        e = m.e
        calls = [lambda: e.state_task_facts([1, 1], cancelled=[1, 1]), lambda: e.state_task_facts([9], cancelled=[1]),
                 lambda: e.state_task_facts([1], max_runtime_ms=[-2]),
                 lambda: e.state_finish([1, 1]), lambda: e.state_finish([9]),
                 lambda: e.state_finish([1], [NOW - 2 * 10 ** 6], [1]),                     # ends before its start
                 lambda: e.state_finish([1], [NOW - 10 ** 6 + 2 ** 31 * 1000], [1]),        # 2^31 s
                 lambda: e.lib.cook_state_finish(e.pool, 1, abi.ptr(np.array([1], np.int64), abi.P_I64), None,
                                                 abi.ptr(np.ones(1, np.uint8), abi.P_U8)),
                 lambda: e.state_group_runtimes([-1], [5]), lambda: e.state_group_runtimes([0], [-5]),
                 lambda: e.state_group_runtimes(forget=[-3]),
                 lambda: engine.state_sweep([e], NOW, 1, 1, group_cols(groups, 0)),           # group code >= n_groups
                 lambda: engine.state_sweep([e], NOW, 1, 1, group_cols({0: dict(groups[0], quantile=1.5)}, 1)),
                 lambda: engine.state_sweep([e], NOW, 1, 1, group_cols({0: dict(groups[0], n_jobs=-1)}, 1)),
                 lambda: engine.state_sweep([e, e], NOW, 1, 1, group_cols(groups, 1)),
                 lambda: engine.state_sweep([e], NOW - 2 * 10 ** 6, 1, 1, group_cols(groups, 1))]   # start after now
        for k, call in enumerate(calls):
            try:
                rc = call()
            except CookError as x:
                rc = x.code
            assert rc == abi.COOK_E_BADARG, k
            d = m.e.state_digest(16)
            assert d["running"] == before["running"] and np.array_equal(d["running_buckets"], before["running_buckets"]), k
        # nothing was written: the records and facts are as before
        sweep_all([m], NOW, 1, 1, groups, 1)
        # a capacity below the live rows
        n = np.zeros(1, np.int32)
        h = (abi.C.c_void_p * 1)(e.pool)
        out = np.zeros(4, np.int64), np.zeros(4, np.int32)
        rc = e.lib.cook_state_sweep(h, 1, NOW, 1, 1, 0, None, None, None, None, 2, abi.ptr(out[0], abi.P_I64),
                                    abi.ptr(out[1], abi.P_I32), abi.ptr(n, abi.P_I32), None, None, None, 0, None, None,
                                    None, None, None)
        assert rc == abi.COOK_E_BADARG
    finally:
        m.close()


def test_transfers():
    m = Mirror("bytes")
    try:
        rng = np.random.default_rng(3)
        m.upsert(random_rows(rng, 500, 10, 8))
        tids = sorted(m.rows)[:100]
        m.facts(tids, max_runtime=np.full(100, 5), cancelled=np.ones(100))
        assert m.e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 100 * (4 + 8 + 1)
        m.facts(tids[:10], unknown=np.ones(10))
        assert m.e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 10 * (4 + 1)
        m.finish(tids[:30], [m.rows[t]["start"] + 5000 for t in tids[:30]], [1] * 30)
        assert m.e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 30 * 13
        m.e.state_finish(tids[30:40])
        for t in tids[30:40]:
            m.rows.pop(t)
        assert m.e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 10 * 4
        m.seed([1, 2, 3], [4, 5, 6], forget=[7, 7, 6])
        assert m.e.last_stats(abi.PHASE_STATE)["h2d_bytes"] == 2 * 4 + 3 * 8
        groups = churn_groups(rng, 8)
        got = sweep_all([m], NOW, 3_600_000, 5 * 3_600_000, groups, 8)
        st = got["stats"]
        assert st["h2d_bytes"] == 24 * 8
        assert st["d2h_bytes"] == 16 + 12 * (len(got["linger"]) + len(got["cancel"])) + 16 * len(got["straggler"])
        assert len(got["linger"]) and len(got["cancel"])
    finally:
        m.close()


def test_kill_lists():
    """cycle.kill_lists: the three lists with the reference's kill reasons, from the timeouts' hours."""
    from cook_b200 import cycle
    m = Mirror("kill")
    try:
        dflt, mx = cycle.lingering_timeouts_ms(timeout_hours=4)
        assert (dflt, mx) == (4 * 3_600_000, 4 * 3_600_000)
        base = dict(user=0, job_id=1, cpus=1.0, mem=64.0)
        m.upsert([dict(base, task_id=1, start=NOW - 5 * 3_600_000, groups=[0]),
                  dict(base, task_id=2, start=NOW - 3 * 3_600_000, groups=[0])])
        m.facts([2], cancelled=[1])
        m.seed([0], [60])
        groups = {0: dict(kind="quantile-deviation", quantile=0.0, multiplier=2.0, n_jobs=1)}
        got = cycle.kill_lists([m.e], NOW, dflt, mx, group_cols(groups, 1))
        assert got == [("max-runtime-exceeded", 1, 0, None), ("straggler", 1, 0, 0), ("straggler", 2, 0, 0),
                       ("reason-killed-by-user", 2, 0, None)]
    finally:
        m.close()
