"""-m gpu: cook_state_user_stats, cook_state_instance_stats, cook_state_history_stats and cook_state_list_completed over
handle sets whose rows reach pools[0] through the gather step (state.cu): a handle on another device compacts its rows on
its own stream into its own scratch, and pools[0]'s stream copies them into its range with cudaMemcpyPeerAsync.

Two layouts.  staged: every handle on device 0 with COOK_STAGE_HANDLES=1, so each handle after pools[0] takes the gather
path, and every call through engine is made twice, without and with the variable, the answers and their transfers and
launch counts equal.  two: the handles alternate over devices 1 and 0, pools[0] on device 1 (skipped when one device is
visible).  In both, the churn drivers of the resident tests run unchanged over three handles past one sort tile and check
each call after every batch, bit for bit, against instance_stats_ref, history_ref, completed_ref and monitor_ref; the
seg_cap retry of history stats finds the segments needed over all handles.  The cases of their own: pools[0] holding no
row, a handle whose selection is empty, a job whose latest record is on a later handle than an older one and the
reverse, a user past 2^43 in a quota group's folds (off the exact grid).  The calls without a gather step still refuse
handles on two devices.
"""
import itertools
import struct

import numpy as np
import pytest

import completed_ref as CR
import history_ref as Hr
import list_ref as L
import resident_model as M
import test_state_history_stats as THS
import test_state_instance_stats as TIS
import test_state_list_completed as TLC
import test_state_monitor as TM
from cook_b200 import abi, engine
from cook_b200.engine import CookError

pytestmark = pytest.mark.gpu

STAGE = "COOK_STAGE_HANDLES"
GATHERED = ("state_user_stats", "state_instance_stats", "state_history_stats", "state_list_completed")


def device_count():
    import torch
    return torch.cuda.device_count()


def canon(x):
    """An answer with every float as its bits and the statistics without their times."""
    if isinstance(x, dict):
        return {k: ({s: v for s, v in x[k].items() if not s.startswith("ms_")} if k == "stats" else canon(x[k]))
                for k in sorted(x)}
    if isinstance(x, np.ndarray):
        return (str(x.dtype), x.shape, x.tobytes())
    if isinstance(x, (list, tuple)):
        return [canon(v) for v in x]
    if isinstance(x, float):
        return struct.unpack("<q", struct.pack("<d", x))[0]
    return x


def outcome(fn, a, k):
    try:
        return fn(*a, **k), None
    except CookError as e:
        return None, e


def twice(monkeypatch, fn):
    """fn made once without COOK_STAGE_HANDLES and once with it; both answers (or error codes) equal.  Returns the
    staged answer, the variable left set."""
    def call(*a, **k):
        monkeypatch.delenv(STAGE, raising=False)
        plain, pe = outcome(fn, a, k)
        monkeypatch.setenv(STAGE, "1")
        got, ge = outcome(fn, a, k)
        assert (pe and pe.code) == (ge and ge.code)
        if ge:
            raise ge
        assert canon(plain) == canon(got)
        return got
    return call


@pytest.fixture(params=["staged", "two"])
def layout(request, monkeypatch):
    if request.param == "two":
        if device_count() < 2:
            pytest.skip("one CUDA device visible: handles on two devices need two")
        monkeypatch.delenv(STAGE, raising=False)
        init, seq = engine.GpuEngine.__init__, itertools.count()

        def placed(self, pool_name="no-pool", dru_mode=0, device=None, lib=None):
            init(self, pool_name, dru_mode, (1 if next(seq) % 2 == 0 else 0) if device is None else device, lib)
        monkeypatch.setattr(engine.GpuEngine, "__init__", placed)
    else:
        monkeypatch.setenv(STAGE, "1")
        for name in GATHERED:
            monkeypatch.setattr(engine, name, twice(monkeypatch, getattr(engine, name)))
    return request.param


# ---- the resident tests' churns and edges over the gather step ----------------------------------------------------
REUSED = [
    ("instance_stats-churn-grid", TIS.test_churn, ("grid",)),
    ("instance_stats-churn-off", TIS.test_churn, ("off",)),
    ("instance_stats-golden-edges", TIS.test_golden_edges, ()),
    ("history_stats-churn-grid", THS.test_churn, ("grid",)),
    ("history_stats-churn-off", THS.test_churn, ("off",)),
    ("history_stats-golden-edges", THS.test_golden_edges, ()),
    ("history_stats-seg-cap-retry", THS.test_seg_cap_retry, ()),
    ("list_completed-churn", TLC.test_churn_against_the_restatement, ()),
    ("user_stats-quota-group", TM.test_quota_group_of_three_handles, ()),
]


@pytest.mark.parametrize("test,args", [r[1:] for r in REUSED], ids=[r[0] for r in REUSED])
def test_resident_driver(layout, test, args):
    test(*args)


# ---- the quota group's folds: a churn over three handles, pools[0] empty, a user past 2^43 ------------------------
@pytest.mark.parametrize("regime", ["off", "mixed"])
def test_user_stats_churn(layout, regime):
    rng = np.random.default_rng({"off": 61, "mixed": 62}[regime])
    U = 40
    pools = [TM.stats_pool(f"md-us{k}") for k in range(3)]
    empty, only_run = TM.stats_pool("md-us-empty"), TM.stats_pool("md-us-run")
    tid, jid = [1_000], [5_000_000]

    def runs(n):
        rows = M.random_rows(rng, regime, n, U, tid[0], list(range(20)))
        tid[0] += 2 * n + 2
        return rows

    def jobs(n):
        rows = M.pending_rows(rng, regime, n, U, jid[0], TM.CODES)
        jid[0] += 2 * n + 2
        return M.keyed(rows)

    try:
        for p in pools:
            p.apply(run_up=runs(500), up=jobs(600))
        only_run.apply(run_up=runs(300))   # no pending row: it takes no part in the waiting fold
        for b in range(4):
            t = TM._table(rng, U, [r for p in pools for r in p.run.values()])
            got = TM.check(pools, U, t)
            TM.check([empty] + pools, U, t)                            # pools[0] holds no row
            TM.check([pools[2], only_run, empty, pools[0]], U, t)
            if regime == "mixed":   # user 0 passes 2^43 over the handles: the serial chain, not a scan
                assert got["mem"][abi.STATS_WAITING][0] > 2.0 ** 43 and got["mem"][abi.STATS_RUNNING][0] > 2.0 ** 43
            for p in pools:
                fin = [k for k in p.run if rng.random() < 0.05]
                p.apply(run_up=runs(150), up=jobs(200), run_rm=fin, rm=list(rng.choice(sorted(p.pend), 30, replace=False)))
                launch = list(rng.choice(sorted(p.pend), 120, replace=False))
                tids = [tid[0] + 2 * i for i in range(len(launch))]
                tid[0] += 2 * len(launch) + 2
                p.launch(launch, tids, np.full(len(launch), M.START, np.int64))
            assert sum(len(p.run) + len(p.pend) for p in pools) > 2048
        TM.check([empty], U, t)                                         # no row at all: no device work
    finally:
        for p in pools + [empty, only_run]:
            p.close()


# ---- instance stats: pools[0] empty, a handle whose rows are all unknown -------------------------------------------
def test_instance_stats_empty_lead_and_selection(layout):
    rng = np.random.default_rng(71)
    ps = TIS.Pools(["e", "a", "b", "u"])
    try:
        rows = M.random_rows(rng, "off", 5400, 12, 10 ** 6, [-1])
        for r in rows:
            r.update(start_time=M.START - int(rng.integers(0, 10 ** 6)), reason=int(rng.choice([-1, 1001, 2003])))
        ps.load([[], [dict(r, unknown=bool(rng.random() < 0.3)) for r in rows[:2500]], rows[2500:4000],
                 [dict(r, unknown=True) for r in rows[4000:]]])
        now = M.START + 1
        for status in ("running", "unknown"):   # u selects nothing running, b nothing unknown
            ps.check(now, status, 0, now)
            ps.check(now, status, 0, now, idx=[3, 1, 0, 2])
            ps.check(now, status, M.START - 400_000, M.START - 100_000, 10 ** 6 + 2000, 10 ** 6 + 9000)
        ps.check(now, "running", 0, now, idx=[0, 3])                    # rows gathered, none selected
    finally:
        ps.close()


# ---- history stats: pools[0] empty, a handle with no success -------------------------------------------------------
def test_history_stats_empty_lead_and_selection(layout):
    rng = np.random.default_rng(72)
    ps = THS.Pools(["e", "a", "f", "b"])
    since = M.START - 10 ** 7

    def rows(n, t0, success):
        out = []
        for i in range(n):
            s = since + int(rng.integers(0, 10 ** 6))
            out.append(dict(task_id=t0 + 3 * i, user=int(rng.integers(0, 9)), start=s, end=s + int(rng.integers(0, 90000)),
                            cpus=float(rng.choice([0.1, 0.5, 2.0])), mem=float(rng.integers(1, 9000)) / 7.0,
                            success=success(i), reason=int(rng.choice([-1, 1001, 3001]))))
        return out

    try:
        THS.seed(ps.e[0], ps.h[0], since, [])
        THS.seed(ps.e[1], ps.h[1], since, rows(2200, 10, lambda i: bool(rng.integers(0, 2))))
        THS.seed(ps.e[2], ps.h[2], since, rows(900, 11, lambda i: False))    # no success: an empty selection
        THS.seed(ps.e[3], ps.h[3], since, rows(1400, 12, lambda i: bool(rng.integers(0, 2))))
        for status in (Hr.SUCCESS, Hr.FAILED):
            ps.check(status, since, since + 10 ** 7)
            ps.check(status, since, since + 10 ** 7, idx=[2, 0, 3, 1])
            ps.check(status, since + 200_000, since + 700_000, 1000, 5000)
        THS.check([ps.e[k] for k in (0, 2, 1, 3)], [ps.h[k] for k in (0, 2, 1, 3)], Hr.FAILED, since,
                  since + 10 ** 7, seg_cap=1)   # the retry: the segments needed over every handle
        ps.check(Hr.SUCCESS, since, since + 10 ** 7, idx=[0, 2])         # nothing selected anywhere
    finally:
        ps.close()


# ---- list_completed: pools[0] empty, moves in both directions ------------------------------------------------------
def test_list_completed_moves(layout):
    rng = np.random.default_rng(73)
    es = [engine.GpuEngine(pool_name=f"md-lc{k}") for k in range(3)]
    lgs = [{} for _ in es]
    since = M.START
    try:
        for e, lg in zip(es, lgs):
            TLC.seed(e, lg, since, [])
        # job 1: older on a, latest on b; job 2: older on b, latest on a; job 3: equal stamps, b's later
        TLC.record(es[1], lgs[1], [(1, 5, 0, since + 10, 0, 0, CR.SUCCESS), (2, 9, 0, since + 20, 1, 0, CR.FAILED),
                                   (3, 4, 0, since + 30, -1, 1, CR.SUCCESS)])
        TLC.record(es[2], lgs[2], [(1, 7, 0, since + 10, 0, 0, CR.FAILED), (2, 3, 0, since + 20, 1, 0, CR.SUCCESS),
                                   (3, 4, 0, since + 30, -1, 1, CR.FAILED)])
        bulk = [[], []]
        for j in range(10, 3010):   # user 0's records past one sort tile, some of them moved
            k = int(rng.integers(0, 2))
            r = (j, int(rng.integers(1, 50)), int(rng.choice(3, p=[0.8, 0.1, 0.1])), since + int(rng.integers(0, 40_000)),
                 int(rng.integers(-1, 3)), int(rng.integers(-1, 2)), int(rng.choice([CR.SUCCESS, CR.FAILED, CR.REOPENED])))
            bulk[k].append(r)
            if rng.random() < 0.2:
                bulk[1 - k].append(r[:1] + (max(0, r[1] + int(rng.integers(-3, 4))),) + r[2:6] + (CR.SUCCESS,))
        for k in range(2):
            TLC.record(es[k + 1], lgs[k + 1], bulk[k])
        hp = [0, 1, 2]
        for idx in ([0, 1, 2], [2, 1, 0], [1, 2]):   # pools[0] empty; the handles reversed; two handles
            sub = [es[k] for k in idx]
            for s in TLC.STATES:
                for q in (L.query(0, 0, since, since + 50_000),
                          L.query(0, 0, since, since + 50_000, 2, 2000, 1, [hp[k] for k in idx], False, 700),
                          L.query(1, 0, since + 5000, since + 30_000)):
                    got, _ = TLC.ask(sub, q, s)
                    assert got == CR.list_completed([lgs[k] for k in idx], q, s), (idx, q, s)
            # each moved job is listed from the handle of its latest record, wherever that handle sits
            got, _ = TLC.ask(sub, L.query(0, 0, since, since + 50_000, 1, 3), CR.L_COMPLETED)
            assert [(j, p) for j, _, p in got] == [(1, idx.index(2)), (2, idx.index(1))]
    finally:
        for e in es:
            e.close()


# ---- the calls without a gather step --------------------------------------------------------------------------------
def test_other_multi_handle_calls_refuse_two_devices():
    if device_count() < 2:
        pytest.skip("one CUDA device visible: handles on two devices need two")
    es = [engine.GpuEngine(pool_name="md-one", device=1), engine.GpuEngine(pool_name="md-two", device=0)]
    try:
        for call in (lambda: engine.state_user_usage(es),
                     lambda: engine.state_list_jobs(es, 0, abi.LJ_WAITING, 0, 1),
                     lambda: engine.state_sweep(es, M.START, 1000, 2000)):
            with pytest.raises(CookError) as ei:
                call()
            assert ei.value.code == abi.COOK_E_BADARG and "handles on different devices" in str(ei.value)
        for e in es:   # the four with a gather step take them
            e.state_completed_seed(M.START, [], [], [], [], [], [], [])
            e.state_history_seed(M.START, [], [], [], [], [], [], [], [])
        assert engine.state_instance_stats(es, M.START, abi.IS_RUNNING, 0, M.START)["stats"]["n_launches"] == 0
        assert len(engine.state_history_stats(es, abi.IS_SUCCESS, M.START, M.START + 1)["kind"]) == 0
        assert len(engine.state_list_completed(es, 0, abi.LC_COMPLETED, M.START, M.START + 1)["job_id"]) == 0
        assert engine.state_user_stats(es, abi.make_users(3))["users"]["total"] == 0
    finally:
        for e in es:
            e.close()
