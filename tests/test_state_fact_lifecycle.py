"""Every per-row fact a resident handle keeps outside its digest and export, through every call that parks, requeues,
frees or reuses its row (fact_model.FATE).

CPU: the table has a fate for every (fact, event) cell and the model reads every one of them, every state-changing entry point is an event or a declared
setter or reader, the model's retry decisions equal the golden transitions and retry_ref.decide, and hand-computed
sequences give the answers written here.

GPU (-m gpu): a twin of a handle and fact_model.Model, every reader compared bit for bit after every call:
cook_state_sweep (lingering, cancelled, stragglers), cook_state_instance_stats (running, unknown),
cook_state_history_stats (success, failed), cook_state_list_jobs (entries and missing), cook_state_export (novel list,
reserved_host, allowed, plugin_accept), cook_state_status outcomes and attempts, cook_state_retry_facts' BADARG on a
job not held, cook_state_match_metrics after a match round, the digest's row counts and cook_state_queue (the last
rank's queue without the jobs removed, replaced or launched since).  The digest's fingerprints and the whole export are
restated in test_state_audit.py; the facts here are outside both.  The matrix runs each exit event followed by each
entry event on a fresh handle whose freed slot is the only one the entering row can take; the reason fact is followed
through reason_code NULL; list facts sent while the job runs stay off its parked copy; and a seeded churn over three
handles interleaves every call past a pending-table doubling, a novel-arena compaction that keeps parked entries, and
a user of more than 2048 rows.
"""
import json
import os
import re
import struct
import time

import numpy as np
import pytest

import fact_model as F
import match_metrics_ref as MR
import resident_model as M
import retry_ref as RR
from cook_b200 import abi, engine, traces

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "cook_gpu.h")
GOLDEN = json.load(open(os.path.join(HERE, "golden", "retry_golden.json")))
REASONS = GOLDEN["reasons"]
CODE = {k: v["code"] for k, v in REASONS.items()}
REASON_OF = {v["code"]: v for v in REASONS.values()}
LIMIT = GOLDEN["mea_culpa_limit"]
START = M.START
NOW = START + 10 ** 7
MEA = CODE["mesos-executor-terminated"]     # mea culpa, the global limit
PLAIN = CODE["unknown"]
OUTCOME = {abi.JOB_COMPLETED: "completed", abi.JOB_RUNNING: "running", abi.JOB_WAITING: "waiting",
           abi.JOB_WAITING_UNRETAINED: "waiting_unretained", abi.JOB_NO_FACTS: "no_facts"}
G = 4
GROUPS = {g: dict(kind="quantile-deviation", quantile=0.5, multiplier=1.0, n_jobs=3) for g in range(G)}


# ---- CPU: the table ----------------------------------------------------------------------------------------------
def test_table_has_every_cell():
    missing = [(f, e) for f in F.FACTS for e in F.EVENTS if (f, e) not in F.FATE]
    assert not missing, f"cells without a fate: {missing}"
    lines = open(HEADER).read().split("\n")
    for f in F.FACTS:
        for e in F.EVENTS:
            fate, cite = F.FATE[(f, e)]
            assert fate in F.FATES, (f, e)
            m = re.fullmatch(r"cook_gpu\.h:(\d+)", cite)
            assert m and lines[int(m.group(1)) - 1].lstrip().startswith(("*", "/*")), (f, e, cite)
    assert set(F.FATE) == {(f, e) for f in F.FACTS for e in F.EVENTS}
    made = {e for evs in F.WRITERS.values() for e in evs}
    assert made == set(F.EVENTS), "every event is made by some call, and every call's events are events"
    assert set(F.EXITS).isdisjoint(F.ENTRIES)


def test_model_reads_every_cell():
    """A sequence that makes every event: the model reads every cell of the table on the way, so no cell is
    decoration."""
    F.CONSULTED.clear()
    m = F.Model(LIMIT, REASON_OF)
    m.hist.seed(0, [])
    m.apply(up=[(1, prow()), (2, prow()), (3, prow()), (4, prow()), (5, prow())])
    m.apply(up=[(1, prow())])                                     # pending_upsert_live
    m.apply(rm=[5])                                               # pending_rm
    m.retry_facts([1, 2, 3], [3, 1, 3], [0, 0, 0], [[], [], []])
    m.launch([1, 2, 3, 4], [10, 20, 30, 40], [START] * 4, [7] * 4)   # launch_park x3, launch_free, launch
    m.apply(run_up=[rrow(1, 11), rrow(9, 90)])                    # running_upsert
    m.apply(run_up=[rrow(1, 11)])                                 # running_upsert_live
    m.retry_facts([9], [3], [0], [[]])
    assert m.status([10], [0], [START + 1], [PLAIN]) == [("running", 1)]
    assert m.status([11], [0], [START + 1], [PLAIN]) == [("waiting", 2)]          # and requeue
    assert m.status([20], [0], [START + 1], [PLAIN]) == [("completed", 1)]
    assert m.status([90], [0], [START + 1], [PLAIN]) == [("waiting_unretained", 1)]
    assert m.status([40], [0], [START + 1], [PLAIN]) == [("no_facts", -1)]
    m.apply(up=[(3, prow())])                                     # pending_upsert_parked
    m.retry_facts([1], [3], [0], [[]])
    m.launch([1], [12], [START], [7])
    m.apply(run_rm=[12])                                          # running_rm
    m.retry_facts([1], [3], [abi.RF_COMPLETED], [[]])             # retry_facts_completed
    m.apply(up=[(6, prow()), (7, prow())])
    m.launch([6, 7], [60, 70], [START] * 2, [7] * 2)
    m.finish([60], [START + 1], [1])                              # finish
    m.finish([70], [START + 1], [1], history=True)                # finish_history
    m.apply(reset=True)                                           # reset
    assert F.CONSULTED == set(F.FATE), sorted(set(F.FATE) - F.CONSULTED)


def test_every_state_call_is_declared():
    calls = {n for n in abi.ARGTYPES if n.startswith("cook_state_")}
    declared = set(F.WRITERS) | set(F.SETTERS) | set(F.READERS)
    assert calls - declared == set(), "a new cook_state_* call must say which events it makes, or that it only reads"
    assert declared - calls == set()
    assert set(F.WRITERS).isdisjoint(F.SETTERS) and set(F.READERS).isdisjoint(set(F.WRITERS) | set(F.SETTERS))
    for facts in F.SETTERS.values():
        assert set(facts) <= set(F.FACTS)


# ---- CPU: the model's decisions --------------------------------------------------------------------------------
def prow(user=0, cpus=1.0, mem=1024.0, novel=(), groups=(1,), **kw):
    return dict(M.DEFAULTS, user=user, priority=50, cpus=cpus, mem=mem, novel=list(novel), attr=[],
                groups=list(groups), **kw)


def rrow(jid, tid, user=0, host=7, start=START, groups=(1,)):
    return dict(user=user, priority=50, start_time=start, task_id=tid, job_id=jid, cpus=1.0, mem=1024.0, gpus=0.0,
                host=host, groups=list(groups))


def _replayable(case):
    ups = [(k, st, r) for k, (st, r) in enumerate(case["updates"]) if st is not None]
    return len(ups) == 1 and ups[0][1] in RR.DONE and case["instances"][ups[0][0]][0] in ("running", "unknown")


@pytest.mark.parametrize("case", [c for c in GOLDEN["transitions"] if _replayable(c)], ids=lambda c: c["name"])
def test_model_golden_transition(case):
    (k, st, r), = [(k, st, r) for k, (st, r) in enumerate(case["updates"]) if st is not None]
    m = F.Model(LIMIT, REASON_OF)
    m.apply(up=[(1, prow())])
    others = [j for j in range(len(case["instances"])) if j != k]
    live = [j for j in others if case["instances"][j][0] in ("running", "unknown")]
    m.apply(run_up=[rrow(1, 100 + j) for j in live])
    done = [CODE[rr] if rr else -1 for s, rr in (case["instances"][j] for j in others) if s in RR.DONE]
    flags = (abi.RF_DISABLE_MEA_CULPA if case["disable"] else 0) | (
        abi.RF_COMPLETED if case["old_job_state"] == "completed" else 0)
    m.retry_facts([1], [case["retry_count"]], [flags], [done])
    want = RR.decide(dict(max_retries=case["retry_count"], disable=case["disable"],
                          completed=case["old_job_state"] == "completed", done=done), REASON_OF, st == "success",
                     CODE[r], bool(live), LIMIT)
    m.launch([1], [1], [START], [7])
    m.task_reason([1], [CODE[r]])
    (name, att), = m.status([1], [st == "success"], [START + 1000])    # reason_code NULL: the fact
    assert (name.replace("_unretained", ""), att) == (case["new_job_state"], want[1]) == want[:2]
    assert (1 in m.pend) == (case["new_job_state"] == "waiting")


@pytest.mark.parametrize("case", GOLDEN["batch"], ids=lambda c: c["name"])
def test_model_golden_batch(case):
    m = F.Model(LIMIT, REASON_OF)
    m.apply(up=[(1, prow())])
    m.retry_facts([1], [case["retry_count"]], [0], [[]])
    m.launch([1], [10], [START], [3])
    m.apply(run_up=[rrow(1, 11, host=4)])
    out = m.status([10 + k for k, _, _ in case["order"]], [s == "success" for _, s, _ in case["order"]],
                   [START + 5] * 2, [CODE[r] for _, _, r in case["order"]])
    assert [n for n, _ in out] == case["outcomes"] and [a for _, a in out] == case["attempts"]


def test_model_hand_sequences():
    # a mea-culpa reason fact read through reason_code NULL requeues; the history row carries the same code
    m = F.Model(LIMIT, REASON_OF)
    m.hist.seed(0, [])
    m.apply(up=[(5, prow(novel=[2], reserved_host=9, allowed=0))])
    m.job_facts([5], [dict(facts=abi.JF_GPUS, gpu_model=3)])
    m.list_facts([5], [START - 5], [2], [0])
    m.retry_facts([5], [1], [0], [[]])
    m.launch([5], [50], [START], [8])
    assert m.run[50]["lf"] == (START - 5, 2, 0) and m.parked[5]["jf"] == dict(facts=abi.JF_GPUS, gpu_model=3)
    m.task_reason([50], [MEA])
    assert m.status([50], [0], [START + 10]) == [("waiting", 0)]
    assert m.pend[5]["jf"] is None and m.pend[5]["lf"] == (START - 5, 2, 0)
    assert m.export_rows()[5] == ([2, 8], -1, 0, 1)
    assert m.hist.rows[-1]["reason"] == MEA and 5 in m.retry
    # the same failure without the fact completes (one plain attempt of one) and frees the copy
    m.launch([5], [51], [START + 20], [8])
    assert m.status([51], [0], [START + 30]) == [("completed", 1)]
    assert m.hist.rows[-1]["reason"] == -1 and not m.holds(5) and 5 not in m.retry
    # list facts sent while the job runs reach the running row only: the requeued row has none
    m.apply(up=[(6, prow())])
    m.retry_facts([6], [3], [0], [[]])
    m.launch([6], [60], [START], [1])
    m.list_facts([6], [START], [-1], [1])
    assert m.status([60], [0], [START + 1], [PLAIN]) == [("waiting", 1)]
    got = F.list_answer([m], 0, abi.LJ_WAITING | abi.LJ_RUNNING, 0, 1 << 62)
    assert got == ([], 1)
    # a success appends one record per group; a reset drops them and every fact
    m.launch([6], [61], [START + 2000], [1])
    m.finish([61], [START + 9500], [1])
    assert m.records == [(1, 7)] and 6 not in m.retry
    m.apply(reset=True)
    assert (m.records, m.pend, m.parked, m.retry, m.hist.on) == ([], {}, {}, {}, False)


# ---- GPU: the twin ---------------------------------------------------------------------------------------------
def bits(x):
    return struct.unpack("<q", struct.pack("<d", float(x)))[0]


def _is_eq(got, want):
    segs, lc, lm = want
    assert len(got["kind"]) == len(segs)
    for d, w in enumerate(segs):
        assert (int(got["kind"][d]), int(got["user"][d]), int(got["reason"][d]), int(got["count"][d])) == w[:4], d
        assert [bits(x) for x in got["total"][d]] == [bits(x) for x in w[4]], d
        assert [[bits(x) for x in p] for p in got["pct"][d]] == [[bits(x) for x in p] for p in w[5]], d
    for g, w in ((got["leaders_cpu"], lc), (got["leaders_mem"], lm)):
        assert [(u, bits(t)) for u, t in g] == [(u, bits(t)) for u, t in w]


def _sweep_cols():
    return {"kind": np.full(G, abi.SWEEP_QUANTILE_DEVIATION, np.int32), "quantile": np.full(G, 0.5),
            "multiplier": np.full(G, 1.0), "n_jobs": np.full(G, 3, np.int32)}


class Twin:
    """Handles and their models, fed the same calls; `check` compares every reader."""

    def __init__(self, n=1, users=2):
        self.e = [engine.GpuEngine(pool_name=f"facts{k}") for k in range(n)]
        self.m = [F.Model(LIMIT, REASON_OF) for _ in range(n)]
        self.n_users = users
        for e, m in zip(self.e, self.m):
            e.state_retry_config(LIMIT, [(v["code"], v["mea_culpa"], -2 if v["failure_limit"] is None
                                          else v["failure_limit"]) for v in REASONS.values()])
            e.state_history_seed(0)
            m.hist.seed(0, [])
        self.checks = 0
        self.queue = [None] * n          # the last rank's queue, None before a rank or after a reset
        self.gone = [set() for _ in range(n)]   # the jobs removed, replaced or launched since

    def close(self):
        for e in self.e:
            e.close()

    # -- calls -----------------------------------------------------------------------------------------------------
    def apply(self, k=0, up=(), rm=(), run_up=(), run_rm=(), reset=False):
        up, run_up = list(up), list(run_up)
        self.e[k].state_apply(M.delta(reset, up, rm, run_up, run_rm, hosts=True, lists=True))
        self.m[k].apply(up, rm, run_up, run_rm, reset)
        self.gone[k] |= set(rm) | {j for j, _ in up}
        if reset:
            self.queue[k] = None
            self.e[k].state_history_seed(0)
            self.m[k].hist.seed(0, [])

    def launch(self, k, jobs, tids, starts, hosts):
        self.e[k].state_launch(jobs, tids, starts, hosts)
        self.m[k].launch(jobs, tids, starts, hosts)
        self.gone[k] |= set(jobs)

    def patch(self, k, jobs, **cols):
        self.e[k].state_patch(jobs, **cols)
        self.m[k].patch(jobs, **cols)

    def task_facts(self, k, tids, **cols):
        self.e[k].state_task_facts(tids, **cols)
        self.m[k].task_facts(tids, cols.get("max_runtime_ms"), cols.get("cancelled"), cols.get("unknown"))

    def task_reason(self, k, tids, codes):
        self.e[k].state_task_reason(tids, codes)
        self.m[k].task_reason(tids, codes)

    def job_facts(self, k, jobs, facts):
        col = lambda c, dt: np.array([f.get(c, 0) for f in facts], dt)
        self.e[k].state_job_facts(jobs, col("facts", np.uint8), col("gpu_model", np.int32),
                                  col("disk_request", np.float64), col("disk_limit", np.float64),
                                  col("disk_type", np.int32))
        self.m[k].job_facts(jobs, facts)

    def list_facts(self, k, jobs, submit, pool, executor):
        self.e[k].state_list_facts(jobs, submit, pool, executor)
        self.m[k].list_facts(jobs, submit, pool, executor)

    def retry_facts(self, k, jobs, max_retries, flags, done):
        self.e[k].state_retry_facts(jobs, max_retries, flags, done)
        self.m[k].retry_facts(jobs, max_retries, flags, done)

    def status(self, k, tids, ok, end, reason=None, pre=None):
        oc, att = self.e[k].state_status(tids, ok, end, reason, pre)
        want = self.m[k].status(tids, ok, end, reason, pre)
        assert [(OUTCOME[int(o)], int(a)) for o, a in zip(oc, att)] == want
        return want

    def finish(self, k, tids, end, ok, history=False, reason=None):
        if history:
            self.e[k].state_finish_history(tids, end, ok, reason)
        else:
            self.e[k].state_finish(tids, end, ok)
        self.m[k].finish(tids, end, ok, history, reason)

    def advance(self, k, since):
        self.e[k].state_history_advance(since)
        self.m[k].hist.advance(since)

    def runtimes(self, k, add=(), forget=()):
        self.e[k].state_group_runtimes([g for g, _ in add], [s for _, s in add], forget)
        self.m[k].group_runtimes(add, forget)

    # -- readers ---------------------------------------------------------------------------------------------------
    def check(self, probe=()):
        self.checks += 1
        sw = engine.state_sweep(self.e, NOW, 10 ** 6, 5 * 10 ** 6, groups=_sweep_cols())
        want = F.sweep_answer(self.m, NOW, 10 ** 6, 5 * 10 ** 6, GROUPS)
        assert (sw["linger"], sw["cancel"], sw["straggler"]) == want, "sweep"
        for st, code in (("running", abi.IS_RUNNING), ("unknown", abi.IS_UNKNOWN)):
            _is_eq(engine.state_instance_stats(self.e, NOW, code, 0, NOW + 1), F.instance_answer(self.m, NOW, st, 0, NOW + 1))
        since = max(m.hist.since for m in self.m)   # no window before a horizon
        for st, code in (("success", abi.IS_SUCCESS), ("failed", abi.IS_FAILED)):
            _is_eq(engine.state_history_stats(self.e, code, since, NOW + 1), F.history_answer(self.m, st, since, NOW + 1))
        for u in range(self.n_users):
            got = engine.state_list_jobs(self.e, u, abi.LJ_WAITING | abi.LJ_RUNNING, 0, 1 << 62)
            want, missing = F.list_answer(self.m, u, abi.LJ_WAITING | abi.LJ_RUNNING, 0, 1 << 62)
            assert list(zip(got["state"].tolist(), got["job_id"].tolist(), got["submit_ms"].tolist(),
                            got["pool"].tolist())) == want, ("list", u)
            assert got["missing"] == missing, ("missing", u)
        for k, (e, m) in enumerate(zip(self.e, self.m)):
            d = e.state_digest()
            assert d["consistent"] and (d["pending"][2], d["running"][2]) == (len(m.pend), len(m.run)), "digest"
            if self.queue[k] is not None:   # parked and requeued jobs are off the queue until the next rank
                assert e.state_queue().tolist() == [j for j in self.queue[k] if j not in self.gone[k]], "queue"
            x = e.state_export()
            off, nh = x["pending"].col("novel_off"), x["pending"].col("novel_host")
            got = {j: (nh[off[i]:off[i + 1]].tolist(), int(x["pending"].col("reserved_host")[i]),
                       int(x["pending"].col("allowed")[i]), int(x["pending"].col("plugin_accept")[i]))
                   for i, j in enumerate(x["pending_job_id"].tolist())}
            assert got == m.export_rows(), "export"
            for j in probe:   # held with facts: the same facts again change nothing; not held: BADARG
                f = m.retry.get(j)
                if m.holds(j) and f is not None:
                    e.state_retry_facts([j], [f["max_retries"]], [(1 if f["disable"] else 0) | (2 if f["completed"] else 0)],
                                        [f["done"]])
                elif not m.holds(j):
                    with pytest.raises(engine.CookError) as ei:
                        e.state_retry_facts([j], [1], [0], [[]])
                    assert ei.value.code == abi.COOK_E_BADARG

    def metrics(self, k, offers, users, params):
        """A match round on handle k, then cook_state_match_metrics against match_metrics_ref on the model's facts."""
        e, m = self.e[k], self.m[k]
        self.queue[k], self.gone[k] = e.state_rank(users).tolist(), set()
        got_m = e.state_match(offers, users, params)
        ids = [int(j) for j in got_m["considerable"]]
        got = e.state_match_metrics(users.n_users)
        jobs = [m.metrics_job(j) for j in ids]
        matched = [i for i, a in enumerate(got_m["assign"].tolist()) if a >= 0]
        want = MR.answer(jobs, matched, m.mm_prev, 500, users.n_users)
        m.mm_prev = want["cycles"]
        for key in ("considerable", "matched", "head_job_id", "uris", "too_long"):
            assert got[key] == want[key], key
        assert got["user_considerable"].tolist() == want["user_considerable"]
        if ids:
            assert got["keys"] == want["keys"]
            for row in got["rows"]:
                j = jobs[row["position"]]
                assert row["facts"] == j["facts"], (row["job_id"], row["facts"], j)
                assert row["gpu_model"] == (j["gpu_model"] if j["facts"] & abi.JF_GPUS else -1)
                assert row["disk_type"] == (j["disk_type"] if j["facts"] & abi.JF_DISK else -1)
        return ids


def offers_of(n, cpus=64.0):
    return abi.OffersSoA(n=n, hostname_id=np.arange(n, dtype=np.int32), name_rank=np.arange(n, dtype=np.int32),
                         cpus=np.full(n, cpus), mem=np.full(n, 10.0 ** 6), run_cpus=np.zeros(n), run_mem=np.zeros(n),
                         run_count=np.zeros(n, np.int32), n_attr_cols=0, attr=np.zeros(0, np.int32))


# ---- GPU: the matrix -------------------------------------------------------------------------------------------
J, T = 10, 100            # the row that leaves
J2, T2 = 20, 200          # the row that enters
FACTS_JF = dict(facts=abi.JF_GPUS | abi.JF_DISK | abi.JF_DISK_REQUEST, gpu_model=2, disk_type=1, disk_request=512.0)


def _give_pending(tw):
    """Distinctive pending facts on job J: job facts, list facts, allowed 0, plugin_accept 0, a reservation."""
    tw.job_facts(0, [J], [FACTS_JF])
    tw.list_facts(0, [J], [START - 7], [3], [1])
    tw.patch(0, [J], allowed=[0], plugin_accept=[0], reserved_host=[4])


def _give_running(tw, tid=T):
    """Distinctive running facts on task tid: max-runtime, cancelled, unknown and a mea-culpa reason."""
    tw.task_facts(0, [tid], max_runtime_ms=[1000], cancelled=[1], unknown=[1])
    tw.task_reason(0, [tid], [MEA])


def _launched(tw, retry, max_retries=3):
    """Job J pending with every pending fact, retry facts when `retry`, launched as task T; the running facts on T."""
    tw.apply(up=[(J, prow(novel=[5]))])
    _give_pending(tw)
    if retry:
        tw.retry_facts(0, [J], [max_retries], [0], [[]])
    tw.launch(0, [J], [T], [START], [6])
    _give_running(tw)


def _exit(tw, ev):
    """Set job J / task T up for the exit event and run it."""
    if ev in ("pending_rm", "pending_upsert_live", "launch_free", "launch_park", "reset"):
        tw.apply(up=[(J, prow(novel=[5]))])
        _give_pending(tw)
        if ev == "launch_park":
            tw.retry_facts(0, [J], [3], [0], [[]])
        tw.check([J])
        if ev == "pending_rm":
            tw.apply(rm=[J])
        elif ev == "pending_upsert_live":
            tw.apply(up=[(J, prow(novel=[5]))])
        elif ev == "reset":
            tw.apply(reset=True)
        else:
            tw.launch(0, [J], [T], [START], [6])
            _give_running(tw)
        return
    if ev in ("running_rm", "running_upsert_live"):
        _launched(tw, False)
        tw.check([J])
        tw.apply(run_rm=[T]) if ev == "running_rm" else tw.apply(run_up=[rrow(J, T)])
        return
    if ev == "status_waiting_unretained":
        tw.apply(run_up=[rrow(J, T)])
        _give_running(tw)
        tw.retry_facts(0, [J], [3], [0], [[]])
        tw.check([J])
        assert tw.status(0, [T], [0], [START + 10]) == [("waiting_unretained", 0)]
        return
    _launched(tw, ev != "status_no_facts", max_retries=1 if ev == "status_completed" else 3)
    if ev == "status_running":
        tw.apply(run_up=[rrow(J, T + 1)])
    tw.check([J])
    if ev in ("finish", "finish_history"):
        tw.finish(0, [T], [START + 4000], [1], history=ev == "finish_history")
    elif ev == "pending_upsert_parked":
        tw.apply(up=[(J, prow(novel=[5]))])
    elif ev == "retry_facts_completed":
        tw.apply(run_rm=[T])
        tw.check([J])
        tw.retry_facts(0, [J], [3], [abi.RF_COMPLETED], [[]])
    else:
        name = ev[len("status_"):]
        got = tw.status(0, [T], [0], [START + 10], None if ev != "status_completed" else [PLAIN])
        assert got[0][0] == name


def _entry(tw, ev):
    """A new row in, on the slot the exit freed (the only free one)."""
    if ev == "pending_upsert":
        tw.apply(up=[(J2, prow(novel=[1]))])
    elif ev == "running_upsert":
        tw.apply(run_up=[rrow(J2, T2, start=START + 1)])
    elif ev == "launch":
        tw.apply(up=[(J2, prow())])
        tw.launch(0, [J2], [T2], [START + 1], [2])
    elif ev == "requeue":   # the requeued row runs again and fails again: its facts as after the first requeue
        tw.launch(0, [J], [T2], [START + 20], [6])
        tw.check([J])
        tw.status(0, [T2], [0], [START + 30], [PLAIN], [1])


MATRIX = [(x, n) for x in F.EXITS for n in F.ENTRIES if (n == "requeue") == (x == "status_waiting")]


def _cells(x, n):
    return [f for f in F.FACTS if F.fate(f, x) != F.NONE or F.fate(f, n) != F.NONE]


@pytest.mark.gpu
@pytest.mark.parametrize("exit_ev,entry_ev", MATRIX, ids=lambda v: v)
def test_matrix(exit_ev, entry_ev):
    tw = Twin()
    try:
        _exit(tw, exit_ev)
        tw.check([J])
        _entry(tw, entry_ev)
        tw.check([J, J2])
        # a match round over what the exit and the entry left, before anything else writes a job fact: the requeued
        # row's cleared facts, the entering row's on a reused slot.  Patched allowed and plugin-accepted first (their
        # keeping through the requeue was checked above), so that every live row is considerable.
        m = tw.m[0]
        live = sorted(m.pend)
        if live:
            tw.patch(0, live, allowed=[1] * len(live), plugin_accept=[1] * len(live))
        considered = tw.metrics(0, offers_of(4), abi.make_users(2), traces.match_params(16))
        assert sorted(considered) == live
        tw.check([J, J2])
        # the entering row's facts are the absent ones until sent; sent now, the readers follow
        if J2 in m.pend:
            tw.job_facts(0, [J2], [dict(facts=abi.JF_DISK, disk_type=3)])
            tw.list_facts(0, [J2], [START], [-1], [0])
        if T2 in m.run:
            tw.task_reason(0, [T2], [PLAIN])
            tw.finish(0, [T2], [START + 5000], [1], history=True)
        tw.check([J, J2])
        tw.metrics(0, offers_of(4), abi.make_users(2), traces.match_params(16))
        tw.check([J, J2])
        print(f"[matrix] {exit_ev} -> {entry_ev}: {len(_cells(exit_ev, entry_ev))} (fact, exit, entry) cells")
    finally:
        tw.close()


def test_matrix_covers_every_cell():
    """Every (fact, exit, entry) triple with a fate other than none on either side runs in some matrix case."""
    covered = {(f, x, n) for x, n in MATRIX for f in _cells(x, n)}
    for f in F.FACTS:
        for x in F.EXITS:
            if F.fate(f, x) != F.NONE:
                assert any((f, x, n) in covered for n in F.ENTRIES), (f, x)
        for n in F.ENTRIES:
            if F.fate(f, n) != F.NONE:
                assert any((f, x, n) in covered for x in F.EXITS), (f, n)


# ---- GPU: the reason fact through reason_code NULL ---------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("how", ["fresh", "running_upsert", "launch_into_slot"])
def test_reason_null(how):
    """A mea-culpa reason fact, read through reason_code NULL, requeues a job of one retry that would otherwise
    complete; the history row carries the same code through cook_state_status and cook_state_finish_history.  After a
    running upsert of the same task id (the fact back to -1) the failure completes the job; a launch into the slot the
    reasoned row left starts without it."""
    tw = Twin()
    try:
        tw.apply(up=[(J, prow()), (J2, prow(user=1))])
        tw.retry_facts(0, [J, J2], [1, 1], [0, 0], [[], []])
        tw.launch(0, [J], [T], [START], [6])
        tw.task_reason(0, [T], [MEA])
        if how == "running_upsert":
            tw.apply(run_up=[rrow(J, T, host=6)])
        elif how == "launch_into_slot":
            tw.finish(0, [T], [START + 1], [0], history=True)      # reason NULL: the history row takes MEA
            assert tw.m[0].hist.rows[-1]["reason"] == MEA and not tw.m[0].holds(J)
            tw.check([J])
            tw.launch(0, [J2], [T2], [START + 2], [6])              # the freed running slot, reasoned before
        tid, jid = (T2, J2) if how == "launch_into_slot" else (T, J)
        tw.check([jid])
        want = ("waiting", 0) if how == "fresh" else ("completed", 1)
        assert tw.status(0, [tid], [0], [START + 10]) == [want]
        assert tw.m[0].hist.rows[-1]["reason"] == (MEA if how == "fresh" else -1)
        tw.check([J, J2])
    finally:
        tw.close()


# ---- GPU: list facts sent while the job runs ---------------------------------------------------------------------
@pytest.mark.gpu
def test_list_facts_while_running():
    tw = Twin()
    try:
        tw.apply(up=[(J, prow())])
        tw.retry_facts(0, [J], [3], [0], [[]])
        tw.launch(0, [J], [T], [START], [6])
        tw.list_facts(0, [J], [START - 1], [-1], [0])
        tw.check([J])
        assert tw.status(0, [T], [0], [START + 10], [PLAIN]) == [("waiting", 1)]
        got = engine.state_list_jobs(tw.e, 0, abi.LJ_WAITING | abi.LJ_RUNNING, 0, 1 << 62)
        assert got["job_id"].tolist() == [] and got["missing"] == 1
        tw.check([J])
    finally:
        tw.close()


# ---- GPU: the interleaved churn ----------------------------------------------------------------------------------
class Arena:
    """The pending novel-host arena's sizes as cook_state_apply, _launch and _status leave them: its tail, and the
    entries of live and parked rows; a compaction when the dead entries pass the kept ones."""

    def __init__(self):
        self.tail, self.compactions_parked = 0, 0

    def after(self, m, appended):
        self.tail += appended
        kept = sum(len(r["novel"]) for r in m.pend.values()) + sum(len(r["novel"]) for r in m.parked.values())
        if self.tail - kept > kept:
            self.compactions_parked += bool(m.parked) and kept > 0
            self.tail = kept


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_churn(seed):
    rng = np.random.default_rng(seed)
    U = 3
    tw = Twin(n=3, users=U)
    arenas = [Arena() for _ in range(3)]
    users, offers, params = abi.make_users(U), offers_of(64), traces.match_params(256)
    nid = [1000]
    hw = [0, 0, 0]
    big_user = [0]
    t0 = time.time()

    def ids(n):
        nid[0] += 2 * n
        return list(range(nid[0] - 2 * n, nid[0], 2))

    def amounts(n):
        grid = rng.random() < 0.5
        cpus = rng.choice([0.5, 1.0, 2.0] if grid else [0.1, 0.3, 0.7], n)
        mem = 512.0 * rng.integers(1, 9, n) if grid else rng.integers(1, 4000, n) / 7.0
        return cpus.tolist(), mem.tolist()

    def new_rows(n, user=None):
        cpus, mem = amounts(n)
        return [(j, prow(user=int(rng.integers(0, U)) if user is None else user, cpus=c, mem=me,
                         novel=rng.choice(40, int(rng.integers(0, 4)), replace=False).tolist(),
                         groups=[int(rng.integers(0, G))] if rng.random() < 0.7 else []))
                for j, c, me in zip(ids(n), cpus, mem)]

    try:
        for step in range(70):
            k = int(rng.integers(0, 3))
            m = tw.m[k]
            appended = 0
            op = rng.choice(["up", "rm", "run_up", "run_rm", "launch", "patch", "task_facts", "task_reason",
                             "job_facts", "list_facts", "retry_facts", "status", "finish", "finish_history",
                             "advance", "runtimes", "reset"],
                            p=[.12, .05, .05, .04, .12, .04, .05, .05, .06, .06, .08, .12, .04, .04, .02, .03, .03])
            if step < 3 or (step == 20 and k == 0):   # the pending table past 1024 slots, one user past 2048 rows
                k, m = 0, tw.m[0]
                rows = new_rows(1100, user=0)
                tw.apply(0, up=rows)
                appended = sum(len(r["novel"]) for _, r in rows)
                op = "bulk"
            pend, run = sorted(m.pend), sorted(m.run)
            if step == 30:   # park 300 jobs of handle 0, then kill most others: the arena compacts around them
                k, m = 0, tw.m[0]
                pend = sorted(m.pend)
                assert len(pend) > 400
                jobs = [j for j in pend if m.pend[j]["novel"]][:300]
                tw.retry_facts(0, jobs, [3] * len(jobs), [0] * len(jobs), [[] for _ in jobs])
                tw.launch(0, jobs, ids(len(jobs)), [START] * len(jobs), rng.integers(-1, 30, len(jobs)).tolist())
                arenas[0].after(m, 0)
                rest = sorted(m.pend)
                tw.apply(0, rm=rest[:len(rest) - 50])
                op = "drill"
            if op == "up":
                rows = new_rows(int(rng.integers(1, 60)))
                if pend and rng.random() < 0.5:   # some ids live already, some parked
                    rows += [(j, prow(user=m.pend[j]["user"], novel=[int(rng.integers(0, 40))]))
                             for j in rng.choice(pend, min(5, len(pend)), replace=False).tolist()]
                rows += [(j, prow(user=r["user"])) for j, r in list(m.parked.items())[:2]]
                tw.apply(k, up=rows)
                appended = sum(len(r["novel"]) for _, r in rows)
            elif op == "rm" and pend:
                tw.apply(k, rm=rng.choice(pend, min(20, len(pend)), replace=False).tolist())
            elif op == "run_up":
                jobs = rng.choice(pend, min(5, len(pend)), replace=False).tolist() if pend and rng.random() < 0.5 else ids(5)
                rows = [rrow(int(j), t, user=int(rng.integers(0, U)), host=int(rng.integers(-1, 30)),
                             start=START + int(rng.integers(0, 10 ** 6)), groups=[int(rng.integers(0, G))])
                        for j, t in zip(jobs, ids(len(jobs)))]
                if run and rng.random() < 0.5:   # an upsert of a live task id: its facts reset
                    r = m.run[run[0]]
                    rows.append(rrow(r["job_id"], run[0], r["user"], r["host"], r["start_time"], r["groups"]))
                tw.apply(k, run_up=rows)
            elif op == "run_rm" and run:
                tw.apply(k, run_rm=rng.choice(run, min(10, len(run)), replace=False).tolist())
            elif op == "launch" and pend:
                jobs = rng.choice(pend, min(int(rng.integers(1, 300)), len(pend)), replace=False).tolist()
                tw.launch(k, jobs, ids(len(jobs)), (START + rng.integers(0, 10 ** 6, len(jobs))).tolist(),
                          rng.integers(-1, 30, len(jobs)).tolist())
            elif op == "patch" and pend:
                jobs = rng.choice(pend, min(30, len(pend)), replace=False).tolist()
                tw.patch(k, jobs, allowed=rng.integers(0, 2, len(jobs)).tolist(),
                         plugin_accept=rng.integers(0, 2, len(jobs)).tolist(),
                         reserved_host=rng.integers(-1, 30, len(jobs)).tolist())
            elif op == "task_facts" and run:
                t = rng.choice(run, min(40, len(run)), replace=False).tolist()
                tw.task_facts(k, t, max_runtime_ms=rng.choice([-1, 10 ** 5, 3 * 10 ** 6], len(t)).tolist(),
                              cancelled=rng.integers(0, 2, len(t)).tolist(), unknown=(rng.random(len(t)) < 0.3).tolist())
            elif op == "task_reason" and run:
                t = rng.choice(run, min(40, len(run)), replace=False).tolist()
                tw.task_reason(k, t, rng.choice([-1, MEA, PLAIN, CODE["preempted-by-rebalancer"]], len(t)).tolist())
            elif op == "job_facts" and pend:
                jobs = rng.choice(pend, min(200, len(pend)), replace=False).tolist()
                tw.job_facts(k, jobs, [dict(facts=int(rng.choice([0, 1, 2, 6, 15])), gpu_model=int(rng.integers(-1, 3)),
                                            disk_type=int(rng.integers(-1, 2)), disk_request=float(rng.choice([256.0, 0.3])),
                                            disk_limit=2048.0) for _ in jobs])
            elif op == "list_facts":
                held = sorted(set(pend) | {r["job_id"] for r in m.run.values()})
                if held:
                    jobs = rng.choice(held, min(200, len(held)), replace=False).tolist()
                    tw.list_facts(k, jobs, (START - rng.integers(0, 10 ** 6, len(jobs))).tolist(),
                                  rng.integers(-1, 3, len(jobs)).tolist(), rng.integers(-1, 2, len(jobs)).tolist())
            elif op == "retry_facts":
                held = sorted(set(pend) | set(m.parked) | {r["job_id"] for r in m.run.values()})
                if held:
                    jobs = rng.choice(held, min(400, len(held)), replace=False).tolist()
                    tw.retry_facts(k, jobs, rng.integers(1, 4, len(jobs)).tolist(),
                                   [int(rng.random() < 0.15) | (2 * int(rng.random() < 0.05)) for _ in jobs],
                                   [rng.choice([-1, MEA, PLAIN], int(rng.integers(0, 3))).tolist() for _ in jobs])
            elif op in ("status", "finish", "finish_history") and run:
                t = rng.choice(run, min(int(rng.integers(1, 200)), len(run)), replace=False).tolist()
                end = [m.run[x]["start_time"] + int(rng.integers(0, 10 ** 6)) for x in t]
                ok = (rng.random(len(t)) < 0.3).astype(int).tolist()
                reason = None if rng.random() < 0.5 else rng.choice([-1, MEA, PLAIN], len(t)).tolist()
                if op == "status":
                    before = {j: len(r["novel"]) for j, r in m.parked.items()}
                    tw.status(k, t, ok, end, reason, (rng.random(len(t)) < 0.2).astype(int).tolist())
                    appended = sum(len(m.pend[j]["novel"]) for j, n in before.items()
                                   if j in m.pend and len(m.pend[j]["novel"]) != n)
                else:
                    tw.finish(k, t, end, ok, history=op == "finish_history", reason=reason)
            elif op == "advance" and m.hist.on:
                tw.advance(k, max(m.hist.since, START) + 100_000)
            elif op == "runtimes":
                tw.runtimes(k, add=[(int(rng.integers(0, G)), int(rng.integers(0, 2000))) for _ in range(3)],
                            forget=[int(rng.integers(0, G))] if rng.random() < 0.3 else [])
            elif op == "reset" and step > 40 and rng.random() < 0.3:
                tw.apply(k, reset=True)
            arenas[k].after(m, appended)
            hw[k] = max(hw[k], len(m.pend) + len(m.parked))
            big_user[0] = max(big_user[0], sum(1 for r in m.pend.values() if r["user"] == 0))
            tw.check(probe=(1000 + 2 * rng.integers(0, (nid[0] - 1000) // 2, 6)).tolist())
            if step % 5 == 4:
                tw.metrics(k, offers, users, params)
        assert max(hw) > 1024, "the pending table passed 1024 slots"
        assert sum(a.compactions_parked for a in arenas) > 0, "a novel-arena compaction with parked entries kept"
        assert big_user[0] > 2048, "one user past a 2048-wide sort tile"
        print(f"[churn {seed}] {tw.checks} checks, pending high water {hw}, "
              f"compactions with parked entries {[a.compactions_parked for a in arenas]}, "
              f"{time.time() - t0:.1f} s")
    finally:
        tw.close()
