"""One plain model of the per-row facts a resident handle keeps outside cook_state_digest and cook_state_export, and of
what every call that writes a slot does to each of them (include/cook_gpu.h).

`FATE[(fact, event)]` is the header's rule for one fact under one event, transcribed as (fate, header line):
  reset  the row the event leaves (or brings in) holds the fact's absent value
  keep   the row, or the job's parked copy, keeps the value it had
  copy   the value moves to the row (or history row, or record) the event makes
  drop   the value leaves with the row
  none   the event does not concern the fact
Exit events take a row out (their fate says what becomes of the leaving row's fact); entry events put a row in (their
fate says what the entering row holds).  Every cell is written out: the table has no default, so a cell left out is
missing, not silently `none`.  `Model` reads every cell of an event as the event happens (`CONSULTED` records them).
The cells that choose a value (what an entering, upserted or requeued row holds; whether a parked copy and retry
facts go) steer it.  For the facts of a row the event deletes, it refuses a cell that would keep them.  It projects
its rows onto the inputs of the existing restatements (sweep_ref, instance_stats_ref, history_ref, list_ref,
match_metrics_ref, retry_ref).

A pending row is a resident_model row (JOB_COLS, user, priority, novel, attr, groups) plus jf (None, or the job facts
as match_metrics_ref reads them) and lf (None, or (submit ms, submit pool, custom executor)).  A running row is a
resident_model running row plus max_runtime, cancelled, unknown, reason and lf.
"""
import history_ref as HR
import instance_stats_ref as IR
import list_ref as LR
import retry_ref as RR
import sweep_ref as SR

RESET, KEEP, COPY, DROP, NONE = "reset", "keep", "copy", "drop", "none"
FATES = (RESET, KEEP, COPY, DROP, NONE)

FACTS = ("max_runtime", "cancelled", "unknown", "reason", "job_facts", "list_facts", "retry_facts", "parked_copy",
         "allowed", "reserved_host", "records")
EXITS = ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "launch_free", "launch_park", "running_rm",
         "running_upsert_live", "finish", "finish_history", "status_completed", "status_running", "status_waiting",
         "status_waiting_unretained", "status_no_facts", "retry_facts_completed", "reset")
ENTRIES = ("pending_upsert", "running_upsert", "launch", "requeue")
EVENTS = EXITS + ENTRIES

_STATUS_EXITS = ("status_completed", "status_running", "status_waiting", "status_waiting_unretained", "status_no_facts")


def _cells(*groups):
    """One fact's row of the table from (fate, header line, events) groups.  There is no default: an event no group
    names is missing from the table, and an event two groups name is refused."""
    out = {}
    for fate_, line, events in groups:
        for e in events:
            if e in out:
                raise ValueError(f"event {e} given twice")
            out[e] = (fate_, f"cook_gpu.h:{line}")
    return out


_TABLE = {
    # cook_state_task_facts: "every running upsert ... and every cook_state_launch writes the absent facts"
    "max_runtime": _cells(
        (NONE, 965, ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "launch_free", "launch_park",
                     "retry_facts_completed", "pending_upsert", "requeue")),
        (DROP, 442, ("running_rm", "status_completed", "status_running", "status_waiting",
                     "status_waiting_unretained", "status_no_facts", "reset")),
        (RESET, 965, ("running_upsert_live", "running_upsert", "launch")),
        (DROP, 987, ("finish",)),
        (DROP, 1027, ("finish_history",)),
    ),
    "cancelled": _cells(
        (NONE, 965, ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "launch_free", "launch_park",
                     "retry_facts_completed", "pending_upsert", "requeue")),
        (DROP, 442, ("running_rm", "status_completed", "status_running", "status_waiting",
                     "status_waiting_unretained", "status_no_facts", "reset")),
        (RESET, 965, ("running_upsert_live", "running_upsert", "launch")),
        (DROP, 987, ("finish",)),
        (DROP, 1027, ("finish_history",)),
    ),
    "unknown": _cells(
        (NONE, 965, ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "launch_free", "launch_park",
                     "retry_facts_completed", "pending_upsert", "requeue")),
        (DROP, 442, ("running_rm", "status_completed", "status_running", "status_waiting",
                     "status_waiting_unretained", "status_no_facts", "reset")),
        (RESET, 965, ("running_upsert_live", "running_upsert", "launch")),
        (DROP, 987, ("finish",)),
        (DROP, 1027, ("finish_history",)),
    ),
    # cook_state_task_reason: a running upsert and a launch write -1; with reason_code NULL a finished row's reason and the
    # retry decision's are the running row's fact
    "reason": _cells(
        (NONE, 974, ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "launch_free", "launch_park",
                     "retry_facts_completed", "pending_upsert", "requeue")),
        (DROP, 442, ("running_rm", "reset")),
        (RESET, 978, ("running_upsert_live", "running_upsert", "launch")),
        (DROP, 987, ("finish",)),
        (COPY, 1012, ("finish_history",)),
        (COPY, 1112, _STATUS_EXITS),
    ),
    # cook_state_job_facts: on live pending rows; an upsert writes flags 0, a requeue clears them as an upsert would
    "job_facts": _cells(
        (DROP, 442, ("pending_rm", "reset")),
        (RESET, 1327, ("pending_upsert_live", "pending_upsert_parked", "pending_upsert")),
        (DROP, 444, ("launch_free",)),
        (KEEP, 1055, ("launch_park",)),
        (NONE, 1319, ("running_rm", "running_upsert_live", "status_running", "status_waiting",
                      "status_waiting_unretained", "status_no_facts", "running_upsert", "launch")),
        (DROP, 1081, ("finish", "finish_history")),
        (DROP, 1079, ("status_completed",)),
        (DROP, 1101, ("retry_facts_completed",)),
        (RESET, 1073, ("requeue",)),
    ),
    # cook_state_list_facts: every upsert writes "no facts", a launch copies them, a parked copy and a requeue keep them
    "list_facts": _cells(
        (DROP, 442, ("pending_rm", "running_rm", "finish", "finish_history", "status_completed", "status_running",
                     "status_waiting", "status_waiting_unretained", "status_no_facts", "reset")),
        (RESET, 1414, ("pending_upsert_live", "pending_upsert_parked", "running_upsert_live", "pending_upsert",
                       "running_upsert")),
        (COPY, 1415, ("launch_free", "launch")),
        (KEEP, 1416, ("launch_park",)),
        (DROP, 1101, ("retry_facts_completed",)),
        (KEEP, 1417, ("requeue",)),
    ),
    # cook_state_retry_facts: per job; a pending upsert or removal drops them, they survive launch and requeue
    "retry_facts": _cells(
        (DROP, 1082, ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "reset")),
        (NONE, 1058, ("launch_free",)),
        (KEEP, 1100, ("launch_park", "running_rm", "running_upsert_live", "status_running", "status_waiting",
                      "status_waiting_unretained", "launch", "requeue")),
        (DROP, 1083, ("finish", "finish_history", "status_completed")),
        (NONE, 1111, ("status_no_facts",)),
        (DROP, 1101, ("retry_facts_completed",)),
        (NONE, 1082, ("pending_upsert",)),
        (NONE, 1097, ("running_upsert",)),
    ),
    # the parked pending copy: made by a launch of a job with retry facts, live again by a requeue, freed otherwise
    "parked_copy": _cells(
        (NONE, 1053, ("pending_rm", "pending_upsert_live", "launch_free", "running_rm", "running_upsert_live",
                      "status_waiting_unretained", "status_no_facts", "pending_upsert", "running_upsert", "launch")),
        (DROP, 1081, ("pending_upsert_parked", "finish", "finish_history")),
        (KEEP, 1055, ("launch_park",)),
        (DROP, 1079, ("status_completed",)),
        (KEEP, 1068, ("status_running",)),
        (KEEP, 1071, ("status_waiting", "requeue")),
        (DROP, 1080, ("retry_facts_completed",)),
        (DROP, 1082, ("reset",)),
    ),
    # cook_state_patch's allowed and plugin_accept: pending columns; a parked copy and a requeue keep them
    "allowed": _cells(
        (DROP, 442, ("pending_rm", "reset")),
        (RESET, 442, ("pending_upsert_live",)),
        (RESET, 1081, ("pending_upsert_parked",)),
        (DROP, 444, ("launch_free",)),
        (KEEP, 1055, ("launch_park",)),
        (NONE, 491, ("running_rm", "running_upsert_live", "status_running", "status_waiting_unretained",
                     "status_no_facts", "running_upsert", "launch")),
        (DROP, 1081, ("finish", "finish_history")),
        (DROP, 1079, ("status_completed",)),
        (KEEP, 1073, ("status_waiting", "requeue")),
        (DROP, 1101, ("retry_facts_completed",)),
        (RESET, 430, ("pending_upsert",)),
    ),
    # reserved_host: as allowed, except that a requeue sets it to -1 (the reservation was consumed at launch)
    "reserved_host": _cells(
        (DROP, 442, ("pending_rm", "reset")),
        (RESET, 442, ("pending_upsert_live",)),
        (RESET, 1081, ("pending_upsert_parked",)),
        (DROP, 444, ("launch_free",)),
        (KEEP, 1055, ("launch_park",)),
        (NONE, 491, ("running_rm", "running_upsert_live", "status_running", "status_waiting_unretained",
                     "status_no_facts", "running_upsert", "launch")),
        (DROP, 1081, ("finish", "finish_history")),
        (DROP, 1079, ("status_completed",)),
        (KEEP, 1071, ("status_waiting",)),
        (DROP, 1101, ("retry_facts_completed",)),
        (RESET, 430, ("pending_upsert",)),
        (RESET, 1072, ("requeue",)),
    ),
    # the straggler records: a success appends one per entry of its group list; a reset drops them
    "records": _cells(
        (NONE, 986, ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "launch_free", "launch_park",
                     "running_rm", "running_upsert_live", "retry_facts_completed", "pending_upsert",
                     "running_upsert", "launch", "requeue")),
        (COPY, 987, ("finish",)),
        (COPY, 1027, ("finish_history",)),
        (COPY, 1108, _STATUS_EXITS),
        (DROP, 990, ("reset",)),
    ),
}
FATE = {(f, e): cell for f, row in _TABLE.items() for e, cell in row.items()}
CONSULTED = set()   # the cells fate() has read

# the C entry points that change a handle, by the events they are made of; and those that only read
WRITERS = {
    "cook_state_apply": ("pending_rm", "pending_upsert_live", "pending_upsert_parked", "running_rm",
                         "running_upsert_live", "reset", "pending_upsert", "running_upsert"),
    "cook_state_launch": ("launch_free", "launch_park", "launch"),
    "cook_state_finish": ("finish",),
    "cook_state_finish_history": ("finish_history",),
    "cook_state_status": ("status_completed", "status_running", "status_waiting", "status_waiting_unretained",
                          "status_no_facts", "requeue"),
    "cook_state_retry_facts": ("retry_facts_completed",),
}
# calls that write a fact in place (no row in or out): the fact they set, or what they keep outside the rows
SETTERS = {
    "cook_state_task_facts": ("max_runtime", "cancelled", "unknown"), "cook_state_task_reason": ("reason",),
    "cook_state_job_facts": ("job_facts",), "cook_state_list_facts": ("list_facts",),
    "cook_state_patch": ("allowed", "reserved_host"), "cook_state_retry_config": ("retry_facts",),
    "cook_state_group_runtimes": ("records",),
    # outside the rows: the history, the completed-job log, the live offers, the queue and the last match round
    "cook_state_history_seed": (), "cook_state_history_advance": (), "cook_state_completed_seed": (),
    "cook_state_completed_record": (), "cook_state_completed_advance": (), "cook_state_offers_add": (),
    "cook_state_rank": (), "cook_state_rank_offensive": (), "cook_state_considerable": (), "cook_state_match": (),
    "cook_state_match_derived": (), "cook_state_match_offers": (), "cook_state_match_metrics": (),
}
READERS = ("cook_state_rebalance", "cook_state_rebalance_derived", "cook_state_rebalance_offers", "cook_state_usage",
           "cook_state_cotasks", "cook_state_digest", "cook_state_counts_compare", "cook_state_export",
           "cook_state_queue", "cook_state_user_stats", "cook_state_sweep", "cook_state_unscheduled",
           "cook_state_user_usage", "cook_state_instance_stats", "cook_state_history_stats", "cook_state_list_jobs",
           "cook_state_list_completed")

OUTCOME_EVENT = {"completed": "status_completed", "running": "status_running", "waiting": "status_waiting",
                 "waiting_unretained": "status_waiting_unretained", "no_facts": "status_no_facts"}


def fate(fact, event):
    CONSULTED.add((fact, event))
    return FATE[(fact, event)][0]


# ---- the model ---------------------------------------------------------------------------------------------------
_RUNNING_FACTS = ("max_runtime", "cancelled", "unknown", "reason", "list_facts")   # on a running row
_PENDING_FACTS = ("job_facts", "list_facts", "allowed", "reserved_host")             # on a pending row
_COL_FACT = {"jf": "job_facts", "lf": "list_facts"}
_RUN_ABSENT = dict(max_runtime=-1, cancelled=0, unknown=0, reason=-1)
_PEND_ABSENT = dict(allowed=1, plugin_accept=1, reserved_host=-1)


class Model:
    """What one handle should hold: pending {job id: row}, parked {job id: row}, running {task id: row}, retry {job
    id: facts (retry_ref.decide's dict)}, the history (history_ref.History), the records [(group, runtime_s)] and the
    unmatched counts of the last counted match round {job id: cycles}."""

    def __init__(self, mea_culpa_limit=5, reason_of=None):
        self.pend, self.parked, self.run, self.retry = {}, {}, {}, {}
        self.hist, self.records, self.mm_prev = HR.History(), [], {}
        self.limit, self.reason_of = mea_culpa_limit, dict(reason_of or {})

    # -- rows in and out, each through its cells --------------------------------------------------------------------
    def _pending_in(self, row, event, old=None):
        """The row a pending upsert (event pending_upsert) or a requeue (event requeue) makes live."""
        self._event(event)
        r = dict(row)
        r["jf"] = None if fate("job_facts", event) == RESET else (old or r).get("jf")
        r["lf"] = None if fate("list_facts", event) == RESET else (old or r).get("lf")
        for c in ("allowed", "plugin_accept"):
            r[c] = (old or r).get(c, _PEND_ABSENT[c]) if fate("allowed", event) == KEEP else row.get(c, _PEND_ABSENT[c])
        if fate("reserved_host", event) == RESET and event == "requeue":
            r["reserved_host"] = -1
        return r

    def _running_in(self, row, event, lf=None):
        self._event(event)
        r = dict(row)
        for f, v in _RUN_ABSENT.items():
            if fate(f, event) == RESET:
                r[f] = v
        r["lf"] = lf if fate("list_facts", event) == COPY else None
        return r

    @staticmethod
    def _event(event, gone=()):
        """Every fact's cell for `event`, read as the event happens.  `gone` are the facts of a row the event deletes:
        their cells must say that they leave with it (drop) or move on (copy)."""
        cells = {f: fate(f, event) for f in FACTS}
        for f in gone:
            if cells[f] not in (DROP, COPY):
                raise ValueError(f"the model deletes the row that holds {f} at {event}, the table says {cells[f]}")
        return cells

    def _free(self, j, event, keep_facts=False):
        """The job's parked copy and retry facts after `event`, as their cells say; keep_facts: the header keeps the
        facts whatever the cell while the job has a live pending row or another live instance."""
        cells = self._event(event)
        if cells["parked_copy"] == DROP:
            self.parked.pop(j, None)
        if cells["retry_facts"] == DROP and not keep_facts:
            self.retry.pop(j, None)

    def apply(self, up=(), rm=(), run_up=(), run_rm=(), reset=False):
        if reset:
            self._event("reset", gone=FACTS)
            self.pend, self.parked, self.run, self.retry = {}, {}, {}, {}
            self.hist.reset()
            self.records, self.mm_prev = [], {}
        for j in rm:
            del self.pend[j]
            self._event("pending_rm", gone=_PENDING_FACTS)
            self._free(j, "pending_rm")
        for t in run_rm:
            del self.run[t]
            self._event("running_rm", gone=_RUNNING_FACTS)
        for j, r in up:   # an upsert of a held id resets by its exit cells, a new id by the entry's
            ev = "pending_upsert_parked" if j in self.parked else "pending_upsert_live" if j in self.pend else None
            if ev:
                self._free(j, ev)
            self.pend[j] = self._pending_in(r, ev or "pending_upsert")
        for r in run_up:
            ev = "running_upsert_live" if r["task_id"] in self.run else "running_upsert"
            self.run[r["task_id"]] = self._running_in(r, ev)

    def launch(self, jobs, tids, starts, hosts=None):
        for k, j in enumerate(jobs):
            p = self.pend.pop(j)
            park = j in self.retry
            cells = self._event("launch_park" if park else "launch_free", gone=() if park else _PENDING_FACTS)
            if park and cells["parked_copy"] == KEEP:
                self.parked[j] = dict(p, **{f: None for f in ("jf", "lf") if cells[_COL_FACT[f]] != KEEP})
            run = dict(user=p["user"], priority=p.get("priority", 50), start_time=int(starts[k]), task_id=int(tids[k]),
                       job_id=j, cpus=p["cpus"], mem=p["mem"], gpus=p.get("gpus", 0.0),
                       host=-1 if hosts is None else int(hosts[k]), groups=list(p.get("groups", [])))
            self.run[int(tids[k])] = self._running_in(run, "launch", p.get("lf"))

    def patch(self, jobs, allowed=None, plugin_accept=None, reserved_host=None):
        for k, j in enumerate(jobs):
            for c, v in (("allowed", allowed), ("plugin_accept", plugin_accept), ("reserved_host", reserved_host)):
                if v is not None:
                    self.pend[j][c] = int(v[k])

    def task_facts(self, tids, max_runtime=None, cancelled=None, unknown=None):
        for k, t in enumerate(tids):
            for c, v in (("max_runtime", max_runtime), ("cancelled", cancelled), ("unknown", unknown)):
                if v is not None:
                    self.run[t][c] = int(v[k])

    def task_reason(self, tids, codes):
        for t, c in zip(tids, codes):
            self.run[t]["reason"] = int(c)

    def job_facts(self, jobs, facts):
        """facts: one dict per job (facts, gpu_model, disk_type, disk_request, disk_limit)."""
        for j, f in zip(jobs, facts):
            self.pend[j]["jf"] = dict(f)

    def list_facts(self, jobs, submit, pool, executor):
        for j, s, p, x in zip(jobs, submit, pool, executor):
            lf = (int(s), int(p), int(x))
            if j in self.pend:
                self.pend[j]["lf"] = lf
            for r in self.run.values():
                if r["job_id"] == j:
                    r["lf"] = lf

    def holds(self, j):
        return j in self.pend or j in self.parked or any(r["job_id"] == j for r in self.run.values())

    def retry_facts(self, jobs, max_retries, flags, done):
        for j, m, f, d in zip(jobs, max_retries, flags, done):
            self.retry[j] = dict(max_retries=int(m), disable=bool(f & 1), completed=bool(f & 2), done=list(d))
            if f & 2 and j in self.parked and not any(r["job_id"] == j for r in self.run.values()):
                self._free(j, "retry_facts_completed")

    def group_runtimes(self, add=(), forget=()):
        self.records = [x for x in self.records if x[0] not in set(forget)] + [tuple(x) for x in add]

    def _leave(self, t, end, ok, reason, event):
        """A running row leaves by a finish, finish_history or status: its records and history row."""
        r = self.run.pop(t)
        self._event(event, gone=_RUNNING_FACTS)
        if ok and fate("records", event) == COPY:
            self.records += [(g, SR.runtime_s(r["start_time"], end)) for g in r["groups"]]
        if event != "finish":
            code = r["reason"] if reason is None and fate("reason", event) == COPY else reason
            self.hist.finish({t: dict(r, reason=code)}, [t], [end], [ok], None if code is None else [code])
        return r

    def finish(self, tids, end=None, success=None, history=False, reason=None):
        event = "finish_history" if history else "finish"
        for i, t in enumerate(tids):
            ok = bool(success[i]) if success is not None else False
            r = self._leave(t, end[i] if end is not None else 0, ok, None if reason is None else reason[i], event)
            j = r["job_id"]
            if j in self.retry and not any(x["job_id"] == j for x in self.run.values()):
                self._free(j, event, keep_facts=j in self.pend)

    def status(self, tids, success, end, reason=None, preempted=None):
        """cook_state_status: the outcomes (names of OUTCOME_EVENT) and attempts, the requeues done."""
        out = []
        for i, t in enumerate(tids):
            probe = self.run[t]
            code = probe["reason"] if reason is None else int(reason[i])
            j, host = probe["job_id"], probe["host"]
            if j not in self.retry:
                self._leave(t, end[i], bool(success[i]), None if reason is None else reason[i], "status_no_facts")
                out.append(("no_facts", -1))
                continue
            other = any(x["job_id"] == j and x["task_id"] != t for x in self.run.values())
            name, att, facts = RR.decide(self.retry[j], self.reason_of, bool(success[i]), code, other, self.limit)
            if name == "waiting" and j not in self.parked:
                name = "waiting_unretained"
            event = OUTCOME_EVENT[name]
            self._leave(t, end[i], bool(success[i]), None if reason is None else reason[i], event)
            self.retry[j] = facts
            if name != "waiting":
                self._free(j, event, keep_facts=other or j in self.pend)
            elif fate("parked_copy", event) != KEEP:
                raise ValueError("a requeue needs the parked copy kept")
            else:
                row = self.parked.pop(j)
                pre = bool(preempted[i]) if preempted is not None else False
                row = dict(row, novel=RR.novel_after(row["novel"], host, pre))
                self.pend[j] = self._pending_in(row, "requeue", row)
            out.append((name, att))
        return out

    # -- projections onto the restatements' inputs -------------------------------------------------------------------
    def sweep_rows(self, pool=0):
        return [dict(task_id=t, start=r["start_time"], max_runtime=r["max_runtime"], cancelled=bool(r["cancelled"]),
                     status="unknown" if r["unknown"] else "running", groups=r["groups"], pool=pool)
                for t, r in sorted(self.run.items())]

    def instance_rows(self):
        return {t: dict(user=r["user"], start_time=r["start_time"], cpus=r["cpus"], mem=r["mem"],
                        unknown=bool(r["unknown"]), reason=r["reason"]) for t, r in self.run.items()}

    def list_handle(self):
        return {"pending": [(r["user"], j, r["lf"]) for j, r in self.pend.items()],
                "running": [(r["user"], r["job_id"], t, r["lf"]) for t, r in self.run.items()]}

    def export_rows(self):
        """{job id: (novel, reserved_host, allowed, plugin_accept)} of the live pending rows."""
        return {j: (list(r["novel"]), r["reserved_host"], r["allowed"], r["plugin_accept"]) for j, r in self.pend.items()}

    def metrics_job(self, j):
        """A live pending row as match_metrics_ref reads it."""
        r, f = self.pend[j], self.pend[j]["jf"] or {"facts": 0}
        return dict(job_id=j, user=r["user"], cpus=r["cpus"], mem=r["mem"], gpus=r.get("gpus", 0.0),
                    ports=r.get("ports", 0),
                    **{k: f.get(k, 0) for k in ("facts", "gpu_model", "disk_type", "disk_request", "disk_limit")})


def sweep_answer(models, now, default_timeout_ms, max_timeout_ms, groups):
    rows = [x for p, m in enumerate(models) for x in m.sweep_rows(p)]
    return (SR.lingering(rows, now, default_timeout_ms, max_timeout_ms), SR.cancelled(rows),
            SR.stragglers(rows, [x for m in models for x in m.records], groups, now))


def instance_answer(models, now, status, start_ms, end_ms):
    return IR.answer([m.instance_rows() for m in models], now, status, start_ms, end_ms)


def history_answer(models, status, start_ms, end_ms):
    return HR.answer([m.hist for m in models], status, start_ms, end_ms)


def list_answer(models, user, states, start_ms, end_ms):
    return LR.list_jobs([m.list_handle() for m in models], LR.query(user, states, start_ms, end_ms))
