"""Plain-Python restatement of a failed task's way back to the queue, as Cook decides it.

- `reasons_attempts_consumed`: :job/reasons->attempts-consumed (scheduler/src/cook/schema.clj:1154-1172).
- `attempts_consumed`: :job/attempts-consumed (:1174-1189) over a job's instances: the done (success or failed) ones.
- `job_state_after`: :instance/update-state's job-state cond (:1242-1300) for one status, with the transition check.
- `transact`: several :instance/update-state calls in one transaction, each reading the state before it.
- `previous_hosts_to_avoid`: job->previous-hosts-to-avoid (scheduler/constraints.clj:84-91).
- `requeued_row`: the pending row a requeue leaves: reserved_host -1 and the failed host appended to the novel list.

A reason is None (nil) or a dict with code, mea_culpa and failure_limit (None: unset).  An instance is a dict with
status ("unknown", "running", "success", "failed") and reason.
"""
from collections import Counter

DONE = ("success", "failed")
TRANSITIONS = {"unknown": ("running", "failed", "success"), "running": ("failed", "success"), "success": (),
               "failed": ()}


def _key(reason):
    return None if reason is None else (reason["code"], bool(reason["mea_culpa"]), reason.get("failure_limit"))


def reasons_attempts_consumed(mea_culpa_limit, disable_mea_culpa, reasons):
    """frequencies of the reasons; a mea-culpa reason's count beyond its limit, every other reason's whole count."""
    total = 0
    for key, count in Counter(_key(r) for r in reasons).items():
        if key is None or not key[1]:          # a nil reason counts as a plain failure
            total += count
            continue
        limit = 0 if disable_mea_culpa else (key[2] if key[2] is not None else mea_culpa_limit)
        total += 0 if limit == -1 else max(0, count - limit)
    return total


def attempts_consumed(instances, mea_culpa_limit=5, disable_mea_culpa=False):
    return reasons_attempts_consumed(mea_culpa_limit, disable_mea_culpa,
                                     [i.get("reason") for i in instances if i["status"] in DONE])


def job_state_after(job, instances, k, new_status, reason, mea_culpa_limit=5):
    """The job state writes of :instance/update-state of instance k to new_status: None when the transition is not
    valid (nothing written), [] for no job change, else [new job state].  job: state, max_retries, disable."""
    if new_status not in TRANSITIONS[instances[k]["status"]]:
        return None
    states = [new_status] + [i["status"] for j, i in enumerate(instances) if j != k]
    after = [dict(i) for i in instances]
    after[k] = dict(status=new_status, reason=reason)
    # the job entity with this instance's new status and reason conj'd onto its instances (the old one stays too)
    consumed = attempts_consumed(instances + [after[k]], mea_culpa_limit, job["disable"])
    if job["state"] == "completed":
        return []
    if (all(s == "failed" for s in states) and job["max_retries"] <= consumed) or "success" in states:
        return ["completed"]
    if "running" in states or "unknown" in states:
        return ["running"]
    return ["waiting"]


def transact(job, instances, updates, mea_culpa_limit=5):
    """The job state after one transaction of updates [(k, new_status, reason)], each reading the state before the
    transaction (Datomic's transaction functions see the database as of its start).  Equal writes merge; a
    transaction that writes two different states would be refused by Datomic and raises here."""
    writes = set()
    for k, st, reason in updates:
        w = job_state_after(job, instances, k, st, reason, mea_culpa_limit)
        writes.update(w or [])
    if len(writes) > 1:
        raise ValueError("conflicting job states in one transaction")
    return writes.pop() if writes else job["state"]


def in_order(job, instances, updates, mea_culpa_limit=5):
    """The job state after the updates, one transaction each, in order (how Cook writes task statuses)."""
    job, instances = dict(job), [dict(i) for i in instances]
    for k, st, reason in updates:
        w = job_state_after(job, instances, k, st, reason, mea_culpa_limit)
        if w is None:
            continue
        instances[k] = dict(status=st, reason=reason)
        if w:
            job["state"] = w[0]
    return job["state"]


def previous_hosts_to_avoid(instances):
    """The hostnames of the job's instances that were not preempted, as a set."""
    return {i["hostname"] for i in instances if i.get("preempted") is not True}


def novel_after(novel, host, preempted):
    """A parked job's novel-host list after a requeue from a failure on hostname code `host`."""
    if host == -1 or preempted or host in novel:
        return list(novel)
    return list(novel) + [host]


def requeued_row(row, host, preempted):
    """The pending row a requeue leaves (the columns of resident_model's rows)."""
    return dict(row, reserved_host=-1, novel=novel_after(row["novel"], host, preempted))


def decide(facts, reason_of, success, reason, other_live, mea_culpa_limit=5):
    """One status on the resident handle: (outcome, attempts) as cook_state_status returns them, and the facts after.
    facts: dict(max_retries, disable, completed, done=[reason codes]); reason_of: code -> reason dict or None."""
    facts = dict(facts, done=list(facts["done"]) + [reason])
    att = reasons_attempts_consumed(mea_culpa_limit, facts["disable"],
                                    [reason_of.get(c) if c != -1 else None for c in facts["done"]])
    if facts["completed"]:
        return "completed", att, facts
    if success or (not other_live and att >= facts["max_retries"]):
        return "completed", att, dict(facts, completed=True)
    return ("running" if other_live else "waiting"), att, facts
