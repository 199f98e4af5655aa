"""Plain-Python restatement of /unscheduled_jobs (cook.unscheduled, unscheduled.clj) and of cook_state_unscheduled.

The reference's functions over plain values: how-job-would-exceed-resource-limits (usage maps folded left with
merge-with +), check-queue-position (same-user-task-comparator over the running jobs' last running instance and the
waiting jobs' synthetic tasks, with the reference's waiting cap as an optional argument), fenzo-failures-for-user and
reasons.  `answer` is what cook_state_unscheduled returns over a host mirror of a handle's rows: pending {job id: row}
and running {task id: row}, every live row counted, one row per running job (its greatest task id), the usage a left
fold in ascending task id of those rows, then plus the job.
"""
import functools

AHEAD = 10
INT64_MAX = 2 ** 63 - 1
ABSENT, WAITING, RUNNING = 0, 1, 2
CONSTRAINT_MESSAGES = {
    "novel_host_constraint": "Job already ran on this host.",
    "gpu_host_constraint": "Host has no GPU support.",
    "non_gpu_host_constraint": "Host is reserved for jobs that need GPU support.",
    "attribute-equals-host-placement-group-constraint": "Host had a different attribute than other jobs in the group."}


def job_usage(job):
    """tools/job->usage: {count 1, cpus, mem}, gpus when the job has them."""
    u = {"count": 1, "cpus": job["cpus"], "mem": job["mem"]}
    if job.get("gpus") is not None:
        u["gpus"] = job["gpus"]
    return u


def merge_with_plus(a, b):
    out = dict(a)
    for k, v in b.items():
        out[k] = out[k] + v if k in out else v
    return out


def how_job_would_exceed_resource_limits(limits, running_jobs, job):
    total = functools.reduce(merge_with_plus, [job_usage(j) for j in list(running_jobs) + [job]])
    return {k: {"limit": v, "usage": total.get(k)} for k, v in limits.items() if (total.get(k) or 0) > v}


def feature(task):
    """task->feature-vector (tools.clj:614-628): a running row, or a pending job's synthetic task."""
    if "task_id" in task:
        return (-task["priority"], task["start_time"], task["task_id"], task["job_id"])
    return (-task["priority"], INT64_MAX, -1, task["job_id"])


def check_queue_position(job_id, running_tasks, waiting_jobs, cap=None):
    """check-queue-position (:120-148): running_tasks one row per running job, waiting_jobs pending rows (with
    job_id) in the order the reference's query returns them, the first `cap` kept.  None or [message, {jobs}]."""
    waiting = list(waiting_jobs)[:cap] if cap is not None else list(waiting_jobs)
    tasks = sorted(list(running_tasks) + waiting, key=feature)
    pos = next((i for i, t in enumerate(tasks) if t["job_id"] == job_id), len(tasks))
    ahead = tasks[:min(pos, AHEAD)]
    if not ahead:
        return None
    msg = (f"You have at least {pos} other jobs ahead in the queue." if pos == len(tasks)
           else f"You have {pos} other jobs ahead in the queue.")
    return [msg, {"jobs": [t["job_id"] for t in ahead]}]


def fenzo_failures_for_user(summary):
    return ([{"reason": f"Not enough {k} available.", "host_count": v} for k, v in summary.get("resources", {}).items()] +
            [{"reason": CONSTRAINT_MESSAGES.get(k, k), "host_count": v} for k, v in summary.get("constraints", {}).items()])


def reasons(job, running_jobs, running_tasks, waiting_jobs, *, quota=None, share=None, attempts_consumed=0,
            max_retries=None, enforcing_rate_limit=False, num_rate_limited=0, plugin_status=None, plugin="",
            plugin_message=None, placement_failure=None, cap=None):
    """reasons (:172-200): job {job_id, state, cpus, mem[, gpus]}; running_jobs their usage rows; running_tasks one
    row per running job; waiting_jobs the user's waiting rows (cap: the reference's 100)."""
    if job["state"] == "running":
        return [["The job is running now.", {}]]
    if job["state"] == "completed":
        return [["The job already completed.", {}]]
    out = []
    if max_retries is not None and attempts_consumed >= max_retries:
        out.append(["Job has exhausted its maximum number of retries.",
                    {"max-retries": max_retries, "instance-count": attempts_consumed}])
    for limits, msg in ((quota, "The job would cause you to exceed resource quotas."),
                        (share, "The job would cause you to exceed resource shares.")):
        ways = how_job_would_exceed_resource_limits(limits or {}, running_jobs, job)
        if ways:
            out.append([msg, ways])
    if enforcing_rate_limit and num_rate_limited > 0:
        out.append(["You are currently rate limited on how many jobs you launch per minute.",
                    {"num-ratelimited": num_rate_limited}])
    if plugin_status == "deferred":
        out.append(["The launch filter plugin is blocking the job launch.", {"plugin": plugin, "message": plugin_message}])
    q = check_queue_position(job["job_id"], running_tasks, waiting_jobs, cap)
    if q:
        out.append(q)
    if placement_failure:
        out.append(["The job couldn't be placed on any available hosts.",
                    {"reasons": fenzo_failures_for_user(placement_failure)}])
    else:
        out.append(["The job is now under investigation. Check back in a minute for more details!", {}])
    return out


# ---- cook_state_unscheduled over a host mirror -------------------------------------------------------------------
def representatives(run):
    """{(user, job id): the row with the greatest task id} of running rows {task id: row}."""
    rep = {}
    for t, r in run.items():
        k = (r["user"], r["job_id"])
        if k not in rep or t > rep[k]["task_id"]:
            rep[k] = r
    return rep


def answer(pend, run, job_ids):
    """Per queried id: (status, usage (count, cpus, mem, gpus), position, ahead job ids, plugin deferred)."""
    rep = representatives(run)
    reps_of, entries_of = {}, {}
    for (u, _), r in rep.items():
        reps_of.setdefault(u, []).append(r)
        entries_of.setdefault(u, []).append(r)
    for j, r in pend.items():
        entries_of.setdefault(r["user"], []).append(dict(r, job_id=j))
    top = {}   # job id -> its running row with the greatest task id, over every user
    for t, r in run.items():
        if r["job_id"] not in top or t > top[r["job_id"]]["task_id"]:
            top[r["job_id"]] = r
    order, fold = {}, {}   # per user: its entries in order with each feature's position; its running fold
    out = []
    for j in job_ids:
        if j in pend:
            st, row = WAITING, dict(pend[j], job_id=j)
        elif j in top:
            st, row = RUNNING, top[j]
        else:
            out.append((ABSENT, (0.0, 0.0, 0.0, 0.0), -1, [], 0))
            continue
        u = row["user"]
        if u not in order:
            es = sorted(entries_of[u], key=feature)
            order[u] = (es, {feature(e): i for i, e in enumerate(es)})
            c, m, g = 0.0, 0.0, 0.0
            rs = sorted(reps_of.get(u, []), key=lambda r: r["task_id"])
            for r in rs:   # the left fold in ascending task id
                c, m, g = c + r["cpus"], m + r["mem"], g + r.get("gpus", 0.0)
            fold[u] = (float(len(rs)), c, m, g)
        es, at = order[u]
        pos = at[feature(row)]
        ahead = [e["job_id"] for e in es[:min(pos, AHEAD)]]
        usage, plugin = (0.0, 0.0, 0.0, 0.0), 0
        if st == WAITING:
            n, c, m, g = fold[u]
            usage = (n + 1.0, c + row["cpus"], m + row["mem"], g + row.get("gpus", 0.0))
            plugin = int(row.get("plugin_accept", 1) == 0)
        out.append((st, usage, pos, ahead, plugin))
    return out


def engine_answer(pend, run, job_ids):
    """`answer` in engine.state_unscheduled's shape (numpy columns), for cycle.unscheduled_reasons on the CPU."""
    import numpy as np
    a = answer(pend, run, job_ids)
    return {"job_id": np.asarray(job_ids, np.int64), "status": np.array([x[0] for x in a], np.uint8),
            "usage": np.array([x[1] for x in a], np.float64).reshape(len(a), 4),
            "position": np.array([x[2] for x in a], np.int32), "ahead": [x[3] for x in a],
            "plugin_deferred": np.array([x[4] for x in a], np.uint8)}
