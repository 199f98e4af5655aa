"""The completed-job log and its listing restated over record lists in plain Python: get-completed-jobs-by-user
(tools.clj:393-434) as cook_state_list_completed answers it.

A record is (job id, stamp, user, submit ms, submit pool code, custom executor -1 / 0 / 1, kind).  A log is
{"since": horizon, "rows": [record]} in arrival order.  A job's state is its record with the greatest (stamp, handle
index, row); REOPENED means not completed.
"""
SUCCESS, FAILED, REOPENED = 1, 2, 3          # record kinds
L_SUCCESS, L_FAILED, L_COMPLETED = 1, 2, 3   # listed states
NAMES = {"success": L_SUCCESS, "failed": L_FAILED, "completed": L_COMPLETED}
INT32_MAX = (1 << 31) - 1


def seed(since, rows):
    return {"since": since, "rows": [tuple(r) for r in rows]}


def record(log, rows):
    """cook_state_completed_record: appended in order, those submitted before the horizon skipped."""
    log["rows"] += [tuple(r) for r in rows if r[3] >= log["since"]]


def advance(log, since):
    log["since"] = since
    log["rows"] = [r for r in log["rows"] if r[3] >= since]


def refused(logs, start):
    """A listing that starts before a handle's horizon is refused (the caller keeps the Datomic path)."""
    return any(lg["since"] > start for lg in logs)


def list_completed(logs, q, state):
    """cook_state_list_completed: [(job id, submit ms, handle index)] in ascending job id, cut to q["limit"]; q as
    list_ref.query."""
    best = {}
    for k, lg in enumerate(logs):
        for pos, r in enumerate(lg["rows"]):
            j, stamp, user = r[0], r[1], r[2]
            if user != q["user"] or not q["lo"] <= j < q["hi"]:
                continue
            if j not in best or (stamp, k, pos) > best[j][0]:
                best[j] = ((stamp, k, pos), k, r)
    out = []
    for j in sorted(best):
        _, k, (_, _, _, submit, spool, cex, kind) = best[j]
        if kind == REOPENED or (state != L_COMPLETED and kind != state):
            continue
        if not q["start"] <= submit < q["end"]:
            continue
        if not (q["pool"] == -1 or q["handle_pool"][k] == q["pool"] or spool == q["pool"]):
            continue
        if not (q["include_custom_executor"] or cex == 0):
            continue
        out.append((j, submit, k))
    return out[:q["limit"]]
