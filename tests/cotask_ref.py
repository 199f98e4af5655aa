"""Each group's running cotasks (cook_state_cotasks), restated in plain Python from the live running rows.

A group's cotasks are the running instances of its jobs (group->running-task-set, group.clj:47-57) that Fenzo's
tracker knows, i.e. that have a host (get-cotasks-from-tracker-state, constraints.clj:539-552).  Each is listed
with its hostname code and the value of the group's attribute on that host (0, nil, when the host is not in the
table or the group names no column).  Within a group the entries are in ascending task id (DESIGN.md §2).
"""


def cotasks(rows, n_groups, attr_col=None, hostname_id=None, attr=None):
    """rows: dicts with task_id, host (hostname code, -1 unknown) and groups (group codes).  attr_col[g]: the
    group's attribute column or -1; hostname_id[h] and attr[c][h]: the host table (None: no table).
    Returns (off[n_groups + 1], hostname_id, attr_val) as lists: the CSR cook_groups.cot_* holds."""
    index = {int(c): h for h, c in enumerate(hostname_id)} if hostname_id is not None else {}
    per = [[] for _ in range(n_groups)]
    for r in sorted(rows, key=lambda r: r["task_id"]):
        if r["host"] == -1:
            continue
        h = index.get(int(r["host"]))
        for g in r["groups"]:
            c = int(attr_col[g]) if attr_col is not None else -1
            val = int(attr[c][h]) if h is not None and c >= 0 else 0
            per[g].append((int(r["host"]), val))
    off = [0]
    for p in per:
        off.append(off[-1] + len(p))
    return off, [h for p in per for h, _ in p], [v for p in per for _, v in p]
