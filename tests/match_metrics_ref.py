"""Plain-Python restatement of the match-cycle metrics (handle-match-cycle-metrics, scheduler.clj:1210-1280; the
unmatched tracking, :1399-1486) and of cook_state_match_metrics.

A job is a dict {job_id, user, cpus, mem, gpus, ports, facts (abi.JF_* bits), gpu_model, disk_type, disk_request,
disk_limit} in take order.  `resource_maps` is jobs->resource-maps with the gpu model and disk type as codes (-1:
unspecified); `stats` is resource-maps->stats, or ERROR when two or more jobs carry uris (merge-with + adds two
vectors and throws, so jobs->stats returns its error string).  `answer` is what the device call returns for one round
given the previous round's unmatched cycles {job id: cycles}.  The first ten jobs unmatched too long are taken in take
order: the reference's hash-map order is unspecified.
"""
import functools

from instance_stats_ref import percentile

JF_GPUS, JF_DISK, JF_DISK_REQUEST, JF_DISK_LIMIT, JF_URIS = 1, 2, 4, 8, 16
MM_GPUS, MM_DISK_REQUEST, MM_DISK_LIMIT = 0, 1, 2
ERROR = "Error collecting job stats"
FIRST = 10
BLOCK_BYTES = 440   # the counts, amounts, rows and first ten, downloaded as one block


def resource_map(job):
    """job->resource-map: {"cpus", "mem", ("gpus", model), ("disk", kind, type), "uris"} -> amount."""
    m = {"cpus": job["cpus"], "mem": job["mem"]}
    f = job.get("facts", 0)
    if f & JF_GPUS:
        m[(MM_GPUS, job.get("gpu_model", -1))] = job.get("gpus", 0.0)
    if f & JF_DISK:
        if f & JF_DISK_REQUEST:
            m[(MM_DISK_REQUEST, job.get("disk_type", -1))] = job["disk_request"]
        if f & JF_DISK_LIMIT:
            m[(MM_DISK_LIMIT, job.get("disk_type", -1))] = job["disk_limit"]
    if f & JF_URIS:
        m["uris"] = ["uri"]
    return m


def merge_plus(a, b):
    out = dict(a)
    for k, v in b.items():
        if k in out:
            if isinstance(v, list):
                raise TypeError("merge-with + over two uri vectors")
            out[k] = out[k] + v
        else:
            out[k] = v
    return out


def stats(jobs):
    """jobs->stats: percentiles 50/95/100 and the last maximal row (positions) of cpus and mem, and the totals, or
    ERROR."""
    maps = [resource_map(j) for j in jobs]
    try:
        totals = functools.reduce(merge_plus, maps) if maps else None
    except TypeError:
        return ERROR
    out = {"percentiles": {}, "largest-by": {}, "totals": totals}
    for r in ("cpus", "mem"):
        vals = sorted(m[r] for m in maps)
        out["percentiles"][r] = {p: percentile(vals, p) for p in (50, 95, 100)}
        order = sorted(range(len(maps)), key=lambda k: maps[k][r])   # stable, so `last` is the last maximal row
        out["largest-by"][r] = order[-1] if order else None
    return out


def unmatched_cycles(prev, considerable, matched):
    """The new {job id: cycles} map: the considerable jobs not matched, each prev + 1."""
    return {j: prev.get(j, 0) + 1 for j in considerable if j not in matched}


def answer(jobs, matched_positions, prev, threshold, n_users):
    """cook_state_match_metrics' answer for one round: jobs in take order, the positions matched after the drops."""
    N = len(jobs)
    matched = set(matched_positions)
    ids = [j["job_id"] for j in jobs]
    cyc = unmatched_cycles(prev, ids, {ids[k] for k in matched})
    ucons, umat = [0] * n_users, [0] * n_users
    for k, j in enumerate(jobs):
        ucons[j["user"]] += 1
        umat[j["user"]] += k in matched
    too_long = [(ids[k], cyc[ids[k]]) for k in range(N) if ids[k] in cyc and cyc[ids[k]] > threshold]
    out = {"considerable": N, "matched": len(matched), "head_job_id": ids[0] if N else -1,
           "head_matched": int(0 in matched), "user_considerable": ucons, "user_matched": umat,
           "too_long": len(too_long), "first": too_long[:FIRST], "cycles": cyc}
    uris = [k for k, j in enumerate(jobs) if j.get("facts", 0) & JF_URIS]
    out["uris"] = len(uris)
    out["uris_position"] = uris[0] if len(uris) == 1 else -1
    if not N:
        out["keys"] = []
        return out
    maps = [resource_map(j) for j in jobs]
    keyed = {}
    for m in maps:
        for k, v in m.items():
            if isinstance(k, tuple):
                keyed[k] = keyed[k] + v if k in keyed else v
    out["keys"] = sorted((k[0], k[1], v) for k, v in keyed.items())
    out["total_cpus"] = functools.reduce(lambda a, b: a + b, (j["cpus"] for j in jobs))
    out["total_mem"] = functools.reduce(lambda a, b: a + b, (j["mem"] for j in jobs))
    for r in ("cpus", "mem"):
        vals = sorted(j[r] for j in jobs)
        out["pct_" + r] = [percentile(vals, p) for p in (50, 95, 100)]
        out["largest_" + r] = sorted(range(N), key=lambda k: jobs[k][r])[-1]
    return out


def down_bytes(n_considerable, n_users, n_keys, changed=False):
    """The call's downloads when it answers."""
    if not n_considerable:
        return 0
    return 32 + (4 * n_considerable if changed else 0) + BLOCK_BYTES + 8 * n_users + 16 * n_keys


def golden_rounds(case):
    """A golden case's rounds with each "repeat": k expanded into k rounds without an expected answer."""
    for r in case:
        for _ in range(r.get("repeat", 1)):
            yield r


def named_job(ref_job, gpu_codes, disk_codes):
    """A transcribed reference job ({gpu_model name or None, resources}) as a row, with the names coded through the
    given dictionaries (filled as new names appear)."""
    res = ref_job["resources"]
    f, row = 0, {"job_id": 0, "user": 0, "cpus": res["cpus"], "mem": res["mem"], "gpus": res.get("gpus", 0.0),
                 "ports": 0, "gpu_model": -1, "disk_type": -1, "disk_request": 0.0, "disk_limit": 0.0}
    if "gpus" in res:
        f |= JF_GPUS
        if ref_job["gpu_model"] is not None:
            row["gpu_model"] = gpu_codes.setdefault(ref_job["gpu_model"], len(gpu_codes))
    if "disk" in res:
        d = res["disk"]
        f |= JF_DISK
        if "type" in d:
            row["disk_type"] = disk_codes.setdefault(d["type"], len(disk_codes))
        if d.get("request") is not None:
            f |= JF_DISK_REQUEST
            row["disk_request"] = d["request"]
        if d.get("limit") is not None:
            f |= JF_DISK_LIMIT
            row["disk_limit"] = d["limit"]
    row["facts"] = f
    return row


def key_name(kind, code, gpu_names, disk_names):
    """A (kind, code) key as the reference's string key."""
    if kind == MM_GPUS:
        return "gpus/" + (gpu_names[code] if code >= 0 else "unspecified-gpu-model")
    t = disk_names[code] if code >= 0 else "unspecified-disk-type"
    return f"disk/{t}/" + ("request" if kind == MM_DISK_REQUEST else "limit")


def named_resource_map(row, gpu_names, disk_names):
    return {k if isinstance(k, str) else key_name(k[0], k[1], gpu_names, disk_names): v
            for k, v in resource_map(row).items()}
