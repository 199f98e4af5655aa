"""The row hash, the set / queue / bucket fingerprints and the export order of cook_state_digest and
cook_state_export (include/cook_gpu.h, "auditing a resident pool"), restated in plain Python over the host model the
state tests keep: pending rows {job id: row} and running rows {task id: row} as dicts.

A pending row: user, priority, cpus, mem, gpus, ports, allowed, plugin_accept, gpu_model, disk_request, disk_type,
est_end_ms, ckpt_location, reserved_host, novel [host], attr [(column, value)], groups [group].  A running row: user,
priority, start_time, job_id, cpus, mem, gpus, host (absent: -1), groups (absent: []).  A missing optional column
takes the absent value cook_state_apply stores for a NULL column.
"""
import struct

import numpy as np

M = (1 << 64) - 1
ABSENT = dict(gpus=0.0, ports=0, allowed=1, plugin_accept=1, gpu_model=-1, disk_request=-1.0, disk_type=-1,
              est_end_ms=-1, ckpt_location=-1, reserved_host=-1)
# the data columns in hash order: name, and whether the word is the bit pattern of a double
PENDING_COLS = [("user", 0), ("priority", 0), ("cpus", 1), ("mem", 1), ("gpus", 1), ("ports", 0), ("allowed", 0),
                ("plugin_accept", 0), ("gpu_model", 0), ("disk_request", 1), ("disk_type", 0), ("est_end_ms", 0),
                ("ckpt_location", 0), ("reserved_host", 0)]
RUNNING_COLS = [("user", 0), ("priority", 0), ("start_time", 0), ("job_id", 0), ("cpus", 1), ("mem", 1), ("gpus", 1),
                ("host", 0)]


def mix(z):
    z &= M
    z ^= z >> 30
    z = (z * 0xbf58476d1ce4e5b9) & M
    z ^= z >> 27
    z = (z * 0x94d049bb133111eb) & M
    return z ^ (z >> 31)


def absorb(h, w):
    return mix(((h ^ (w & M)) + 0x9e3779b97f4a7c15) & M)


def word(x, is_double=False):
    """One column value as its 64-bit word: a double by its bits, an integer sign-extended."""
    if is_double:
        return struct.unpack("<Q", struct.pack("<d", float(x)))[0]
    return int(x) & M


def _row(tag, rid, r, cols, lists):
    h = absorb(tag, word(rid))
    for name, dbl in cols:
        h = absorb(h, word(r.get(name, ABSENT.get(name, -1 if name == "host" else 0)), dbl))
    for entries in lists:
        h = absorb(h, len(entries))
        for e in entries:
            for w in (e if isinstance(e, (tuple, list)) else (e,)):
                h = absorb(h, word(w))
    return h


def pending_hash(job_id, r):
    return _row(1, job_id, r, PENDING_COLS, (r.get("novel", []), r.get("attr", []), r.get("groups", [])))


def running_hash(task_id, r):
    return _row(2, task_id, r, RUNNING_COLS, (r.get("groups", []),))


def fingerprint(hashes):
    s = x = 0
    n = 0
    for h in hashes:
        s = (s + h) & M
        x ^= h
        n += 1
    return (s, x, n)


def queue_fingerprint(job_ids):
    return fingerprint(absorb(absorb(3, p), word(j)) for p, j in enumerate(job_ids))


def bucket(rid, n_buckets):
    return mix(word(rid)) & (n_buckets - 1)


def table_fingerprints(rows, hash_fn, n_buckets=0):
    """(fingerprint of the table, [fingerprint per bucket])."""
    hs = {rid: hash_fn(rid, r) for rid, r in rows.items()}
    per = [[] for _ in range(n_buckets)]
    for rid, h in hs.items():
        if n_buckets:
            per[bucket(rid, n_buckets)].append(h)
    return fingerprint(hs.values()), [fingerprint(b) for b in per]


def digest(pend, run, queue=(), n_buckets=0):
    """What GpuEngine.state_digest returns for these rows and this live queue (without the recount)."""
    p, pb = table_fingerprints(pend, pending_hash, n_buckets)
    r, rb = table_fingerprints(run, running_hash, n_buckets)
    return dict(pending=p, running=r, queue=queue_fingerprint(queue), pending_buckets=pb, running_buckets=rb,
                entries=[sum(len(x.get("novel", [])) for x in pend.values()), sum(len(x.get("attr", [])) for x in pend.values()),
                         sum(len(x.get("groups", [])) for x in pend.values()), sum(len(x.get("groups", [])) for x in run.values())])


def buckets_as_tuples(arr):
    """An abi.FP_DTYPE array as [(sum, xor, n)]."""
    return [(int(a["sum"]), int(a["xr"]), int(a["n"])) for a in arr]


def selected(rows, mask):
    """The ids of `rows` an export with bucket_mask `mask` (None: all) returns, in export order."""
    return sorted(i for i in rows if mask is None or mask[bucket(i, len(mask))])


def _csr(lists):
    off = np.zeros(len(lists) + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in lists])
    return off, np.array([e for x in lists for e in x], np.int32)


def export(pend, run, mask=None):
    """The arrays cook_state_export returns for these rows: {name: array}, pending_* then running_*."""
    pi, ri = selected(pend, mask), selected(run, mask)
    pr, rr = [pend[j] for j in pi], [run[t] for t in ri]
    dt = dict(user=np.int32, priority=np.int32, cpus=np.float64, mem=np.float64, gpus=np.float64, ports=np.int32,
              allowed=np.uint8, plugin_accept=np.uint8, gpu_model=np.int32, disk_request=np.float64, disk_type=np.int32,
              est_end_ms=np.int64, ckpt_location=np.int32, reserved_host=np.int32, start_time=np.int64, job_id=np.int64,
              host=np.int32)
    out = {"pending_job_id": np.array(pi, np.int64), "running_task_id": np.array(ri, np.int64)}
    for name, _ in PENDING_COLS:
        out["pending_" + name] = np.array([r.get(name, ABSENT.get(name)) for r in pr], dt[name])
    out["pending_novel_off"], out["pending_novel_host"] = _csr([r.get("novel", []) for r in pr])
    out["pending_attr_off"], out["pending_attr_col"] = _csr([[c for c, _ in r.get("attr", [])] for r in pr])
    out["pending_attr_val"] = _csr([[v for _, v in r.get("attr", [])] for r in pr])[1]
    out["pending_group_off"], out["pending_group_idx"] = _csr([r.get("groups", []) for r in pr])
    for name, _ in RUNNING_COLS:
        out["running_" + name] = np.array([r.get(name, -1 if name == "host" else 0) for r in rr], dt[name])
    out["running_group_off"], out["running_group_idx"] = _csr([r.get("groups", []) for r in rr])
    return out
