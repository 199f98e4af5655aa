"""cook_state_digest, cook_state_export and cook_state_queue: the read side of the resident pool state.

CPU: the hash pinned to constants computed by an independent C program, the struct layouts and prototypes against the
C compiler, the exports and the phase code, the properties of the fingerprint on the restatement
(state_digest_ref.py), the count comparison, and cycle.resync on model pairs through a model engine.
GPU (-m gpu): after every batch of a churn the digest equals the restatement, the recount is consistent and the full
export equals the model sorted by id, bit for bit; layout independence; the round trip into a fresh handle, then
rank, match and rebalance bit-identical; nothing resident moves; the live queue after every kind of step; a
divergence drill repaired by cycle.resync; the edges, errors and transfer formulas.
"""
import ctypes as C
import os

import numpy as np
import pytest

import state_digest_ref as R
from cook_b200 import abi, cycle, engine, traces
from cook_b200.engine import CookError, GpuEngine
from resident_model import OPTIONAL, START, pending_kw, pool_rows, rebalance_trace, rows_of, running_kw


# two pending and two running rows whose hashes an independent C program computed from the header's definition
PEND_A = dict(user=3, priority=50, cpus=1.5, mem=2048.0)
PEND_B = dict(user=0, priority=99, cpus=0.1, mem=64.0, gpus=2.0, ports=3, allowed=0, plugin_accept=1, gpu_model=4,
              disk_request=512.5, disk_type=2, est_end_ms=1700000000123, ckpt_location=6, reserved_host=11,
              novel=[5, 9], attr=[(0, 7), (2, -1)], groups=[4])
RUN_A = dict(user=2, priority=50, start_time=START, job_id=1001, cpus=4.0, mem=8192.0, gpus=-0.0)
RUN_B = dict(user=2, priority=50, start_time=START, job_id=1002, cpus=4.0, mem=8192.0, gpus=1.0, host=12, groups=[3, 1])


# ---- CPU ---------------------------------------------------------------------------------------------------
def test_hash_pinned():
    assert R.mix(0) == 0 and R.mix(1) == 0x5692161d100b05e5 and R.mix(R.M) == 0xb4d055fcf2cbbd7b
    assert R.absorb(1, 42) == 0xba69ec90eb4fef88 and R.absorb(0, R.word(-1)) == 0xe4d971771b652c20
    assert R.pending_hash(1001, PEND_A) == 0x2159e3c4e6a17f49
    assert R.pending_hash(-7, PEND_B) == 0xf8beff18fed24f69
    assert R.running_hash(77, RUN_A) == 0x68a1087bbc4e51bb
    assert R.running_hash(78, RUN_B) == 0x4def8e4ea95b9c01
    assert R.queue_fingerprint([1001, -7]) == (0x78510fc1fc93719c, 0x782c8fb9f34c8d5a, 2)
    assert R.queue_fingerprint([]) == (0, 0, 0)
    assert R.bucket(1001, 16) == 3 and R.bucket(-7, 65536) == 63219


def test_counts_compare():
    """The `consistent` comparison of cook_state_digest: a pure host function over two count vectors."""
    if not os.path.exists(engine.LIB_PATH):
        pytest.skip("libcookgpu.so not built")
    lib = engine.load_library()
    host = np.arange(abi.AUDIT_N, dtype=np.int64) - 1
    first = C.c_int32(99)
    p = lambda a: abi.ptr(a, abi.P_I64)
    assert lib.cook_state_counts_compare(p(host), p(host.copy()), C.byref(first)) == 0 and first.value == -1
    for k in range(abi.AUDIT_N):
        dev = host.copy()
        dev[k:] += 1                                       # the first difference is reported
        assert lib.cook_state_counts_compare(p(host), p(dev), C.byref(first)) == 0 and first.value == k
    first = C.c_int32(99)
    assert lib.cook_state_counts_compare(None, p(host), C.byref(first)) == abi.COOK_E_BADARG
    assert lib.cook_state_counts_compare(p(host), p(host), None) == abi.COOK_E_BADARG and first.value == 99
    assert len(abi.AUDIT_NAMES) == 24 and abi.AUDIT_NAMES[15] == "reserved_rows" and abi.AUDIT_NAMES[23] == "max_hostname_running"


def _model(rng, n_p=300, n_r=200):
    pend = {int(j): dict(user=int(rng.integers(9)), priority=int(rng.integers(100)), cpus=float(rng.choice([0.1, 1, 2.5])),
                         mem=float(rng.integers(1, 64) * 64), gpus=float(rng.choice([0, 0, 1])), ports=int(rng.integers(3)),
                         allowed=int(rng.random() < 0.9), plugin_accept=int(rng.random() < 0.9),
                         gpu_model=int(rng.integers(-1, 3)), disk_request=float(rng.choice([-1.0, 100.0])),
                         disk_type=int(rng.integers(-1, 2)), est_end_ms=int(rng.choice([-1, START + 5])),
                         ckpt_location=int(rng.integers(-1, 3)), reserved_host=int(rng.choice([-1, -1, 4, 9])),
                         novel=[int(x) for x in rng.integers(0, 50, int(rng.integers(0, 3)))],
                         attr=[(int(rng.integers(3)), int(rng.integers(-1, 9))) for _ in range(int(rng.integers(0, 3)))],
                         groups=[int(x) for x in rng.choice(20, int(rng.integers(0, 3)), replace=False)])
            for j in rng.choice(10 ** 6, n_p, replace=False) - 1000}
    run = {int(t): dict(user=int(rng.integers(9)), priority=50, start_time=START + int(t), task_id=int(t),
                        job_id=int(t) + 10 ** 7, cpus=1.0, mem=64.0, gpus=0.0, host=int(rng.integers(-1, 30)),
                        groups=[int(x) for x in rng.choice(20, int(rng.integers(0, 3)), replace=False)])
           for t in rng.choice(10 ** 6, n_r, replace=False)}
    return pend, run


def test_fingerprint_properties():
    rng = np.random.default_rng(1)
    pend, run = _model(rng)
    d = R.digest(pend, run, sorted(pend)[:50], 64)
    for t in ("pending", "running"):                            # the buckets add up to the table
        b = d[t + "_buckets"]
        assert (sum(x[0] for x in b) & R.M, int(np.bitwise_xor.reduce(np.array([x[1] for x in b], np.uint64))),
                sum(x[2] for x in b)) == d[t]
    perm = {j: pend[j] for j in rng.permutation(sorted(pend)).tolist()}
    assert R.digest(perm, run)["pending"] == d["pending"]       # row order does not count
    j = sorted(pend)[0]
    base = R.pending_hash(j, pend[j])
    changed = dict(user=7, priority=3, cpus=9.5, mem=1.0, gpus=0.5, ports=5, allowed=1 - pend[j]["allowed"],
                   plugin_accept=1 - pend[j]["plugin_accept"], gpu_model=7, disk_request=3.5, disk_type=5, est_end_ms=77,
                   ckpt_location=8, reserved_host=21, novel=pend[j]["novel"] + [1], attr=pend[j]["attr"] + [(1, 1)],
                   groups=pend[j]["groups"] + [19])
    seen = {base}
    for k, v in changed.items():                                # every single column and list
        h = R.pending_hash(j, dict(pend[j], **{k: v}))
        assert h not in seen, k
        seen.add(h)
    assert R.pending_hash(j + 1, pend[j]) != base
    t = sorted(run)[0]
    rbase = R.running_hash(t, run[t])
    for k, v in dict(user=8, priority=1, start_time=5, job_id=6, cpus=7.0, mem=8.0, gpus=9.0, host=77, groups=[1, 2, 3]).items():
        assert R.running_hash(t, dict(run[t], **{k: v})) != rbase, k
    row = dict(PEND_B)
    assert R.pending_hash(1, dict(row, novel=[9, 5])) != R.pending_hash(1, row)             # list order
    assert R.pending_hash(1, dict(row, attr=[(0, -1), (2, 7)])) != R.pending_hash(1, row)
    assert R.pending_hash(1, dict(row, gpus=-0.0)) != R.pending_hash(1, dict(row, gpus=0.0))   # the bits, not the value
    # a list entry moved between two rows, and between two lists of one row, changes the table's fingerprint
    a, b = dict(PEND_A, groups=[1, 2]), dict(PEND_A, groups=[3])
    a2, b2 = dict(PEND_A, groups=[1]), dict(PEND_A, groups=[2, 3])
    assert R.digest({1: a, 2: b}, {})["pending"] != R.digest({1: a2, 2: b2}, {})["pending"]
    assert R.pending_hash(1, dict(PEND_A, novel=[4])) != R.pending_hash(1, dict(PEND_A, groups=[4]))
    assert R.queue_fingerprint([1, 2, 3]) != R.queue_fingerprint([2, 1, 3])                # the queue is ordered
    ex = R.export(pend, run)
    assert ex["pending_job_id"].tolist() == sorted(pend) and ex["running_task_id"].tolist() == sorted(run)
    mask = np.zeros(16, np.uint8)
    mask[[2, 11]] = 1
    sel = R.export(pend, run, mask)["pending_job_id"].tolist()
    assert sel == [j for j in sorted(pend) if R.bucket(j, 16) in (2, 11)] and 0 < len(sel) < len(pend)


# ---- rows <-> deltas -------------------------------------------------------------------------------------------
def without(row, drop):
    """The row a delta stores when the columns and lists in `drop` are NULL."""
    row = dict(row)
    for c in drop:
        row[c] = [] if c in ("novel", "attr", "groups") else R.ABSENT[c]
    return row


def delta_of(pend_rows=None, run_rows=None, **kw):
    """The delta that holds exactly these rows (the keyword arguments of make_delta for the rest)."""
    a = dict(kw)
    if pend_rows:
        a.update(pending_kw(sorted(pend_rows.items())))
    if run_rows:
        a.update(running_kw([run_rows[t] for t in sorted(run_rows)]))
    return abi.make_delta(**a)


def flat(ex):
    """GpuEngine.state_export's result under state_digest_ref.export's names, lists cut to their length."""
    p, r = ex["pending"], ex["running"]
    out = {"pending_job_id": ex["pending_job_id"], "pending_priority": ex["pending_priority"],
           "running_task_id": r.col("task_id"), "running_host": ex["running_hostname_id"]}
    for name, _ in R.PENDING_COLS:
        if name != "priority":
            out["pending_" + name] = p.col(name)
    for off, vals in (("novel_off", ("novel_host",)), ("attr_off", ("attr_col", "attr_val")), ("group_off", ("group_idx",))):
        out["pending_" + off] = p.col(off)
        for v in vals:
            out["pending_" + v] = p.col(v)[:p.col(off)[-1]]
    for name, _ in R.RUNNING_COLS:
        if name != "host":
            out["running_" + name] = r.col(name)
    out["running_group_off"] = ex["running_group_off"]
    out["running_group_idx"] = ex["running_group_idx"][:ex["running_group_off"][-1]]
    return out


def same_arrays(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].tobytes() == want[k].tobytes(), k


ROW_BYTES_P, ROW_BYTES_R = 78, 60   # every data column of a pending / running row


def export_bytes(sizes, mask_len=0):
    """The header's transfer formula of a full-column export: (up, down)."""
    P, Rn, E = sizes
    down = 24 + (8 if mask_len else 0) + ROW_BYTES_P * P + ROW_BYTES_R * Rn
    down += 3 * 4 * (P + 1) + 4 * E[0] + 8 * E[1] + 4 * E[2] + 4 * (Rn + 1) + 4 * E[3]
    return mask_len, down


class Twin:
    """A resident handle and the model of what it should hold, with the live queue."""

    def __init__(self, name="audit"):
        self.e = GpuEngine(pool_name=name)
        self.pend, self.run, self.queue = {}, {}, []

    def close(self):
        self.e.close()

    def apply(self, up=(), rm=(), run_up=(), run_rm=(), reset=False, drop=(), hosts=True, lists=True, gpus=True):
        up = [(j, without(r, drop)) for j, r in up]
        run_up = [dict(r, host=r["host"] if hosts else -1, groups=r["groups"] if lists else [],
                       gpus=r["gpus"] if gpus else 0.0) for r in run_up]
        kw = {}
        if up:
            kw.update(pending_kw(up, drop))
        if run_up:
            kw.update(running_kw(run_up, hosts, lists, gpus))
        self.e.state_apply(abi.make_delta(reset=reset, pending_rm=list(rm), running_rm=list(run_rm), **kw))
        if reset:
            self.pend, self.run = {}, {}
        for j in rm:
            del self.pend[j]
        for t in run_rm:
            del self.run[t]
        self.pend.update(up)
        self.run.update({r["task_id"]: r for r in run_up})
        gone = set(rm) | {j for j, _ in up}
        self.queue = [] if reset else [j for j in self.queue if j not in gone]

    def launch(self, jobs, tids, hosts=None):
        self.e.state_launch(jobs, tids, np.full(len(jobs), START, np.int64), hosts)
        for i, (j, t) in enumerate(zip(jobs, tids)):
            p = self.pend.pop(j)
            self.run[t] = dict(user=p["user"], priority=p["priority"], start_time=START, task_id=t, job_id=j,
                               cpus=p["cpus"], mem=p["mem"], gpus=p["gpus"],
                               host=int(hosts[i]) if hosts is not None else -1, groups=list(p["groups"]))
        self.queue = [j for j in self.queue if j not in set(jobs)]

    def patch(self, jobs, clear=False, **cols):
        self.e.state_patch(jobs, clear_reservations=clear, **cols)
        if clear:
            for r in self.pend.values():
                r["reserved_host"] = -1
        for name, vals in cols.items():
            for j, v in zip(jobs, vals):
                self.pend[j][name] = int(v)

    def rank(self, users):
        self.queue = self.e.state_rank(users).tolist()
        return self.queue

    def check(self, n_buckets=16):
        """The digest, the recount, the queue and the full export against the model, with their transfers."""
        d = self.e.state_digest(n_buckets)
        st = self.e.last_stats(abi.PHASE_AUDIT)
        live = len(self.pend) + len(self.run) > 0
        assert (st["h2d_bytes"], st["d2h_bytes"]) == ((0, 72 + 8 * abi.AUDIT_N + 48 * n_buckets) if live else (0, 0))
        assert (st["n_launches"] > 0) == live
        want = R.digest(self.pend, self.run, self.queue, n_buckets)
        assert d["consistent"] and d["first_mismatch"] is None
        for k in ("pending", "running", "queue", "entries"):
            assert d[k] == want[k], k
        for t in ("pending_buckets", "running_buckets"):
            assert R.buckets_as_tuples(d[t]) == want[t], t
        ex = self.e.state_export()
        st = self.e.last_stats(abi.PHASE_AUDIT)
        sizes = (len(self.pend), len(self.run), want["entries"])
        assert (st["h2d_bytes"], st["d2h_bytes"]) == (export_bytes(sizes) if live else (0, 0))
        same_arrays(flat(ex), R.export(self.pend, self.run))
        return d, ex


class ModelEngine:
    """cycle.resync's view of an engine, over a model: state_digest's buckets and state_export with a mask."""

    def __init__(self, pend, run):
        self.pend, self.run = pend, run

    def state_digest(self, nb):
        d = R.digest(self.pend, self.run, (), nb)
        return {t: np.array(d[t], abi.FP_DTYPE) for t in ("pending_buckets", "running_buckets")}

    def state_export(self, mask):
        pi, ri = R.selected(self.pend, mask), R.selected(self.run, mask)
        kw = dict(pending_job_id=np.array(pi, np.int64), running=abi.TasksSoA(n=0))
        if ri:
            kw.update(running_kw([self.run[t] for t in ri]))
        return kw

    def state_apply(self, d, rows):
        """The delta's removals, then `rows` (the model rows the delta upserts)."""
        for j in (d.col("pending_rm_job_id").tolist() if d.n_pending_rm else []):
            del self.pend[j]
        for t in (d.col("running_rm_task_id").tolist() if d.n_running_rm else []):
            del self.run[t]
        self.pend.update(rows[0])
        self.run.update(rows[1])


def host_side(pend, run, nb):
    """What a host computes from its own rows for cycle.resync: its bucket fingerprints and its rows of given buckets."""
    d = R.digest(pend, run, (), nb)
    fps = dict(pending=d["pending_buckets"], running=d["running_buckets"])
    picked = {}

    def rows_of_bucket(buckets):
        p = {j: r for j, r in pend.items() if R.bucket(j, nb) in buckets}
        r = {t: x for t, x in run.items() if R.bucket(t, nb) in buckets}
        picked["rows"] = (p, r)
        kw = {}
        if p:
            kw.update(pending_kw(sorted(p.items())))
        if r:
            kw.update(running_kw([r[t] for t in sorted(r)]))
        return kw
    return fps, rows_of_bucket, picked


def test_resync_on_models():
    rng = np.random.default_rng(2)
    pend, run = _model(rng)
    nb = 32
    fps, rows_of_bucket, picked = host_side(pend, run, nb)
    assert cycle.resync(ModelEngine(dict(pend), dict(run)), fps, rows_of_bucket) == ([], None)
    ids, tids = sorted(pend), sorted(run)
    dp, dr = dict(pend), dict(run)
    del dp[ids[0]], dr[tids[0]]                                            # missing on the device
    dp[10 ** 8] = dict(pend[ids[1]])                                       # extra rows the host does not have
    dr[10 ** 8 + 1] = dict(run[tids[1]], task_id=10 ** 8 + 1)
    dp[ids[2]] = dict(pend[ids[2]], mem=pend[ids[2]]["mem"] + 1)           # altered
    dr[tids[2]] = dict(run[tids[2]], host=run[tids[2]]["host"] + 1)
    touched = {R.bucket(i, nb) for i in (ids[0], tids[0], 10 ** 8, 10 ** 8 + 1, ids[2], tids[2])}
    dev = ModelEngine(dp, dr)
    buckets, delta = cycle.resync(dev, fps, rows_of_bucket)
    assert buckets == sorted(touched)
    assert delta.col("pending_rm_job_id").tolist() == [10 ** 8] and delta.col("running_rm_task_id").tolist() == [10 ** 8 + 1]
    assert set(delta.col("pending_job_id").tolist()) == {j for j in pend if R.bucket(j, nb) in touched}
    dev.state_apply(delta, picked["rows"])
    assert dev.pend == pend and dev.run == run
    assert cycle.resync(dev, fps, rows_of_bucket) == ([], None)
    with pytest.raises(ValueError):
        cycle.resync(dev, dict(pending=fps["pending"][:3], running=fps["running"][:3]), rows_of_bucket)


# ---- GPU: churn ------------------------------------------------------------------------------------------------
def c3_rows(seed, n_jobs=1500, n_running=500, rng=None):
    """A config-#3 pool as model rows: every pending column and list in use, amounts on and off the 2^-10 grid,
    running rows with hosts and group lists."""
    t = traces.gen_c3_pool(seed, n_jobs=n_jobs, n_offers=160, n_users=24, n_running=n_running)
    rng = rng or np.random.default_rng(seed)
    pend, run = pool_rows(t)
    G, hn = t["groups"].n_groups, t["offers"].col("hostname_id")
    for i, r in enumerate(pend.values()):
        if i % 7 == 0:
            r["cpus"] = 0.1 * (1 + i % 5)                                   # off the grid
        if i % 11 == 0:
            r["reserved_host"], r["ckpt_location"] = int(hn[i % len(hn)]), i % 3
    for r in run.values():
        r["host"] = int(hn[rng.integers(len(hn))]) if rng.random() < 0.9 else -1
        r["groups"] = [int(g) for g in rng.choice(G, int(rng.choice([0, 0, 1, 2])), replace=False)]
        if rng.random() < 0.1:
            r["cpus"] = 0.3
    return t, pend, run


@pytest.mark.gpu
def test_churn_digest_and_export():
    rng = np.random.default_rng(31)
    t, pend, run = c3_rows(31, 2600, 700, rng)
    users = t["users"]
    items, tasks = sorted(pend.items()), list(run.values())
    reserve, spare = items[1200:], tasks[400:]
    drops = [(), ("gpus", "ports"), ("allowed", "plugin_accept", "novel"), ("gpu_model", "disk_request", "disk_type", "attr"),
             ("est_end_ms", "ckpt_location", "reserved_host", "groups"), OPTIONAL + ("novel", "attr", "groups")]
    h = Twin()
    tid = 10 ** 9
    try:
        h.check()                                                        # no state yet
        h.apply(up=items[:1200], run_up=tasks[:400])                     # past 1024 pending slots
        h.check()
        for b in range(6):
            h.rank(users)
            live = sorted(h.pend)
            fin = [x for x in h.run if rng.random() < 0.1]
            kill = [int(j) for j in rng.choice(live, 40, replace=False)]
            again = [(int(j), dict(h.pend[int(j)], priority=int(rng.integers(100)), mem=h.pend[int(j)]["mem"] + 64.0))
                     for j in rng.choice([j for j in live if j not in set(kill)], 30, replace=False)]   # replacements
            new = [reserve.pop() for _ in range(min(len(reserve), 150))]
            more = [spare.pop() for _ in range(min(len(spare), 40))]
            h.apply(up=new + again, rm=kill, run_up=more, run_rm=fin, drop=drops[b], hosts=b % 2 == 0,
                    lists=b % 3 != 1, gpus=b % 2 == 1)
            h.check(n_buckets=[0, 1, 16, 2048, 16, 65536][b])
            jobs = [int(j) for j in rng.choice(sorted(h.pend), 100, replace=False)]
            tids = [tid + 3 * i for i in range(len(jobs))]
            tid += 3 * len(jobs) + 3
            h.launch(jobs, tids, np.array(rng.integers(0, 160, len(jobs)), np.int32) if b % 2 else None)
            h.check()
            some = [int(j) for j in rng.choice(sorted(h.pend), 50, replace=False)]
            h.patch(some, clear=b % 2 == 0, allowed=rng.integers(0, 2, 50).astype(np.uint8),
                    reserved_host=rng.integers(-1, 40, 50).astype(np.int32))
            h.patch(some[:10], plugin_accept=np.zeros(10, np.uint8))
            h.check()
        h.apply(rm=[j for j in h.pend if rng.random() < 0.8], run_rm=[x for x in h.run if rng.random() < 0.8])
        h.check()                                                        # dead entries outnumber live: compaction
        h.apply(up=[reserve.pop() for _ in range(300)], run_up=[spare.pop() for _ in range(min(len(spare), 100))])
        h.check()                                                        # the freed slots are taken again
        h.rank(users)
        h.apply(reset=True, up=items[:500], run_up=tasks[:300])
        h.check()
        h.apply(rm=list(h.pend), run_rm=list(h.run))
        h.check()                                                        # nothing live
    finally:
        h.close()


@pytest.mark.gpu
def test_layout_independence():
    """The same rows reached by one batch in id order, or after junk rows whose freed slots the real rows take in a
    permuted order over two batches: equal digests and exports."""
    rng = np.random.default_rng(37)
    _, pend, run = c3_rows(37, 1800, 600, rng)
    _, junk_p, junk_r = c3_rows(38, 900, 300)
    junk_p = {j + 10 ** 8: r for j, r in junk_p.items()}
    junk_r = {x + 10 ** 8: dict(r, task_id=x + 10 ** 8) for x, r in junk_r.items()}
    a, b = Twin("a"), Twin("b")
    try:
        a.apply(up=sorted(pend.items()), run_up=[run[x] for x in sorted(run)])
        b.apply(up=list(junk_p.items()), run_up=list(junk_r.values()))
        pp = [list(pend.items())[i] for i in rng.permutation(len(pend))]
        rp = [list(run.values())[i] for i in rng.permutation(len(run))]
        jp, jr = list(junk_p), list(junk_r)
        b.apply(up=pp[:800], rm=jp[:600], run_up=rp[:250], run_rm=jr[:200])
        b.apply(up=pp[800:], rm=jp[600:], run_up=rp[250:], run_rm=jr[200:])
        (da, ea), (db, eb) = a.check(256), b.check(256)
        for k in ("pending", "running", "queue", "entries"):
            assert da[k] == db[k]
        assert da["pending_buckets"].tobytes() == db["pending_buckets"].tobytes()
        assert da["running_buckets"].tobytes() == db["running_buckets"].tobytes()
        same_arrays(flat(ea), flat(eb))
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_round_trip_rank_match_rebalance():
    """export -> a reset delta on a fresh handle -> equal digest; then rank and a config-#3 match with groups, and a
    config-#4 rebalance, bit-identical on the two handles."""
    t, pend, run = c3_rows(41)
    a, b = Twin("orig"), Twin("copy")
    try:
        a.apply(up=sorted(pend.items()), run_up=list(run.values()))
        a.apply(rm=sorted(pend)[::3], run_rm=sorted(run)[::4])                  # holes in the tables and arenas
        b.e.state_apply(abi.make_delta(reset=True, **a.e.state_export()))
        b.pend, b.run = dict(a.pend), dict(a.run)
        da, _ = a.check(64)
        db, _ = b.check(64)
        assert da["pending"] == db["pending"] and da["running"] == db["running"]
        users, offers = t["users"], t["offers"]
        assert a.rank(users) == b.rank(users) and len(a.queue) > 500
        prm = traces.match_params(600, host_lifetime_mins=t.get("host_lifetime_mins", 0))
        mp = int(t["jobs"].col("ports").max())
        ma, mb = (x.e.state_match(offers, users, prm, groups=t["groups"], max_ports=mp) for x in (a, b))
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
        assert (ma["assign"] >= 0).any()
        r, codes = rebalance_trace(23, True)
        rp, rr = rows_of(r, codes)
        a.apply(reset=True, up=[(j, dict(R.ABSENT, **x)) for j, x in sorted(rp.items())],
                run_up=[dict(x, groups=[]) for x in rr.values()])
        b.e.state_apply(abi.make_delta(reset=True, **a.e.state_export()))
        b.pend, b.run = dict(a.pend), dict(a.run)
        assert a.rank(r["users"]) == b.rank(r["users"])
        assert a.check()[0]["queue"] == b.check()[0]["queue"]
        ra, rb = (x.e.state_rebalance(r["hosts"], r["users"], r["params"], groups=r["groups"]) for x in (a, b))
        assert ra == rb
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_nothing_resident_moves():
    """A rank, then digest + export + queue, then the match and its failure counts: what a twin without the audit calls
    gives, COOK_PHASE_MATCH's counters and COOK_USAGE_LAST_MATCH included."""
    t, pend, run = c3_rows(47)
    users, offers = t["users"], t["offers"]
    prm = traces.match_params(500, host_lifetime_mins=t.get("host_lifetime_mins", 0))
    mp = int(t["jobs"].col("ports").max())
    a, b = Twin("audited"), Twin("plain")
    cons = abi.ConsiderableParams(400, 0, 1, abi.USAGE_LAST_MATCH, 0)
    try:
        for x in (a, b):
            x.apply(up=sorted(pend.items()), run_up=list(run.values()))
            x.rank(users)
            x.apply(rm=sorted(pend)[:40])
        mask = np.zeros(8, np.uint8)
        mask[3] = 1

        def audit():
            a.check(128)
            a.e.state_export(mask)
            assert a.e.state_queue().tolist() == a.queue

        audit()
        ma, mb = (x.e.state_match(offers, users, prm, groups=t["groups"], max_ports=mp) for x in (a, b))
        sa, sb = a.e.last_stats(abi.PHASE_MATCH), b.e.last_stats(abi.PHASE_MATCH)
        audit()                                                           # between the match and its readers
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(ma[k], mb[k]), k
        assert {k: sa[k] for k in ("h2d_bytes", "d2h_bytes", "n_launches")} == {k: sb[k] for k in ("h2d_bytes", "d2h_bytes", "n_launches")}
        assert a.e.last_stats(abi.PHASE_MATCH) == sa
        k = np.arange(0, len(ma["considerable"]), 7, dtype=np.int32)
        assert a.e.match_failures(k) == b.e.match_failures(k)
        assert np.array_equal(a.e.exchange_usage(users.n_users), b.e.exchange_usage(users.n_users))
        ca, cb = (x.e.state_considerable(users, cons) for x in (a, b))
        assert np.array_equal(ca, cb)
        audit()
        assert np.array_equal(a.e.state_match(offers, users, prm, groups=t["groups"], max_ports=mp)["assign"], ma["assign"])
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_queue_after_every_step():
    t, pend, run = c3_rows(53, 1200, 200)
    users = abi.make_users(t["users"].n_users)                        # no quota: the rank keeps every job
    h = Twin()
    try:
        h.apply(up=sorted(pend.items()), run_up=list(run.values()))
        with pytest.raises(CookError):
            h.e.state_queue()                                             # no rank yet
        assert h.e.state_digest()["queue"] == (0, 0, 0)
        q = h.rank(users)
        assert h.e.state_queue().tolist() == q and len(q) == len(pend)
        assert h.e.last_stats(abi.PHASE_AUDIT)["d2h_bytes"] == 4 + 8 * len(q)
        h.launch(q[5:40], list(range(10 ** 6, 10 ** 6 + 35)))
        assert h.e.state_queue().tolist() == h.queue
        h.apply(rm=q[100:130])                                            # removed
        h.apply(up=[(j, dict(h.pend[j], priority=1)) for j in q[200:220]])   # replaced
        assert h.e.state_queue().tolist() == h.queue and len(h.queue) == len(q) - 35 - 30 - 20
        h.patch(h.queue[:10], allowed=np.zeros(10, np.uint8))             # a patch keeps the entry
        assert h.e.state_queue().tolist() == h.queue
        took = h.e.state_considerable(users, abi.ConsiderableParams(25, 0, 0, abi.USAGE_DERIVED, 1)).tolist()
        assert len(took) == 25
        h.queue = [j for j in h.queue if j not in set(took)]              # consumed
        assert h.e.state_queue().tolist() == h.queue
        d, _ = h.check()
        assert d["queue"] == R.queue_fingerprint(h.queue) and d["queue"][2] == len(h.queue)
        # a match that considers everything, with no filter binding, reads exactly this queue
        h.patch(sorted(h.pend), allowed=np.ones(len(h.pend), np.uint8), plugin_accept=np.ones(len(h.pend), np.uint8))
        m = h.e.state_match(t["offers"], users, traces.match_params(len(h.queue) + 5),
                            groups=t["groups"], max_ports=int(t["jobs"].col("ports").max()))
        assert m["considerable"].tolist() == h.queue
        n = C.c_int32(-5)
        out = np.full(len(h.queue), -9, np.int64)
        lib, pool = h.e.lib, h.e.pool
        assert lib.cook_state_queue(pool, 0, None, C.byref(n)) == 0 and n.value == len(h.queue)
        assert h.e.last_stats(abi.PHASE_AUDIT)["d2h_bytes"] == 4          # the size query
        n = C.c_int32(-5)
        assert lib.cook_state_queue(pool, len(h.queue) - 1, abi.ptr(out, abi.P_I64), C.byref(n)) == abi.COOK_E_BADARG
        assert lib.cook_state_queue(pool, len(h.queue), abi.ptr(out, abi.P_I64), None) == abi.COOK_E_BADARG
        assert n.value == -5 and (out == -9).all()
        assert lib.cook_state_queue(pool, len(h.queue), abi.ptr(out, abi.P_I64), C.byref(n)) == 0    # exactly at capacity
        assert out.tolist() == h.queue
        h.apply(rm=list(h.pend))
        assert h.e.state_queue().tolist() == [] and h.e.state_digest()["queue"] == (0, 0, 0)
    finally:
        h.close()


@pytest.mark.gpu
def test_divergence_drill():
    """A twin fed the same stream with one batch altered: the bucket fingerprints differ in exactly the buckets of the
    touched ids, the masked export returns exactly those buckets' rows, and cycle.resync's delta repairs the twin."""
    rng = np.random.default_rng(59)
    _, pend, run = c3_rows(59, 2000, 600, rng)
    nb = 256
    items, tasks = sorted(pend.items()), [run[x] for x in sorted(run)]
    good, bad = Twin("good"), Twin("bad")
    try:
        for x in (good, bad):
            x.apply(up=items[:1500], run_up=tasks[:400])
        batch_p, batch_r = items[1500:], tasks[400:]
        kill, fin = [j for j, _ in items[:60]], [r["task_id"] for r in tasks[:30]]
        good.apply(up=batch_p, run_up=batch_r, rm=kill, run_rm=fin)
        dropped, changed, skipped, rdrop = batch_p[7][0], batch_p[11][0], kill[3], batch_r[5]["task_id"]
        altered = [(j, dict(r, mem=r["mem"] + 1.0) if j == changed else r) for j, r in batch_p if j != dropped]
        bad.apply(up=altered, run_up=[r for r in batch_r if r["task_id"] != rdrop], rm=[j for j in kill if j != skipped],
                  run_rm=fin)
        dg, db = good.e.state_digest(nb), bad.e.state_digest(nb)
        assert dg["pending"] != db["pending"] and dg["running"] != db["running"] and db["consistent"]
        diff = lambda k: set(np.nonzero([x.tobytes() != y.tobytes() for x, y in zip(dg[k], db[k])])[0].tolist())
        assert diff("pending_buckets") == {R.bucket(j, nb) for j in (dropped, changed, skipped)}
        assert diff("running_buckets") == {R.bucket(rdrop, nb)}
        buckets = sorted(diff("pending_buckets") | diff("running_buckets"))
        mask = np.zeros(nb, np.uint8)
        mask[buckets] = 1
        ex = bad.e.state_export(mask)
        st = bad.e.last_stats(abi.PHASE_AUDIT)
        want = R.export(bad.pend, bad.run, mask)
        same_arrays(flat(ex), want)
        sizes = (len(want["pending_job_id"]), len(want["running_task_id"]),
                 [len(want[k]) for k in ("pending_novel_host", "pending_attr_col", "pending_group_idx", "running_group_idx")])
        assert (st["h2d_bytes"], st["d2h_bytes"]) == export_bytes(sizes, nb) and 0 < sizes[0] < 200
        fps, rows_of_bucket, _ = host_side(good.pend, good.run, nb)
        got, delta = cycle.resync(bad.e, fps, rows_of_bucket)
        assert got == buckets
        bad.e.state_apply(delta)
        bad.pend, bad.run = dict(good.pend), dict(good.run)
        d2, _ = bad.check(nb)
        for k in ("pending", "running"):
            assert d2[k] == dg[k]
        assert cycle.resync(bad.e, fps, rows_of_bucket) == ([], None)
    finally:
        good.close()
        bad.close()


# ---- GPU: edges, errors ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edges():
    h = Twin()
    try:
        d, ex = h.check(4)                                                 # no state
        assert d["pending"] == (0, 0, 0) and ex["pending"].n == 0 and ex["running_group_off"].tolist() == [0]
        assert h.e.last_stats(abi.PHASE_AUDIT) == dict(ms_h2d=0.0, ms_device=0.0, ms_d2h=0.0, h2d_bytes=0, d2h_bytes=0, n_launches=0)
        only_lists = dict(R.ABSENT, user=0, priority=50, cpus=0.0, mem=0.0, novel=[3, 1, 2], attr=[(1, 5)], groups=[2, 0])
        h.apply(up=[(5, only_lists)])                                      # one row, nothing but lists
        d, _ = h.check(1)
        assert d["pending"] == (R.pending_hash(5, only_lists),) * 2 + (1,) and d["entries"] == [3, 1, 2, 0]
        long_row = dict(only_lists, novel=list(range(100, 171)), attr=[(i % 3, i) for i in range(40)], groups=list(range(33)))
        h.apply(up=[(6, long_row)], run_up=[dict(RUN_B, task_id=78, groups=list(range(50, 0, -1)))])   # lists the warp reads
        h.check(65536)
        h.check(1)
        none = np.zeros(65536, np.uint8)
        ex = h.e.state_export(none)                                        # a mask that selects nothing
        assert ex["pending"].n == 0 and ex["running"].n == 0 and ex["pending"].col("attr_off").tolist() == [0]
        st = h.e.last_stats(abi.PHASE_AUDIT)
        assert (st["h2d_bytes"], st["d2h_bytes"]) == export_bytes((0, 0, [0, 0, 0, 0]), 65536)
        lib, pool = h.e.lib, h.e.pool
        n = abi.StateSizes()
        assert lib.cook_state_export(pool, 65536, abi.ptr(none, abi.P_U8), None, None, C.byref(n)) == 0
        assert (n.pending, n.running, list(n.entries)) == (0, 0, [0, 0, 0, 0])
        assert h.e.last_stats(abi.PHASE_AUDIT)["d2h_bytes"] == 32          # the count pass of a masked size query
        assert lib.cook_state_export(pool, 0, None, None, None, C.byref(n)) == 0
        assert (n.pending, n.running, list(n.entries)) == (2, 1, [74, 41, 35, 50])
        assert h.e.last_stats(abi.PHASE_AUDIT)["n_launches"] == 0          # from the host-side counts
        # only some columns: the job ids and the group lists, at exactly the required capacity
        jid, goff, gidx = np.full(2, -9, np.int64), np.full(3, -9, np.int32), np.full(35, -9, np.int32)
        rows = abi.StateRows(pending=abi.JobsRows(group_off=goff, group_idx=gidx), pending_job_id=jid)
        cap = abi.StateSizes(2, 1, (C.c_int32 * 4)(0, 0, 35, 0))
        assert lib.cook_state_export(pool, 0, None, C.byref(cap), C.byref(rows), C.byref(n)) == 0
        assert jid.tolist() == [5, 6] and goff.tolist() == [0, 2, 35] and gidx.tolist() == [2, 0] + list(range(33))
        assert h.e.last_stats(abi.PHASE_AUDIT)["d2h_bytes"] == 24 + 8 * 2 + 4 * 3 + 4 * 35
    finally:
        h.close()


@pytest.mark.gpu
def test_errors_write_nothing():
    rng = np.random.default_rng(61)
    _, pend, run = c3_rows(61, 400, 100, rng)
    h = Twin()
    try:
        h.apply(up=sorted(pend.items()), run_up=list(run.values()))
        want, _ = h.check(16)
        lib, pool = h.e.lib, h.e.pool
        fp = C.POINTER(abi.Fp)
        out = abi.StateDigest()
        C.memset(C.addressof(out), 0x5a, C.sizeof(out))
        pb, rb = np.full(16, 7, abi.FP_DTYPE), np.full(16, 7, abi.FP_DTYPE)
        P, Rb = pb.ctypes.data_as(fp), rb.ctypes.data_as(fp)
        cases = [lib.cook_state_digest(pool, 0, None, None, None), lib.cook_state_digest(pool, -2, C.byref(out), P, Rb),
                 lib.cook_state_digest(pool, 12, C.byref(out), P, Rb), lib.cook_state_digest(pool, 131072, C.byref(out), P, Rb),
                 lib.cook_state_digest(pool, 0, C.byref(out), P, None), lib.cook_state_digest(pool, 16, C.byref(out), P, None),
                 lib.cook_state_digest(pool, 16, C.byref(out), None, Rb)]
        assert cases == [abi.COOK_E_BADARG] * len(cases)
        assert bytes(out) == b"\x5a" * C.sizeof(out) and (pb["n"] == 7).all() and (rb["sum"] == 7).all()
        n = abi.StateSizes(-3, -3, (C.c_int32 * 4)(-3, -3, -3, -3))
        P_, R_ = len(h.pend), len(h.run)
        E = want["entries"]
        jid, goff, gidx = np.full(P_, -9, np.int64), np.full(P_ + 1, -9, np.int32), np.full(max(E[2], 1), -9, np.int32)
        rows = abi.StateRows(pending=abi.JobsRows(group_off=goff, group_idx=gidx), pending_job_id=jid)
        no_vals = abi.StateRows(pending=abi.JobsRows(attr_off=goff, attr_col=gidx))
        ok = abi.StateSizes(P_, R_, (C.c_int32 * 4)(*E))
        short_rows = abi.StateSizes(P_ - 1, R_, (C.c_int32 * 4)(*E))
        short_list = abi.StateSizes(P_, R_, (C.c_int32 * 4)(E[0], E[1], E[2] - 1, E[3]))
        mask = np.ones(16, np.uint8)
        M_ = abi.ptr(mask, abi.P_U8)
        cases = [lib.cook_state_export(pool, 0, None, C.byref(ok), C.byref(rows), None),
                 lib.cook_state_export(pool, 0, None, None, C.byref(rows), C.byref(n)),
                 lib.cook_state_export(pool, 24, M_, C.byref(ok), C.byref(rows), C.byref(n)),
                 lib.cook_state_export(pool, 0, M_, C.byref(ok), C.byref(rows), C.byref(n)),
                 lib.cook_state_export(pool, 0, None, C.byref(ok), C.byref(no_vals), C.byref(n)),
                 lib.cook_state_export(pool, 0, None, C.byref(short_rows), C.byref(rows), C.byref(n)),
                 lib.cook_state_export(pool, 0, None, C.byref(short_list), C.byref(rows), C.byref(n)),
                 lib.cook_state_export(pool, 16, M_, C.byref(short_rows), C.byref(rows), C.byref(n)),
                 lib.cook_state_export(pool, 16, M_, C.byref(short_list), C.byref(rows), C.byref(n))]
        assert cases == [abi.COOK_E_BADARG] * len(cases)
        assert (n.pending, n.running, list(n.entries)) == (-3, -3, [-3] * 4)
        assert (jid == -9).all() and (goff == -9).all() and (gidx == -9).all()
        assert lib.cook_state_export(pool, 16, M_, C.byref(ok), C.byref(rows), C.byref(n)) == 0
        assert jid.tolist() == sorted(h.pend) and n.pending == P_
        for bad_phase in (-1, 9):
            assert lib.cook_last_stats(pool, bad_phase, C.byref(abi.PhaseStats())) == abi.COOK_E_BADARG
        got, _ = h.check(16)                                               # the handle is unchanged
        assert got["pending"] == want["pending"] and got["running"] == want["running"]
    finally:
        h.close()
