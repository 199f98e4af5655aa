"""Steady-state cycles on the resident pool state (cook_state_*) against cook_rank + cook_match on host tables.

Each cycle applies one realistic batch to the resident handle: the jobs the previous match placed are launched
(pending -> running), a few percent of the running tasks finish, as many new jobs are submitted, and a few
priorities change.  Then both arms rank and match the same rows: the resident arm from the device tables, the
host arm from dense host tables built from the same state.  Per cycle and arm it prints the device time per
phase (CUDA events), the host wall time of the library calls, the bytes uploaded, and whether the outputs are
identical.  The host arm's wall time excludes building its tables in Python.

  python tools/prof_state.py --pool c2 --cycles 8
  python tools/prof_state.py --pool c5 --c5-pool 5 --cycles 5      # the config-#5 pool of ~640 k jobs

--rebalance instead loads a config-#4 pool's rebalancer input (running tasks on their hosts, pending jobs) into a
resident handle, ranks it, and per cycle runs cook_state_rebalance against cook_rebalance on host tables holding
the same rows (the queue's first max_preemption jobs): device time, wall time, bytes uploaded, identical outputs.

  python tools/prof_state.py --rebalance --c4-pool 0 --cycles 5

--offers feeds one offer stream (40 % of the hosts offer each cycle, some in two or three leases, 15 s incubation)
to two resident handles holding the same rows: one keeps the offers itself (cook_state_offers_add, then
cook_state_match_offers), the other gets the host's lease cache (cycle.OfferCache, offers_from_cache, then
cook_state_match_derived).  Per cycle it prints each arm's wall time, device time and bytes, and whether the
placements are identical.

  python tools/prof_state.py --offers --cycles 8
  python tools/prof_state.py --offers --c3-pool 0 --cycles 6

--sweeps loads a running table (C2's, or config-#5 pool --c5-pool with --pool c5) into a resident handle, gives
about 20 % of its rows group lists, a few thousand successful runtimes, max-runtimes, cancelled and unknown facts,
and times cook_state_sweep per list and for all three against a numpy restatement over a host mirror of the same
rows (median of --reps calls): device time, wall time, bytes, launches, and whether the lists are identical.

  python tools/prof_state.py --sweeps --pool c2 --reps 30
  python tools/prof_state.py --sweeps --pool c5 --c5-pool 5 --reps 30
--user-usage loads C2, config-#5 pool --c5-pool, or (--c3-group N) config-#3 pools 0 .. N-1 as N handles, on the grid and
off it, and times cook_state_user_usage for the lightest user, the heaviest user and every user, with and without
groups, against numpy over a host mirror:
  python tools/prof_state.py --user-usage --pool c5 --reps 10
--instance-stats loads C2, config-#5 pool --c5-pool, or (--c3-group N) config-#3 pools 0 .. N-1 as N handles, a tenth
of the rows with a reason and a twentieth unknown, and times cook_state_instance_stats for status running and unknown
over a window covering every row, against numpy over a host mirror:
  python tools/prof_state.py --instance-stats --pool c5 --reps 10
--history-stats seeds finished-instance histories over 31 days (--history-rows rows, C2's users and shapes on one
handle, or with --c3-group N config-#3 pools' shapes as N handles) and times cook_state_history_stats for success and
failed over a window covering every row and over the last day, against numpy over a host mirror; then a batch of 1000
finishes through cook_state_finish_history against cook_state_finish, one advance dropping a day, and the device
memory of the table and of the call's scratch:
  python tools/prof_state.py --history-stats --history-rows 1000000 --reps 5
  python tools/prof_state.py --history-stats --history-rows 10000000 --c3-group 4 --reps 3
--match-metrics loads C2 (or config-#5 pool --c5-pool with --pool c5) into a resident handle with every pending job
considerable, gives a tenth of the jobs a gpus fact and a tenth disk facts, and times cook_state_match_metrics after
each match (a tenth of the matches dropped) against the numpy and Python restatement over a host mirror (sorts, folds,
the dict of counters), with the answers compared bit for bit:
  python tools/prof_state.py --match-metrics --pool c2 --reps 10
  python tools/prof_state.py --match-metrics --pool c5 --c5-pool 5 --reps 10
--unscheduled loads C2 (or config-#5 pool --c5-pool with --pool c5) into a resident handle, on the grid and off it,
and times cook_state_unscheduled for one job, 1000 jobs and every waiting job of the user with the most, against numpy
over a host mirror, with the answers compared bit for bit:
  python tools/prof_state.py --unscheduled --pool c2 --reps 20
--status loads C2 (or config-#5 pool --c5-pool with --pool c5) into two resident handles, gives every job of one retry
facts, and per rep launches --status-batch jobs on both (timing cook_state_launch with and without facts), then fails
them: cook_state_status (every job parked, so every one is requeued on the device) against the host path it replaces,
the requeued rows rebuilt from a host mirror, cook_state_finish_history and a cook_state_apply upsert, alternated,
with the two handles' digests compared after every rep:
  python tools/prof_state.py --status --pool c2 --reps 10
  python tools/prof_state.py --status --pool c5 --c5-pool 5 --reps 10

--list loads C2 (or config-#5 pool --c5-pool with --pool c5) into a resident handle, gives every job list facts (a
submit time in one day, no submit pool, no custom executor), and times cook_state_list_jobs for the user with the
most rows and one with the fewest, both states, a 24 h window covering every row, limits Integer/MAX_VALUE and 150,
against numpy over a host mirror, with the answers compared exactly:
  python tools/prof_state.py --list --pool c2 --reps 20
  python tools/prof_state.py --list --pool c5 --c5-pool 5 --reps 20

--list-completed builds one handle's completed-job log of --completed-rows records over 32 days (Zipf users as in
traces.py, reopens, second completions and records sent twice) and times cook_state_list_completed for the heaviest
user and a light one, 24 h and 7 d windows, limits Integer/MAX_VALUE and 150, states completed and success, against
numpy over a host mirror with the answers compared exactly; then one cook_state_completed_record of 1000 rows and one
cook_state_completed_advance that drops a day:
  python tools/prof_state.py --list-completed --reps 10

--launch runs the same cycles on two resident handles instead of the host arm.  Each cycle's launches go to one
handle through cook_state_launch (job ids, task ids, start times, the hosts the match chose) and to its twin through
the equivalent cook_state_apply batch (the jobs' removal plus their task rows); the rest of the batch goes to both
as one delta.  Per cycle and arm it prints the launch call's bytes uploaded, device time and host wall time around
the (synchronising) binding call, and whether the following rank and match outputs of the two handles are identical.

  python tools/prof_state.py --launch --pool c2 --cycles 6
  python tools/prof_state.py --launch --pool c5 --c5-pool 5 --cycles 4

--usage loads the pool's running tasks, each on a random host of the offer table (1 % with host unknown), into a
resident handle and per cycle runs cook_state_usage for every user and every offer's host, on the grid and off it
(cpus + 0.1, mem / 3).  It prints the call's device time, wall time and bytes, the wall time of the same left folds
on the host (what a shim runs without the call), and whether the two agree to the bit.

  python tools/prof_state.py --usage --pool c2 --cycles 5
  python tools/prof_state.py --usage --pool c5 --c5-pool 5 --cycles 5

--cotasks loads a config-#3-shaped pool (its pending jobs, and its running tasks on random hosts of the offer table,
one in five in a group, 1 % with host unknown) and per cycle launches group members, finishes 3 % of the running
tasks and submits new group members.  It then runs cook_state_cotasks against the same lists built by numpy from a
host mirror of the running tasks (task -> host, groups), printing the call's device time, wall time and bytes, the
wall time of the host build, and whether the two are identical.

  python tools/prof_state.py --cotasks --cycles 6

--derived loads the pool's pending jobs and its running tasks (on random hosts of the offer table, 1 % with host
unknown; with the pool's groups, one task in five in a group) and per cycle ranks, then matches twice on the same
handle: the three-call sequence (cook_state_usage and cook_state_cotasks downloaded, then cook_state_match fed with
them) and one cook_state_match_derived.  Per arm it prints the bytes up and down, the host wall time of the library
calls (building the fed tables in Python excluded), the device time of the calls' events, and whether the outputs are
identical.  The placed jobs are then launched on their hosts and 3 % of the running tasks finish.

  python tools/prof_state.py --derived --pool c2 --cycles 6
  python tools/prof_state.py --derived --pool c5 --c5-pool 5 --cycles 4
  python tools/prof_state.py --derived --c3-pool 0 --cycles 4      # a config-#3 pool with groups

--considerable loads the pool's pending jobs and running tasks into a resident handle, ranks it, and per cycle runs
cook_state_considerable (the users' usage given, all of the queue considerable) against cook_match on host tables
holding the same rows in queue order with an empty offer table: the considerable set alone.  Per arm it prints the
device time, the host wall time of the library call, the bytes up and down, and whether the two sets are identical;
each cycle runs pending-jobs->considerable-jobs and, with quota_only, the autoscaling filter.

  python tools/prof_state.py --considerable --pool c2 --cycles 5
  python tools/prof_state.py --considerable --pool c5 --c5-pool 5 --cycles 5

--audit loads the pool into a resident handle, churns it for --cycles batches (3 % of the running tasks finish, one
pending job in a hundred is replaced, one in a hundred removed) and ranks it.  It then times, --reps times each after a
warm-up call: cook_state_digest without buckets and with 4096, the full cook_state_export, the export of 4 of 4096
buckets, and cook_state_queue.  Per call it prints the median, least and largest device time, download time and host
wall time, the bytes down, and (digest) the rate against the bytes the pass must read: the live rows' hashed columns,
live flags, list ranges and list entries.

  python tools/prof_state.py --audit --pool c2
  python tools/prof_state.py --audit --pool c5 --c5-pool 5

--rank-quota loads the pool's pending jobs and running tasks into a resident handle, on the grid and off it (running
cpus + 0.1, mem / 3), and times cook_state_rank --reps times each after a warm-up call: without a quota and with a pool
quota that cuts the queue half way (its start the running usage, folded in ascending task id).  Per kind it prints
the median and least device time and host wall time, the bytes up and down and the launches; COOK_GPU_LIB names
another build of the library to time the same calls on.

  python tools/prof_state.py --rank-quota --pool c2
  python tools/prof_state.py --rank-quota --pool c5 --c5-pool 5

--user-stats loads the pool's pending jobs and running tasks (or, with --c3-group N, config-#3 pools 0 .. N-1 into one
handle each) and per cycle runs cook_state_user_stats over the handles, users' shares and quotas set around their
running usage, on the grid and off it (cpus + 0.1, mem / 3).  It prints the call's device time, wall time, bytes and
launches, the wall time of the same folds and classification in single-threaded numpy (what a shim runs without the
call), and whether the two agree to the bit.

  python tools/prof_state.py --user-stats --pool c2 --cycles 5
  python tools/prof_state.py --user-stats --pool c5 --c5-pool 5 --cycles 5
  python tools/prof_state.py --user-stats --c3-group 4 --cycles 5
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cook_b200 import abi, engine, traces  # noqa: E402
from cook_b200.engine import GpuEngine  # noqa: E402

COLS = ("user", "cpus", "mem", "gpus", "ports", "allowed", "plugin_accept", "gpu_model", "disk_request", "disk_type",
        "est_end_ms", "ckpt_location", "reserved_host")
LISTS = (("novel_off", ("novel_host",)), ("attr_off", ("attr_col", "attr_val")), ("group_off", ("group_idx",)))


def csr_take(off, vals, rows):
    lens = (off[1:] - off[:-1])[rows]
    noff = np.zeros(len(rows) + 1, np.int32)
    np.cumsum(lens, out=noff[1:])
    idx = np.repeat(off[:-1][rows] - noff[:-1], lens) + np.arange(noff[-1])
    return noff, [v[idx] if noff[-1] else np.zeros(1, v.dtype) for v in vals]


class Jobs:
    """Every job of the run (live or not) as columns; rows are positions."""

    def __init__(self, jobs, prio, jid):
        self.c = {n: jobs.col(n) for n in COLS if jobs.col(n) is not None}
        self.l = {o: (jobs.col(o), [jobs.col(v) for v in vs]) for o, vs in LISTS if jobs.col(o) is not None}
        self.prio, self.jid = prio.copy(), jid.copy()

    def soa(self, rows):
        kw = {n: c[rows] for n, c in self.c.items()}
        for o, vs in LISTS:
            if o not in self.l:
                continue
            off, vals = csr_take(self.l[o][0], self.l[o][1], rows)
            kw[o] = off
            kw.update(dict(zip(vs, vals)))
        return abi.JobsSoA(n=len(rows), **kw)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                       "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def rebalance(a):
    r = traces.gen_config_pool("c4", a.c4_pool)["rebalance"]
    rt, hosts, users, groups, prm = r["running"].col("t"), r["hosts"], r["users"], r["groups"], r["params"]
    code = hosts.col("hostname_id")[r["running"].col("host")]
    store = Jobs(r["pending"], r["pending_priority"], r["pending_job_id"])
    print(json.dumps({"card": card(), "pool": f"c4/{a.c4_pool}", "running": rt.n, "pending": r["pending"].n,
                      "hosts": hosts.n, "max_preemption": prm.max_preemption}), flush=True)
    res, host = GpuEngine(pool_name="resident"), GpuEngine(pool_name="host")
    rows = np.arange(r["pending"].n)
    res.state_apply(abi.make_delta(reset=True, running=rt, running_hostname_id=code, pending=store.soa(rows),
                                   pending_priority=store.prio, pending_job_id=store.jid))
    q = res.state_rank(users)
    pos = {int(j): i for i, j in enumerate(store.jid)}
    take = np.array([pos[int(j)] for j in q[:prm.max_preemption]], np.int64)
    hj, tid = store.soa(take), rt.col("task_id")
    for cycle in range(a.cycles):
        w0 = time.perf_counter()
        got = res.state_rebalance(hosts, users, prm, groups=groups)
        w_res = time.perf_counter() - w0
        st_res = res.last_stats(abi.PHASE_REBALANCE)
        w0 = time.perf_counter()
        want = host.rebalance(r["running"], hj, store.jid[take], store.prio[take], hosts, users, prm, groups=groups)
        w_host = time.perf_counter() - w0
        st_host = host.last_stats(abi.PHASE_REBALANCE)
        same = len(got) == len(want) and all(
            (g["pending_idx"], g["host"], g["dru"], g["mem"], g["cpus"], g["gpus"]) ==
            (w["pending_idx"], w["host"], w["dru"], w["mem"], w["cpus"], w["gpus"]) and
            g["victims"] == [int(tid[v]) if v < rt.n else -1 - (v - rt.n) for v in w["victims"]] for g, w in zip(got, want))

        def arm(s, wall):
            return {**{k: round(s[k], 3) for k in ("ms_h2d", "ms_device", "ms_d2h")}, "wall_ms": round(1e3 * wall, 3),
                    "h2d_bytes": s["h2d_bytes"], "n_launches": s["n_launches"]}

        print(json.dumps({"cycle": cycle, "decisions": len(got), "resident": arm(st_res, w_res),
                          "host": arm(st_host, w_host), "identical": bool(same)}), flush=True)
    res.close()
    host.close()


def host_fold(run, host, U, codes):
    """What a shim computes without cook_state_usage: the same sums on the host, in ascending task id.  np.add.at
    and np.cumsum add in index order, so every sum is the left fold."""
    o = np.argsort(run["task_id"], kind="stable")
    u, hc = run["user"][o], host[o]
    amt = [run[k][o] for k in ("cpus", "mem", "gpus")]
    user = np.zeros((4, U))
    np.add.at(user[0], u, 1.0)
    for k in range(3):
        np.add.at(user[k + 1], u, amt[k])
    pool = np.array([float(len(o))] + [np.cumsum(x)[-1] if len(x) else 0.0 for x in amt])
    idx = np.full(max(int(codes.max()), int(hc.max())) + 1, -1, np.int64)
    idx[codes] = np.arange(len(codes))
    hi = np.where(hc >= 0, idx[np.maximum(hc, 0)], -1)
    sel = hi >= 0
    H = len(codes)
    rc, rm, rn = np.zeros(H), np.zeros(H), np.zeros(H, np.int32)
    np.add.at(rc, hi[sel], amt[0][sel])
    np.add.at(rm, hi[sel], amt[1][sel])
    np.add.at(rn, hi[sel], 1)
    return user, pool, rc, rm, rn


def usage(a):
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    rc0, codes, U = t["cols"]["running"], t["offers"].col("hostname_id").astype(np.int32), t["users"].n_users
    rng = np.random.default_rng(a.seed)
    n = len(rc0["task_id"])
    host = codes[rng.integers(0, len(codes), n)].astype(np.int32)
    host[rng.random(n) < 0.01] = -1
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "running": n,
                      "hosts": len(codes), "users": U}), flush=True)
    for regime in ("grid", "off"):
        run = {k: np.asarray(v).copy() for k, v in rc0.items()}
        if regime == "off":   # every partial sum rounds: the folds take the serial chain
            run["cpus"] = run["cpus"] + 0.1
            run["mem"] = run["mem"] / 3.0
        e = GpuEngine(pool_name="usage")
        e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**run), running_hostname_id=host))
        for cycle in range(a.cycles):
            w0 = time.perf_counter()
            got = e.state_usage(U, codes)
            w_dev = time.perf_counter() - w0
            st = e.last_stats(abi.PHASE_USAGE)
            w0 = time.perf_counter()
            user, pool, hc, hm, hn = host_fold(run, host, U, codes)
            w_host = time.perf_counter() - w0
            same = (all(np.array_equal(got["user"][k].view(np.uint64), user[i].view(np.uint64))
                        for i, k in enumerate(("count", "cpus", "mem", "gpus"))) and
                    np.array_equal(got["pool"].view(np.uint64), pool.view(np.uint64)) and
                    np.array_equal(got["run_cpus"].view(np.uint64), hc.view(np.uint64)) and
                    np.array_equal(got["run_mem"].view(np.uint64), hm.view(np.uint64)) and
                    np.array_equal(got["run_count"], hn))
            print(json.dumps({"regime": regime, "cycle": cycle,
                              "state_usage": {**{k: round(st[k], 3) for k in ("ms_h2d", "ms_device", "ms_d2h")},
                                              "wall_ms": round(1e3 * w_dev, 3), "h2d_bytes": st["h2d_bytes"],
                                              "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"]},
                              "host_fold_wall_ms": round(1e3 * w_host, 3), "identical": bool(same)}), flush=True)
        e.close()


def host_user_stats(tables, U, t):
    """What a shim computes without cook_state_user_stats, single-threaded numpy: per table the rows of every pool
    sorted by (user, id) (stable: an id two pools hold in pool order) and summed per user with np.add.at, which adds in
    index order, so each sum is the left fold; the states as cook_state_user_stats classifies them; each "all" entry a
    cumulative sum over the state's users in ascending code."""
    folds = []
    for rows in tables:   # running, then waiting: (user, id, cpus, mem) concatenated in pool order
        u, i, c, m = (np.concatenate([r[k] for r in rows]) for k in range(4))
        o = np.lexsort((i, u))
        f = np.zeros((3, U))
        np.add.at(f[0], u[o], 1.0)
        np.add.at(f[1], u[o], c[o])
        np.add.at(f[2], u[o], m[o])
        folds.append(f)
    (rj, rc, rm), (wj, wc, wm) = folds
    waiting = wj > 0
    starved = waiting & (rc < t["div_cpus"]) & (rm < t["div_mem"])
    wuq = waiting & (rj < t["quota_count"]) & (rc < t["quota_cpus"]) & (rm < t["quota_mem"]) & (t["rest_ok"] > 0)
    member = ((rj > 0).astype(np.uint8) | waiting.astype(np.uint8) << 1 | starved.astype(np.uint8) << 2 |
              wuq.astype(np.uint8) << 3)
    sel = [rj > 0, waiting, starved, wuq]
    jobs = np.stack([rj, wj, np.where(rj > 0, np.minimum(rj, wj), wj),
                     np.minimum(wj, np.maximum(t["quota_count"] - rj, 0.0))]).astype(np.int64)
    cpus = np.stack([rc, wc, np.minimum(wc, t["div_cpus"] - rc), np.minimum(wc, np.maximum(t["quota_cpus"] - rc, 0.0))])
    mem = np.stack([rm, wm, np.minimum(wm, t["div_mem"] - rm), np.minimum(wm, np.maximum(t["quota_mem"] - rm, 0.0))])
    for s in range(4):
        for a in (jobs, cpus, mem):
            a[s][~sel[s]] = 0
    last = lambda x: float(np.cumsum(x)[-1]) if len(x) else 0.0
    tot = [(int(jobs[s][sel[s]].sum()), last(cpus[s][sel[s]]), last(mem[s][sel[s]])) for s in range(4)]
    users = [int((sel[0] | sel[1]).sum()), int(starved.sum()), int(wuq.sum()), int(waiting.sum() - starved.sum()),
             int((sel[0] & ~waiting).sum())]
    return jobs, cpus, mem, member, tot, users


def user_stats_prof(a):
    """--user-stats: cook_state_user_stats against host_user_stats on one pool (--pool) or a quota group of config-#3
    pools (--c3-group N: pools 0 .. N-1, one handle each), on the grid and off it (cpus + 0.1, mem / 3)."""
    from cook_b200.engine import state_user_stats
    if a.c3_group > 0:
        ts = [traces.gen_config_pool("c3", p) for p in range(a.c3_group)]
        name = f"c3/0-{a.c3_group - 1}"
    else:
        ts = [traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)]
        name = a.pool if a.pool == "c2" else f"c5/{a.c5_pool}"
    U = max(t["users"].n_users for t in ts)
    rng = np.random.default_rng(a.seed)
    pend = [(t["cols"]["pending"]["user"].astype(np.int32), t["cols"]["pending"]["job_id"].astype(np.int64),
             t["jobs"].col("cpus"), t["jobs"].col("mem")) for t in ts]
    run = [tuple(np.asarray(t["cols"]["running"][k]) for k in ("user", "task_id", "cpus", "mem")) for t in ts]
    print(json.dumps({"card": card(), "pool": name, "pending": sum(len(p[0]) for p in pend),
                      "running": sum(len(r[0]) for r in run), "users": U}), flush=True)
    used = np.zeros(U)
    for r in run:
        np.add.at(used, r[0], r[2])
    # shares and quotas around the running usage, so that every state is populated
    tab = dict(div_cpus=np.where(rng.random(U) < 0.3, np.finfo(np.float64).max, used + rng.choice([-1.0, 4.0], U)),
               div_mem=np.full(U, np.finfo(np.float64).max), quota_count=rng.integers(0, 500, U).astype(float),
               quota_cpus=used + rng.choice([-1.0, 8.0], U), quota_mem=np.full(U, np.finfo(np.float64).max),
               rest_ok=(rng.random(U) < 0.9).astype(np.uint8))
    users = abi.make_users(U, div_cpus=tab["div_cpus"], div_mem=tab["div_mem"],
                           quota={"count": tab["quota_count"], "cpus": tab["quota_cpus"], "mem": tab["quota_mem"]})
    for regime in ("grid", "off"):
        off = (lambda c, m: (c + 0.1, m / 3.0)) if regime == "off" else (lambda c, m: (c, m))
        tp = [(u, i) + off(c, m) for u, i, c, m in pend]
        tr = [(u, i) + off(c, m) for u, i, c, m in run]
        engines = [GpuEngine(pool_name=f"stats{k}") for k in range(len(ts))]
        for e, p, r in zip(engines, tp, tr):
            n = len(p[0])
            e.state_apply(abi.make_delta(
                reset=True, pending=abi.JobsSoA(n=n, user=p[0], cpus=p[2], mem=p[3]), pending_priority=np.full(n, 50, np.int32),
                pending_job_id=p[1], running=abi.make_tasks(r[0], np.full(len(r[0]), 50, np.int32),
                                                           np.zeros(len(r[0]), np.int64), r[1], r[1] + 1, r[2], r[3])))
        for cycle in range(a.cycles):
            w0 = time.perf_counter()
            got = state_user_stats(engines, users, tab["rest_ok"])
            w_dev = time.perf_counter() - w0
            st = got["stats"]
            w0 = time.perf_counter()
            jobs, cpus, mem, member, tot, cnt = host_user_stats([tr, tp], U, tab)
            w_host = time.perf_counter() - w0
            bits = lambda x, y: np.array_equal(np.asarray(x).view(np.uint64), np.asarray(y).view(np.uint64))
            same = (np.array_equal(got["jobs"], jobs) and bits(got["cpus"], cpus) and bits(got["mem"], mem) and
                    np.array_equal(got["member"], member) and list(got["users"].values()) == cnt and
                    all(got["all"][k][0] == tot[s][0] and bits(np.array(got["all"][k][1:]), np.array(tot[s][1:]))
                        for s, k in enumerate(got["all"])))
            print(json.dumps({"regime": regime, "cycle": cycle,
                              "user_stats": {**{k: round(st[k], 3) for k in ("ms_h2d", "ms_device", "ms_d2h")},
                                             "wall_ms": round(1e3 * w_dev, 3), "h2d_bytes": st["h2d_bytes"],
                                             "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"]},
                              "numpy_wall_ms": round(1e3 * w_host, 3), "users": got["users"],
                              "identical": bool(same)}), flush=True)
        for e in engines:
            e.close()


def host_cotasks(tid, host, gidx, goff, G, acol, codes, attr):
    """What a shim computes without cook_state_cotasks, from its mirror of the running tasks: one entry per (task
    with a host, group), by (group, task id), with the host's attribute in the group's column (0: unlisted)."""
    lens = np.diff(goff)
    keep = np.repeat(host != -1, lens)
    g = gidx[keep]
    t = np.repeat(tid, lens)[keep]
    h = np.repeat(host, lens)[keep]
    o = np.lexsort((t, g))
    g, h = g[o], h[o]
    idx = np.full(max(int(codes.max()), int(h.max()) if len(h) else 0) + 1, -1, np.int64)
    idx[codes] = np.arange(len(codes))
    hi = idx[h]
    c = acol[g]
    val = np.where((hi >= 0) & (c >= 0), attr[np.maximum(c, 0), np.maximum(hi, 0)], 0).astype(np.int32)
    off = np.searchsorted(g, np.arange(G + 1)).astype(np.int32)
    return off, h.astype(np.int32), val


def cotasks_prof(a):
    t = traces.gen_config_pool("c3", a.c3_pool) if a.c3_pool >= 0 else traces.gen_c3_pool(a.seed)
    jobs, pc, rc = t["jobs"], t["cols"]["pending"], t["cols"]["running"]
    offers, groups = t["offers"], t["groups"]
    G, acol = groups.n_groups, groups.col("attr_col")
    codes = offers.col("hostname_id").astype(np.int32)
    attr = offers.col("attr").reshape(offers.n_attr_cols, offers.n)
    rng = np.random.default_rng(a.seed)
    J, R = jobs.n, len(rc["task_id"])
    goff_j, gidx_j = jobs.col("group_off"), jobs.col("group_idx")
    jgroups = [gidx_j[goff_j[i]:goff_j[i + 1]] for i in range(J)]
    members = [i for i in range(J) if len(jgroups[i])]
    # the host mirror: task id -> (host, groups)
    run = {int(rc["task_id"][i]): (int(codes[rng.integers(len(codes))]) if rng.random() > 0.01 else -1,
                                   [int(rng.integers(G))] if rng.random() < 0.2 else []) for i in range(R)}
    print(json.dumps({"card": card(), "pool": f"c3/{a.c3_pool}" if a.c3_pool >= 0 else "c3-shaped", "jobs": J,
                      "running": R, "groups": G, "offers": offers.n}), flush=True)
    e = GpuEngine(pool_name="cotasks")

    def run_delta(items, rm=()):
        tids = np.array([k for k, _ in items], np.int64)
        n = len(items)
        off, idx = abi.csr([v[1] for _, v in items])
        return abi.make_delta(running=abi.make_tasks(user=np.zeros(n, np.int32), priority=np.full(n, 50, np.int32),
                                                     start_time=np.full(n, 1_700_000_000_000, np.int64), task_id=tids,
                                                     job_id=tids + 1, cpus=np.ones(n), mem=np.ones(n)) if n else None,
                              running_hostname_id=np.array([v[0] for _, v in items], np.int32) if n else None,
                              running_group_off=off if n else None, running_group_idx=idx if n else None,
                              running_rm=rm)

    e.state_apply(run_delta(list(run.items())))
    # pending group members, launched a batch per cycle on the device
    jid0 = 10 ** 12
    pend = {jid0 + i: list(map(int, jgroups[m])) for i, m in enumerate(members)}
    off, idx = abi.csr(list(pend.values()))
    n = len(pend)
    e.state_apply(abi.make_delta(pending=abi.JobsSoA(n=n, user=np.zeros(n, np.int32), cpus=np.ones(n), mem=np.ones(n),
                                                     group_off=off, group_idx=idx),
                                 pending_priority=np.full(n, 50, np.int32), pending_job_id=np.array(list(pend), np.int64)))
    next_tid = max(run) + 10
    for cycle in range(a.cycles):
        # ---- the churn: launch group members, finish 3 %, submit as many new members
        nl = min(len(pend), max(1, len(members) // 8))
        lj = [int(j) for j in rng.choice(sorted(pend), nl, replace=False)]
        lt = [next_tid + 2 * i for i in range(nl)]
        next_tid += 2 * nl + 2
        lh = codes[rng.integers(0, len(codes), nl)].astype(np.int32)
        e.state_launch(lj, lt, np.full(nl, 1_700_000_000_000, np.int64), lh)
        for j, t_, h in zip(lj, lt, lh):
            run[t_] = (int(h), pend.pop(j))
        fin = [int(x) for x in rng.choice(sorted(run), int(len(run) * 0.03), replace=False)]
        for x in fin:
            del run[x]
        new = {jid0 + 10 ** 6 * (cycle + 1) + i: [int(rng.integers(G))] for i in range(nl)}
        off, idx = abi.csr(list(new.values()))
        e.state_apply(abi.make_delta(pending=abi.JobsSoA(n=nl, user=np.zeros(nl, np.int32), cpus=np.ones(nl),
                                                         mem=np.ones(nl), group_off=off, group_idx=idx),
                                     pending_priority=np.full(nl, 50, np.int32),
                                     pending_job_id=np.array(list(new), np.int64), running_rm=fin))
        pend.update(new)
        # ---- the lists, on the device and from the host mirror
        w0 = time.perf_counter()
        got = e.state_cotasks(G, acol, offers)
        w_dev = time.perf_counter() - w0
        st = e.last_stats(abi.PHASE_COTASKS)
        w0 = time.perf_counter()
        tid = np.fromiter(run.keys(), np.int64, len(run))
        host = np.fromiter((v[0] for v in run.values()), np.int32, len(run))
        goff = np.zeros(len(run) + 1, np.int64)
        np.cumsum([len(v[1]) for v in run.values()], out=goff[1:])
        gidx = np.fromiter((g for v in run.values() for g in v[1]), np.int32, int(goff[-1]))
        want = host_cotasks(tid, host, gidx, goff, G, acol, codes, attr)
        w_host = time.perf_counter() - w0
        same = all(np.array_equal(x, y) for x, y in zip(got, want))
        print(json.dumps({"cycle": cycle, "running": len(run), "entries": len(got[1]),
                          "state_cotasks": {**{k: round(st[k], 3) for k in ("ms_h2d", "ms_device", "ms_d2h")},
                                            "wall_ms": round(1e3 * w_dev, 3), "h2d_bytes": st["h2d_bytes"],
                                            "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"]},
                          "host_build_wall_ms": round(1e3 * w_host, 3), "identical": bool(same)}), flush=True)
    e.close()


def _with(s, **over):
    """A copy of the SoA struct `s` with fields replaced (None: NULL)."""
    kw = {n: s.col(n) if t in (abi.P_I32, abi.P_I64, abi.P_F64, abi.P_U8) else getattr(s, n) for n, t in s._fields_}
    kw.update(over)
    return type(s)(**kw)


def derived_prof(a):
    if a.c3_pool >= 0:
        t, name = traces.gen_config_pool("c3", a.c3_pool), f"c3/{a.c3_pool}"
    elif a.pool == "c2":
        t, name = traces.gen_c2(), "c2"
    else:
        t, name = traces.gen_config_pool("c5", a.c5_pool), f"c5/{a.c5_pool}"
    jobs, pc, rc = t["jobs"], t["cols"]["pending"], t["cols"]["running"]
    users, offers, groups = t["users"], t["offers"], t.get("groups")
    G = groups.n_groups if groups is not None else 0
    codes = offers.col("hostname_id").astype(np.int32)
    U, R = users.n_users, len(rc["task_id"])
    rng = np.random.default_rng(a.seed)
    host = codes[rng.integers(0, len(codes), R)].astype(np.int32)
    host[rng.random(R) < 0.01] = -1
    rgroups = [[int(rng.integers(G))] if G and rng.random() < 0.2 else [] for _ in range(R)]
    print(json.dumps({"card": card(), "pool": name, "jobs": jobs.n, "running": R, "offers": offers.n, "users": U,
                      "groups": G}), flush=True)
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    e = GpuEngine(pool_name="derived")
    off, idx = abi.csr(rgroups)
    e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**rc), running_hostname_id=host,
                                 running_group_off=off, running_group_idx=idx, **dict(
                                     pending=store.soa(np.arange(jobs.n)), pending_priority=store.prio,
                                     pending_job_id=store.jid)))
    params = traces.match_params(jobs.n, host_lifetime_mins=t.get("host_lifetime_mins", 0))
    max_ports = int(jobs.col("ports").max()) if jobs.col("ports") is not None else 0
    d_users = _with(users, usage_count=None, usage_cpus=None, usage_mem=None, usage_gpus=None)
    d_offers = _with(offers, run_cpus=None, run_mem=None, run_count=None)
    d_groups = _with(groups, cot_off=None, cot_hostname_id=None, cot_attr_val=None) if G else groups
    live = set(int(x) for x in rc["task_id"])
    next_tid = int(max(live)) + 10 if live else 10

    def dev_ms(s):
        return sum(s[k] for k in ("ms_h2d", "ms_device", "ms_d2h") if k in s) + \
            sum(s[k] for k in ("ms_considerable", "ms_match") if k in s)

    for cycle in range(a.cycles):
        e.state_rank(users)
        # ---- the three-call sequence
        w0 = time.perf_counter()
        us = e.state_usage(U, codes)
        wall = time.perf_counter() - w0
        st = [e.last_stats(abi.PHASE_USAGE)]
        f_users = _with(users, usage_count=us["user"]["count"], usage_cpus=us["user"]["cpus"],
                        usage_mem=us["user"]["mem"], usage_gpus=us["user"]["gpus"])
        f_offers = _with(offers, run_cpus=us["run_cpus"], run_mem=us["run_mem"], run_count=us["run_count"])
        f_groups = groups
        if G:
            w0 = time.perf_counter()
            cot = e.state_cotasks(G, groups.col("attr_col"), offers)
            wall += time.perf_counter() - w0
            st.append(e.last_stats(abi.PHASE_COTASKS))
            f_groups = _with(groups, cot_off=cot[0], cot_hostname_id=cot[1] if len(cot[1]) else np.zeros(1, np.int32),
                             cot_attr_val=cot[2] if len(cot[2]) else np.zeros(1, np.int32))
        w0 = time.perf_counter()
        ms = e.state_match(f_offers, f_users, params, groups=f_groups, max_ports=max_ports)
        wall += time.perf_counter() - w0
        st.append(ms["stats"])
        seq = {"h2d_bytes": sum(x["h2d_bytes"] for x in st), "d2h_bytes": sum(x["d2h_bytes"] for x in st),
               "wall_ms": round(1e3 * wall, 3), "device_ms": round(sum(dev_ms(x) for x in st), 3),
               "calls": len(st)}
        # ---- the derived call
        w0 = time.perf_counter()
        md = e.state_match(d_offers, d_users, params, groups=d_groups, max_ports=max_ports, derived=True)
        wall = time.perf_counter() - w0
        sd = md["stats"]
        der = {"h2d_bytes": sd["h2d_bytes"], "d2h_bytes": sd["d2h_bytes"], "wall_ms": round(1e3 * wall, 3),
               "device_ms": round(dev_ms(sd), 3), "ms_h2d": round(sd["ms_h2d"], 3),
               "ms_match_kernel": round(sd["ms_match_kernel"], 3), "calls": 1}
        same = all(np.array_equal(ms[k], md[k]) for k in ("considerable", "assign", "ports", "fail"))
        print(json.dumps({"cycle": cycle, "running": len(live), "entries": int(f_groups.col("cot_off")[-1]) if G else 0,
                          "considerable": len(md["considerable"]), "sequenced": seq, "derived": der,
                          "identical": bool(same)}), flush=True)
        # ---- launches on the chosen hosts, 3 % of the running tasks finish
        ok = md["assign"] >= 0
        jl = md["considerable"][ok]
        tl = next_tid + 2 * np.arange(len(jl), dtype=np.int64)
        next_tid += 2 * len(jl) + 2
        e.state_launch(jl, tl, np.full(len(jl), 1_700_000_000_000 + cycle, np.int64), codes[md["assign"][ok]])
        live.update(int(x) for x in tl)
        fin = [int(x) for x in rng.choice(sorted(live), int(len(live) * 0.03), replace=False)]
        live.difference_update(fin)
        e.state_apply(abi.make_delta(running_rm=fin))
    e.close()


def offers_prof(a):
    """--offers: the same offer stream through the library's live offers (cook_state_offers_add +
    cook_state_match_offers) and through the host's lease cache (cycle.OfferCache, offers_from_cache and
    cook_state_match_derived), on two resident handles holding the same rows."""
    from cook_b200.cycle import OfferCache, offers_from_cache
    if a.c3_pool >= 0:
        t, name = traces.gen_config_pool("c3", a.c3_pool), f"c3/{a.c3_pool}"
    else:
        t, name = traces.gen_c2(), "c2"
    jobs, pc, rc = t["jobs"], t["cols"]["pending"], t["cols"]["running"]
    users, tmpl = t["users"], t["offers"]
    codes = tmpl.col("hostname_id").astype(np.int32)
    names = {int(c): f"node-{int(c):07d}" for c in codes}
    code_of = {n: c for c, n in names.items()}
    U, R, O = users.n_users, len(rc["task_id"]), tmpl.n
    rng = np.random.default_rng(a.seed)
    host = codes[rng.integers(0, O, R)].astype(np.int32)
    print(json.dumps({"card": card(), "pool": name, "jobs": jobs.n, "running": R, "hosts": O, "users": U}), flush=True)
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    arms = {k: GpuEngine(pool_name=k) for k in ("resident", "cache")}
    # the leases carry cpus, mem and hostnames only (what offers_from_cache merges), and no job holds a reservation;
    # the cache arm's table is as wide as the attribute columns the jobs name, as the library's is
    pend = _with(store.soa(np.arange(jobs.n)), reserved_host=None)
    ac = jobs.col("attr_col")
    W = int(ac.max()) + 1 if ac is not None and len(ac) else 0
    for e in arms.values():
        e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**rc), running_hostname_id=host,
                                     pending=pend, pending_priority=store.prio, pending_job_id=store.jid))
    params = traces.match_params(min(jobs.n, 20_000))
    d_users = _with(users, usage_count=None, usage_cpus=None, usage_mem=None, usage_gpus=None)
    cache, incubate, lid = OfferCache(incubate_ms=15_000), 15_000, 0
    next_tid = int(max(rc["task_id"])) + 10 if R else 10
    now = 1_700_000_000_000
    cpus0, mem0 = tmpl.col("cpus"), tmpl.col("mem")
    for cycle in range(a.cycles):
        now += 5_000
        leases = []   # 40 % of the hosts offer again, some in two or three leases (cpus and mem in halves)
        for h in rng.choice(O, int(O * 0.4), replace=False).tolist():
            k = int(rng.choice([1, 1, 1, 2, 3]))
            for _ in range(k):
                leases.append({"id": lid, "hostname": names[int(codes[h])], "code": int(codes[h]),
                               "cpus": float(np.floor(2 * cpus0[h] / k) / 2), "mem": float(np.floor(mem0[h] / k))})
                lid += 1
        n = len(leases)
        soa = abi.OffersSoA(n=n, n_attr_cols=0, hostname_id=np.array([l["code"] for l in leases], np.int32),
                            cpus=np.array([l["cpus"] for l in leases]), mem=np.array([l["mem"] for l in leases]))
        ids = np.array([l["id"] for l in leases], np.int64)
        for e in arms.values():
            e.state_rank(users)
        # ---- resident offers
        e = arms["resident"]
        w0 = time.perf_counter()
        e.state_offers_add(soa, ids, now, hostnames=[l["hostname"] for l in leases])
        add_stats = e.last_stats(abi.PHASE_STATE)
        mr = e.state_match_offers(now, incubate, d_users, params)
        wall_r = time.perf_counter() - w0
        sr = mr["stats"]
        # ---- the host's lease cache
        e = arms["cache"]
        w0 = time.perf_counter()
        cache.add(leases, now)
        cache.expire(now)
        vm, table = offers_from_cache(cache, code_of)
        if W:
            table = _with(table, n_attr_cols=W, attr=np.zeros(W * table.n, np.int32))
        mc = e.state_match(_with(table, run_cpus=None, run_mem=None, run_count=None), d_users, params, derived=True)
        assign_codes = np.where(mc["assign"] >= 0, table.col("hostname_id")[np.maximum(mc["assign"], 0)], -1)
        cache.after_match({names[int(c)] for c in assign_codes if c >= 0})
        wall_c = time.perf_counter() - w0
        sc = mc["stats"]
        same = np.array_equal(mr["considerable"], mc["considerable"]) and np.array_equal(mr["assign"], assign_codes)
        dev = lambda s: round(s["ms_considerable"] + s["ms_match"] + s["ms_h2d"] + s["ms_d2h"], 3)
        print(json.dumps({"cycle": cycle, "offers_added": n, "vms": int(table.n), "placed": int((mr["assign"] >= 0).sum()),
                          "resident": {"wall_ms": round(1e3 * wall_r, 3),
                                       "device_ms": round(dev(sr) + add_stats["ms_h2d"] + add_stats["ms_device"], 3),
                                       "h2d_bytes": sr["h2d_bytes"] + add_stats["h2d_bytes"], "d2h_bytes": sr["d2h_bytes"]},
                          "cache": {"wall_ms": round(1e3 * wall_c, 3), "device_ms": dev(sc), "h2d_bytes": sc["h2d_bytes"],
                                    "d2h_bytes": sc["d2h_bytes"]},
                          "identical": bool(same)}), flush=True)
        # ---- both arms launch the placements on the chosen hosts
        ok = mr["assign"] >= 0
        jl = mr["considerable"][ok]
        tl = next_tid + 2 * np.arange(len(jl), dtype=np.int64)
        next_tid += 2 * len(jl) + 2
        for e in arms.values():
            e.state_launch(jl, tl, np.full(len(jl), now, np.int64), mr["assign"][ok].astype(np.int32))
    for e in arms.values():
        e.close()


def launch_cycle(cycle, res, twin, job_id, lt, hosts, rest, match_args):
    """One cycle of --launch: the launches by id on `res` and as a delta on `twin`, the rest of the batch on both,
    then rank and match on both.  Returns the jobs the match placed and their hosts' codes."""
    users, offers, params, groups, max_ports = match_args
    n = len(job_id)
    d = abi.make_delta(running=abi.make_tasks(**lt) if n else None, pending_rm=job_id,
                       running_hostname_id=hosts if n else None)
    w0 = time.perf_counter()
    res.state_launch(job_id, lt["task_id"], lt["start_time"], hosts)
    w_launch = time.perf_counter() - w0
    st_launch = res.last_stats(abi.PHASE_STATE)
    w0 = time.perf_counter()
    twin.state_apply(d)
    w_delta = time.perf_counter() - w0
    st_delta = twin.last_stats(abi.PHASE_STATE)
    for e in (res, twin):
        e.state_apply(rest)
    q, q2 = res.state_rank(users), twin.state_rank(users)
    m1 = res.state_match(offers, users, params, groups=groups, max_ports=max_ports)
    m2 = twin.state_match(offers, users, params, groups=groups, max_ports=max_ports)
    same = np.array_equal(q, q2) and all(np.array_equal(m1[k], m2[k]) for k in ("considerable", "assign", "ports", "fail"))

    def arm(s, wall):
        return {"h2d_bytes": s["h2d_bytes"], "ms_h2d": round(s["ms_h2d"], 3), "ms_device": round(s["ms_device"], 3),
                "wall_ms": round(1e3 * wall, 3), "n_launches": s["n_launches"]}

    print(json.dumps({"cycle": cycle, "launched": n, "launch": arm(st_launch, w_launch), "delta": arm(st_delta, w_delta),
                      "identical": bool(same), "n_matched": int(m1["stats"]["n_matched"])}), flush=True)
    ok = m1["assign"] >= 0
    return m1["considerable"][ok], offers.col("hostname_id")[m1["assign"][ok]].astype(np.int32)


def considerable_prof(a):
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    jobs, pc, rc, users = t["jobs"], t["cols"]["pending"], t["cols"]["running"], t["users"]
    J = jobs.n
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "jobs": J,
                      "running": len(rc["task_id"]), "users": users.n_users}), flush=True)
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    rows = np.arange(J)
    res, host = GpuEngine(pool_name="resident"), GpuEngine(pool_name="host")
    res.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**{k: np.asarray(v) for k, v in rc.items()}),
                                   pending=store.soa(rows), pending_priority=store.prio, pending_job_id=store.jid))
    q = res.state_rank(users)
    pos = {int(j): i for i, j in enumerate(store.jid)}
    ranked = np.array([pos[int(j)] for j in q], np.int32)
    empty = abi.OffersSoA(n=0, hostname_id=np.zeros(1, np.int32), name_rank=np.zeros(1, np.int32), cpus=np.zeros(1),
                          mem=np.zeros(1), run_cpus=np.zeros(1), run_mem=np.zeros(1), run_count=np.zeros(1, np.int32),
                          n_attr_cols=0)
    hj = store.soa(rows)
    ones = np.ones(J, np.uint8)
    plain = abi.JobsSoA(n=J, user=hj.col("user"), cpus=hj.col("cpus"), mem=hj.col("mem"), gpus=hj.col("gpus"),
                        allowed=hj.col("allowed") if hj.col("allowed") is not None else ones,
                        plugin_accept=hj.col("plugin_accept") if hj.col("plugin_accept") is not None else ones)
    auto = abi.JobsSoA(n=J, user=hj.col("user"), cpus=hj.col("cpus"), mem=hj.col("mem"), gpus=hj.col("gpus"),
                       allowed=ones, plugin_accept=ones)
    nc = max(len(q), 1)
    for cycle in range(a.cycles):
        for quota_only in (0, 1):
            prm = abi.ConsiderableParams(nc, 0, quota_only, abi.USAGE_GIVEN, 0)
            w0 = time.perf_counter()
            got = res.state_considerable(users, prm)
            w_res = time.perf_counter() - w0
            st = res.last_stats(abi.PHASE_CONSIDERABLE)
            w0 = time.perf_counter()
            mh = host.match(ranked, auto if quota_only else plain, empty, users, traces.match_params(nc))
            w_host = time.perf_counter() - w0
            hs = mh["stats"]
            same = np.array_equal(got, store.jid[mh["considerable"]])
            print(json.dumps({"cycle": cycle, "quota_only": quota_only, "considerable": len(got),
                              "resident": {"ms_h2d": round(st["ms_h2d"], 3), "ms_device": round(st["ms_device"], 3),
                                           "ms_d2h": round(st["ms_d2h"], 3), "wall_ms": round(1e3 * w_res, 3),
                                           "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                                           "n_launches": st["n_launches"]},
                              "host": {"ms_h2d": round(hs["ms_h2d"], 3), "ms_considerable": round(hs["ms_considerable"], 3),
                                       "ms_d2h": round(hs["ms_d2h"], 3), "wall_ms": round(1e3 * w_host, 3),
                                       "h2d_bytes": hs["h2d_bytes"], "d2h_bytes": hs["d2h_bytes"],
                                       "n_launches": hs["n_launches"]},
                              "identical": bool(same)}), flush=True)
    res.close()
    host.close()


def audit_prof(a):
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    jobs, pc, rc, users = t["jobs"], t["cols"]["pending"], t["cols"]["running"], t["users"]
    rng = np.random.default_rng(a.seed)
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    run = {k: np.asarray(v) for k, v in rc.items()}
    res = GpuEngine(pool_name="resident")
    res.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**run), pending=store.soa(np.arange(jobs.n)),
                                   pending_priority=store.prio, pending_job_id=store.jid))
    alive, tids = np.ones(jobs.n, bool), run["task_id"].copy()
    for _ in range(a.cycles):
        live = np.flatnonzero(alive)
        pick = rng.choice(live, max(2, len(live) // 50), replace=False)
        rm, up = pick[:len(pick) // 2], pick[len(pick) // 2:]
        fin = rng.choice(len(tids), len(tids) * 3 // 100, replace=False)
        store.prio[up] = 90
        res.state_apply(abi.make_delta(pending_rm=store.jid[rm], running_rm=tids[fin], pending=store.soa(up),
                                       pending_priority=store.prio[up], pending_job_id=store.jid[up]))
        alive[rm] = False
        tids = np.delete(tids, fin)
    q = res.state_rank(users)
    d = res.state_digest()
    P, Rn, E = d["pending"][2], d["running"][2], d["entries"]
    must_read = P * (78 + 1 + 24) + 4 * E[0] + 8 * E[1] + 4 * E[2] + Rn * (60 + 1 + 8) + 4 * E[3]
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "pending": P, "running": Rn,
                      "entries": E, "queue": len(q), "consistent": d["consistent"], "digest_must_read_bytes": must_read,
                      "reps": a.reps}), flush=True)
    few = np.zeros(4096, np.uint8)
    few[[1, 1000, 2000, 4000]] = 1
    calls = (("digest", lambda: res.state_digest()), ("digest_4096_buckets", lambda: res.state_digest(4096)),
             ("export_all", lambda: res.state_export()), ("export_4_of_4096_buckets", lambda: res.state_export(few)),
             ("queue", lambda: res.state_queue()))
    for name, call in calls:
        call()
        rows = []
        for _ in range(a.reps):
            w0 = time.perf_counter()
            call()
            rows.append((1e3 * (time.perf_counter() - w0), res.last_stats(abi.PHASE_AUDIT)))
        st = rows[-1][1]

        def spread(x):
            return {"median": round(float(np.median(x)), 3), "min": round(float(np.min(x)), 3), "max": round(float(np.max(x)), 3)}

        dev = [s["ms_device"] for _, s in rows]
        out = {"call": name, "ms_device": spread(dev), "ms_d2h": spread([s["ms_d2h"] for _, s in rows]),
               "wall_ms": spread([w for w, _ in rows]), "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
               "n_launches": st["n_launches"]}
        if name.startswith("digest"):
            out["GBps_of_must_read_at_median"] = round(must_read / (np.median(dev) * 1e-3) / 1e9, 1)
        print(json.dumps(out), flush=True)
    res.close()


def host_sweeps(m, now, dflt, mx, gp, lists):
    """The three lists in numpy over the host mirror m (the columns of the handle's rows and records)."""
    out = {}
    if "linger" in lists:
        lim = np.minimum(np.where(m["maxrt"] < 0, dflt, m["maxrt"]), mx)
        k = np.flatnonzero(now - m["start"] > lim)
        out["linger"] = np.sort(m["tid"][k])
    if "cancel" in lists:
        out["cancel"] = np.sort(m["tid"][m["cancelled"]])
    if "straggler" in lists:
        G = len(gp["kind"])
        chk = gp["kind"] == abi.SWEEP_QUANTILE_DEVIATION
        rg, rt = m["rec_group"], m["rec_rt"]
        keep = chk[rg]
        rg, rt = rg[keep], rt[keep]
        o = np.lexsort((rt, rg))
        rg, rt = rg[o], rt[o]
        cnt = np.bincount(rg, minlength=G)
        first = np.concatenate(([0], np.cumsum(cnt)[:-1]))
        idx = ((gp["n_jobs"] - 1).astype(np.float64) * gp["quantile"]).astype(np.int64)
        ok = chk & (idx >= 0) & (cnt > idx)
        limit = np.full(G, np.inf)
        limit[ok] = rt[first[ok] + idx[ok]].astype(np.float64) * gp["multiplier"][ok]
        eg, row = m["e_group"], m["e_row"]
        run = ~m["unknown"][row] & chk[eg]
        secs = (now - m["start"][row]) // 1000
        hit = run & (secs.astype(np.float64) > limit[eg])
        g, t = eg[hit], m["tid"][row[hit]]
        o = np.lexsort((t, g))
        out["straggler"] = (g[o], t[o])
    return out


def sweeps_prof(a):
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    rc = {k: np.asarray(v).copy() for k, v in t["cols"]["running"].items()}
    rng = np.random.default_rng(a.seed)
    n, G = len(rc["task_id"]), 400
    glen = np.where(rng.random(n) < 0.2, rng.integers(1, 3, n), 0)
    goff = np.concatenate(([0], np.cumsum(glen))).astype(np.int32)
    gidx = rng.integers(0, G, int(goff[-1])).astype(np.int32)
    now = int(rc["start_time"].max()) + 3_600_000
    rc["start_time"] = now - rng.integers(1000, 48 * 3_600_000, n)
    e = GpuEngine(pool_name="sweeps")
    e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**rc), running_group_off=goff,
                                 running_group_idx=gidx))
    tid = rc["task_id"].astype(np.int64)
    maxrt = np.where(rng.random(n) < 0.1, rng.integers(3_600_000, 30 * 3_600_000, n), -1).astype(np.int64)
    canc, unk = rng.random(n) < 0.02, rng.random(n) < 0.05
    e.state_task_facts(tid, maxrt, canc, unk)
    n_rec = 4000
    rec_group = rng.integers(0, G, n_rec).astype(np.int32)
    rec_rt = rng.integers(600, 20 * 3600, n_rec).astype(np.int32)
    e.state_group_runtimes(rec_group, rec_rt)
    gp = {"kind": np.where(rng.random(G) < 0.8, abi.SWEEP_QUANTILE_DEVIATION, abi.SWEEP_NONE).astype(np.int32),
          "quantile": rng.choice([0.25, 0.5, 0.9], G), "multiplier": rng.choice([1.5, 2.0, 3.0], G),
          "n_jobs": rng.integers(5, 40, G).astype(np.int32)}
    mirror = {"tid": tid, "start": rc["start_time"].astype(np.int64), "maxrt": maxrt, "cancelled": canc,
              "unknown": unk, "rec_group": rec_group, "rec_rt": rec_rt, "e_group": gidx,
              "e_row": np.repeat(np.arange(n), glen)}
    dflt, mx = 24 * 3_600_000, 36 * 3_600_000
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "running": n,
                      "grouped_rows": int((glen > 0).sum()), "group_entries": int(goff[-1]), "records": n_rec,
                      "groups": G}), flush=True)
    for lists in (("linger",), ("cancel",), ("straggler",), ("linger", "cancel", "straggler")):
        got = None
        for _ in range(3):   # warm-up: the carves and the first launches
            got = engine.state_sweep([e], now, dflt, mx, gp, lists)
        dev, wall, host = [], [], []
        for _ in range(a.reps):
            w0 = time.perf_counter()
            got = engine.state_sweep([e], now, dflt, mx, gp, lists)
            wall.append(time.perf_counter() - w0)
            dev.append(got["stats"]["ms_h2d"] + got["stats"]["ms_device"] + got["stats"]["ms_d2h"])
            w0 = time.perf_counter()
            want = host_sweeps(mirror, now, dflt, mx, gp, lists)
            host.append(time.perf_counter() - w0)
        same = all(np.array_equal([x[0] for x in got[k]], want[k]) for k in ("linger", "cancel") if k in lists)
        if "straggler" in lists:
            same = same and np.array_equal([x[0] for x in got["straggler"]], want["straggler"][0]) and \
                np.array_equal([x[1] for x in got["straggler"]], want["straggler"][1])
        st = got["stats"]
        print(json.dumps({"lists": "+".join(lists), "n": {k: len(got[k]) for k in lists},
                          "device_ms": round(float(np.median(dev)), 4), "wall_ms": round(1e3 * float(np.median(wall)), 4),
                          "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                          "numpy_wall_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same)}),
              flush=True)
    e.close()


def host_unscheduled(m, q):
    """numpy over a host mirror of the rows: cook_state_unscheduled's answers (status, usage, position, ahead)."""
    pj = m["p_pos"]
    rpos = m["r_of_job"]
    out = []
    per_user = {}
    for j in q.tolist():
        if j in pj:
            st, i = 1, pj[j]
            u = int(m["p_user"][i])
        elif j in rpos:
            st, i = 2, rpos[j]
            u = int(m["r_user"][i])
        else:
            out.append((0, (0.0,) * 4, -1, []))
            continue
        if u not in per_user:
            ri = np.flatnonzero(m["r_user"] == u)
            ri = ri[np.lexsort((m["r_tid"][ri], m["r_jid"][ri]))]
            last = np.ones(len(ri), bool)
            last[:-1] = m["r_jid"][ri[1:]] != m["r_jid"][ri[:-1]]
            ri = ri[last]                                       # one row per job: its greatest task id
            ri = ri[np.argsort(m["r_tid"][ri], kind="stable")]   # the fold order
            fold = (float(len(ri)),) + tuple(float(np.cumsum(m["r_" + c][ri])[-1]) if len(ri) else 0.0
                                             for c in ("cpus", "mem", "gpus"))
            pi = np.flatnonzero(m["p_user"] == u)
            key = (np.concatenate([m["r_jid"][ri], m["p_jid"][pi]]),
                   np.concatenate([m["r_tid"][ri], np.full(len(pi), -1)]),
                   np.concatenate([m["r_start"][ri], np.full(len(pi), np.iinfo(np.int64).max)]),
                   -np.concatenate([m["r_prio"][ri], m["p_prio"][pi]]))
            order = np.lexsort(key)
            ids = key[0][order]
            run_at = {int(t): k for k, t in enumerate(np.concatenate([m["r_tid"][ri], np.full(len(pi), -1)])[order])
                      if t >= 0}
            pend_at = {int(x): k for k, (x, t) in enumerate(zip(ids, key[1][order])) if t < 0}
            per_user[u] = (fold, ids, run_at, pend_at)
        fold, ids, run_at, pend_at = per_user[u]
        pos = pend_at[j] if st == 1 else run_at[int(m["r_tid"][i])]
        usage = (0.0,) * 4
        if st == 1:
            usage = (fold[0] + 1.0, fold[1] + m["p_cpus"][i], fold[2] + m["p_mem"][i], fold[3] + m["p_gpus"][i])
        out.append((st, usage, pos, ids[:min(pos, 10)].tolist()))
    return out


def unscheduled_prof(a):
    """cook_state_unscheduled over a resident pool (C2, or config-#5 pool --c5-pool), on the grid and off it, for one
    job, 1000 jobs and every waiting job of the user with the most, against numpy over a host mirror."""
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    jobs, pc, rc0 = t["jobs"], t["cols"]["pending"], t["cols"]["running"]
    J, R = jobs.n, len(rc0["task_id"])
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "pending": J,
                      "running": R}), flush=True)
    rng = np.random.default_rng(a.seed)
    for regime in ("grid", "off"):
        run = {k: np.asarray(v).copy() for k, v in rc0.items()}
        cols = {c: np.asarray(jobs.col(c) if jobs.col(c) is not None else np.zeros(J)).astype(np.float64)
                for c in ("cpus", "mem", "gpus")}
        if regime == "off":
            run["cpus"] = run["cpus"] + 0.1
            run["mem"] = run["mem"] / 3.0
            cols["cpus"] = cols["cpus"] + 0.1
        soa = Jobs(jobs, pc["priority"], pc["job_id"]).soa(np.arange(J))
        soa = abi.JobsSoA(**{n: soa.col(n) if tp in abi._NP else getattr(soa, n) for n, tp in soa._fields_
                             if n not in ("cpus",)}, cpus=cols["cpus"]) if regime == "off" else soa
        e = GpuEngine(pool_name="unscheduled")
        e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**run), pending=soa,
                                     pending_priority=pc["priority"], pending_job_id=pc["job_id"]))
        m = {"p_user": np.asarray(pc["user"]), "p_prio": np.asarray(pc["priority"]), "p_jid": np.asarray(pc["job_id"]),
             "p_cpus": cols["cpus"], "p_mem": cols["mem"], "p_gpus": cols["gpus"],
             "r_user": np.asarray(run["user"]), "r_prio": np.asarray(run["priority"]),
             "r_start": np.asarray(run["start_time"]), "r_tid": np.asarray(run["task_id"]),
             "r_jid": np.asarray(run["job_id"]), "r_cpus": np.asarray(run["cpus"], np.float64),
             "r_mem": np.asarray(run["mem"], np.float64),
             "r_gpus": np.asarray(run["gpus"] if "gpus" in run else np.zeros(R), np.float64)}
        m["p_pos"] = {int(j): i for i, j in enumerate(m["p_jid"])}
        m["r_of_job"] = {}
        for i in np.argsort(m["r_tid"]):
            m["r_of_job"][int(m["r_jid"][i])] = int(i)
        heavy = int(np.bincount(m["p_user"]).argmax())
        sizes = {"1": rng.choice(m["p_jid"], 1), "1000": np.concatenate([rng.choice(m["p_jid"], 900),
                                                                         rng.choice(m["r_jid"], 100)]),
                 "heaviest_user": m["p_jid"][m["p_user"] == heavy]}
        for name, q in sizes.items():
            q = np.asarray(q, np.int64)
            for _ in range(3):   # warm-up: the carves and the first launches
                got = e.state_unscheduled(q)
            dev, wall, host, same = [], [], [], True
            for _ in range(a.reps):
                w0 = time.perf_counter()
                got = e.state_unscheduled(q)
                wall.append(time.perf_counter() - w0)
                st = got["stats"]
                dev.append(st["ms_h2d"] + st["ms_device"] + st["ms_d2h"])
                w0 = time.perf_counter()
                want = host_unscheduled(m, q)
                host.append(time.perf_counter() - w0)
                same = same and all(
                    int(got["status"][i]) == w[0] and np.array_equal(got["usage"][i].view(np.int64),
                                                                     np.array(w[1], np.float64).view(np.int64))
                    and int(got["position"][i]) == w[2] and got["ahead"][i] == w[3] for i, w in enumerate(want))
            print(json.dumps({"regime": regime, "queries": name, "n": len(q),
                              "device_ms": round(float(np.median(dev)), 4), "wall_ms": round(1e3 * float(np.median(wall)), 4),
                              "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                              "numpy_wall_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same)}),
                  flush=True)
        e.close()


def host_user_usage(m, users, per_pool, by_group):
    """numpy over a host mirror of the running rows (every handle's, with its index): cook_state_user_usage's segments
    [(user, scope, group, jobs, cpus, mem, gpus, job ids or None)], each fold sequential in (task id, handle)."""
    i = np.arange(len(m["user"])) if users is None else np.flatnonzero(np.isin(m["user"], users))
    i = i[np.lexsort((m["tid"][i], m["jid"][i], m["pidx"][i]))]
    last = np.ones(len(i), bool)
    last[:-1] = (m["jid"][i[1:]] != m["jid"][i[:-1]]) | (m["pidx"][i[1:]] != m["pidx"][i[:-1]])
    i = i[last]                                          # one row per (handle, job): its greatest task id
    i = i[np.lexsort((m["pidx"][i], m["tid"][i]))]       # the fold order
    out = []
    for sc in [False] + ([True] if per_pool else []):
        for gr in [False] + ([True] if by_group else []):
            scope = m["pidx"][i] if sc else np.full(len(i), -1)
            group = m["grp"][i] if gr else np.full(len(i), -2)
            k = np.lexsort((np.arange(len(i)), group, scope, m["user"][i]))
            ii, key = i[k], np.stack([m["user"][i][k], scope[k], group[k]], 1)
            cut = np.flatnonzero(np.any(key[1:] != key[:-1], 1)) + 1
            for s, e in zip(np.concatenate([[0], cut]), np.concatenate([cut, [len(ii)]])):
                seg = ii[s:e]
                sums = [float(np.cumsum(m[c][seg])[-1]) for c in ("cpus", "mem", "gpus")]
                out.append((int(key[s, 0]), int(key[s, 1]), int(key[s, 2]), e - s, *sums,
                            m["jid"][seg].tolist() if gr else None))
    return sorted(out, key=lambda x: x[:3])


def user_usage_prof(a):
    """cook_state_user_usage over resident pools (C2, config-#5 pool --c5-pool, or --c3-group N config-#3 pools as N
    handles with per_pool), on the grid and off it, for the lightest user, the heaviest user and every user, with and
    without groups, against numpy over a host mirror.  A third of the running rows get a group list of one or two
    groups of 500."""
    if a.c3_group > 0:
        ts = [traces.gen_config_pool("c3", p) for p in range(a.c3_group)]
        name = f"c3/0-{a.c3_group - 1}"
    else:
        ts = [traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)]
        name = a.pool if a.pool == "c2" else f"c5/{a.c5_pool}"
    rng = np.random.default_rng(a.seed)
    runs = [{k: np.asarray(v).copy() for k, v in t["cols"]["running"].items()} for t in ts]
    lists = [[[int(g) for g in rng.choice(500, int(rng.integers(1, 3)), replace=False)] if rng.random() < 1 / 3
              else [] for _ in range(len(r["task_id"]))] for r in runs]
    print(json.dumps({"card": card(), "pools": name, "handles": len(ts),
                      "running": sum(len(r["task_id"]) for r in runs)}), flush=True)
    per_pool = len(ts) > 1
    for regime in ("grid", "off"):
        es, m = [], {k: [] for k in ("user", "tid", "jid", "pidx", "grp", "cpus", "mem", "gpus")}
        for p, (r0, gl) in enumerate(zip(runs, lists)):
            r = dict(r0)
            if regime == "off":
                r["cpus"] = r["cpus"] + 0.1
                r["mem"] = r["mem"] / 3.0
            off, idx = abi.csr(gl)
            e = GpuEngine(pool_name=f"user-usage-{p}")
            e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**r), running_group_off=off,
                                         running_group_idx=idx))
            es.append(e)
            n = len(r["task_id"])
            for k, src in (("user", r["user"]), ("tid", r["task_id"]), ("jid", r["job_id"]), ("cpus", r["cpus"]),
                           ("mem", r["mem"]), ("gpus", r["gpus"] if "gpus" in r else np.zeros(n))):
                m[k].append(np.asarray(src))
            m["pidx"].append(np.full(n, p))
            m["grp"].append(np.array([g[0] if g else -1 for g in gl]))
        m = {k: np.concatenate(v) for k, v in m.items()}
        for k in ("cpus", "mem", "gpus"):
            m[k] = m[k].astype(np.float64)
        cnt = np.bincount(m["user"])
        users = {"light": [int(np.argmin(np.where(cnt > 0, cnt, cnt.max() + 1)))],
                 "heaviest": [int(cnt.argmax())], "all": None}
        for kind, q in users.items():
            for bg in (False, True):
                for _ in range(3):   # warm-up: the carves and the first launches
                    got = engine.state_user_usage(es, q, per_pool, bg)
                dev, wall, host, same = [], [], [], True
                for _ in range(a.reps):
                    w0 = time.perf_counter()
                    got = engine.state_user_usage(es, q, per_pool, bg)
                    wall.append(time.perf_counter() - w0)
                    st = got["stats"]
                    dev.append(st["ms_h2d"] + st["ms_device"] + st["ms_d2h"])
                    w0 = time.perf_counter()
                    want = host_user_usage(m, q, per_pool, bg)
                    host.append(time.perf_counter() - w0)
                    same = same and len(want) == len(got["user"]) and all(
                        (int(got["user"][d]), int(got["scope"][d]), int(got["group"][d]), int(got["jobs"][d])) == w[:4]
                        and np.array_equal(np.array([got[c][d] for c in ("cpus", "mem", "gpus")]).view(np.int64),
                                           np.array(w[4:7], np.float64).view(np.int64)) and got["lists"][d] == w[7]
                        for d, w in enumerate(want))
                print(json.dumps({"regime": regime, "users": kind, "by_group": bg, "per_pool": per_pool,
                                  "segments": len(got["user"]), "jobs": int(sum(got["jobs"][got["scope"] == -1][
                                      got["group"][got["scope"] == -1] == abi.UU_TOTAL])),
                                  "device_ms": round(float(np.median(dev)), 4),
                                  "wall_ms": round(1e3 * float(np.median(wall)), 4), "h2d_bytes": st["h2d_bytes"],
                                  "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                                  "numpy_wall_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same)}),
                      flush=True)
        for e in es:
            e.close()


def host_instance_stats(m, now, unknown):
    """numpy over a host mirror of the running rows (every handle's, with its index): cook_state_instance_stats'
    segments [(kind, user, reason, count, totals, percentiles)] and leaders, each fold sequential in (task id, handle)
    (np.cumsum), each percentile a nearest rank of np.sort."""
    i = np.flatnonzero(m["unknown"] == unknown)
    i = i[np.lexsort((m["pidx"][i], m["tid"][i]))]          # the fold order
    rt = (now - m["start"][i]) / 1000.0
    met = np.stack([rt, rt * m["cpus"][i], rt * m["mem"][i]])
    ranks = lambda n: [(p * n + 99) // 100 - 1 for p in (50, 75, 95, 99, 100)]
    out, lead = [], []
    n = len(i)
    for kind in range(4):
        user = m["user"][i] if kind >= 2 else np.full(n, -1)
        reason = m["reason"][i] if kind in (1, 2) else np.full(n, -1)
        k = np.lexsort((np.arange(n), reason, user))
        key = np.stack([user[k], reason[k]], 1)
        cut = np.flatnonzero(np.any(key[1:] != key[:-1], 1)) + 1
        for s, e in zip(np.concatenate([[0], cut]), np.concatenate([cut, [n]])):
            seg = met[:, k[s:e]]
            tot = [float(np.cumsum(seg[c])[-1]) for c in range(3)]
            if kind == 3:
                lead.append((int(key[s, 0]), tot))
            else:
                r = ranks(e - s)
                out.append((kind, int(key[s, 0]), int(key[s, 1]), e - s, tot,
                            [np.sort(seg[c])[r].tolist() for c in range(3)]))
    lc = sorted(((u, t[1]) for u, t in lead), key=lambda x: (-x[1], x[0]))[:10]
    lm = sorted(((u, t[2]) for u, t in lead), key=lambda x: (-x[1], x[0]))[:10]
    return out, lc, lm


def instance_stats_prof(a):
    """cook_state_instance_stats over resident pools (C2, config-#5 pool --c5-pool, or --c3-group N config-#3 pools as N
    handles) for status running and unknown over a window covering every row, against numpy over a host mirror.  A
    tenth of the rows carry one of three reason codes, a twentieth are unknown."""
    if a.c3_group > 0:
        ts = [traces.gen_config_pool("c3", p) for p in range(a.c3_group)]
        name = f"c3/0-{a.c3_group - 1}"
    else:
        ts = [traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)]
        name = a.pool if a.pool == "c2" else f"c5/{a.c5_pool}"
    rng = np.random.default_rng(a.seed)
    es, m = [], {k: [] for k in ("user", "tid", "pidx", "start", "cpus", "mem", "reason", "unknown")}
    for p, t in enumerate(ts):
        r = {k: np.asarray(v).copy() for k, v in t["cols"]["running"].items()}
        n = len(r["task_id"])
        e = GpuEngine(pool_name=f"instance-stats-{p}")
        e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**r)))
        reason = np.where(rng.random(n) < 0.1, rng.choice([1001, 1002, 2003], n), -1).astype(np.int32)
        unknown = (rng.random(n) < 0.05).astype(np.uint8)
        e.state_task_reason(r["task_id"], reason)
        e.state_task_facts(r["task_id"], unknown=unknown)
        es.append(e)
        for k, src in (("user", r["user"]), ("tid", r["task_id"]), ("start", r["start_time"]), ("cpus", r["cpus"]),
                       ("mem", r["mem"]), ("reason", reason), ("unknown", unknown)):
            m[k].append(np.asarray(src))
        m["pidx"].append(np.full(n, p))
    m = {k: np.concatenate(v) for k, v in m.items()}
    for k in ("cpus", "mem"):
        m[k] = m[k].astype(np.float64)
    now = int(m["start"].max()) + 1
    lo, hi = int(m["start"].min()), now
    print(json.dumps({"card": card(), "pools": name, "handles": len(ts), "running": int(len(m["tid"]))}), flush=True)
    for status in (abi.IS_RUNNING, abi.IS_UNKNOWN):
        for _ in range(3):   # warm-up: the carves and the first launches
            got = engine.state_instance_stats(es, now, status, lo, hi)
        dev, wall, host, same = [], [], [], True
        for _ in range(a.reps):
            w0 = time.perf_counter()
            got = engine.state_instance_stats(es, now, status, lo, hi)
            wall.append(time.perf_counter() - w0)
            st = got["stats"]
            dev.append(st["ms_h2d"] + st["ms_device"] + st["ms_d2h"])
            w0 = time.perf_counter()
            segs, lc, lm = host_instance_stats(m, now, status == abi.IS_UNKNOWN)
            host.append(time.perf_counter() - w0)
            f = lambda x: np.asarray(x, np.float64).view(np.int64).tolist()
            same = same and len(segs) == len(got["kind"]) and all(
                (int(got["kind"][d]), int(got["user"][d]), int(got["reason"][d]), int(got["count"][d])) == w[:4]
                and f(got["total"][d]) == f(w[4]) and f(got["pct"][d]) == f(w[5]) for d, w in enumerate(segs)) and \
                [(u, f([x])) for u, x in got["leaders_cpu"]] == [(u, f([x])) for u, x in lc] and \
                [(u, f([x])) for u, x in got["leaders_mem"]] == [(u, f([x])) for u, x in lm]
        print(json.dumps({"status": "unknown" if status == abi.IS_UNKNOWN else "running",
                          "selected": int(got["count"][0]) if len(got["count"]) else 0, "segments": len(got["kind"]),
                          "device_ms": round(float(np.median(dev)), 4), "wall_ms": round(1e3 * float(np.median(wall)), 4),
                          "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                          "numpy_wall_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same)}), flush=True)
    for e in es:
        e.close()


DAY_MS = 86_400_000


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return int(torch.cuda.mem_get_info(0)[0])


def history_stats_prof(a):
    """cook_state_history_stats over seeded histories against numpy over a host mirror (host_instance_stats with each
    row's start moved to -(end - start) and now = 0, so that its run time is end - start)."""
    if a.c3_group > 0:
        ts = [traces.gen_config_pool("c3", p) for p in range(a.c3_group)]
        name = f"c3/0-{a.c3_group - 1}"
    else:
        ts = [traces.gen_c2()]
        name = "c2"
    rng = np.random.default_rng(a.seed)
    H = len(ts)
    per = a.history_rows // H
    t_end = 1_700_000_000_000
    since = t_end - 31 * DAY_MS
    print(json.dumps({"card": card(), "pools": name, "handles": H, "rows": per * H}), flush=True)
    es, m = [], {k: [] for k in ("user", "tid", "pidx", "start", "end", "cpus", "mem", "reason", "ok")}
    f0 = free_bytes()
    next_tid = 1
    for p, t in enumerate(ts):
        r = t["cols"]["running"]
        k = rng.integers(0, len(r["task_id"]), per)   # C2's (or the pool's) users and shapes
        start = np.sort(rng.integers(since, t_end, per))
        cols = dict(task_id=np.arange(next_tid, next_tid + per, dtype=np.int64), user=np.asarray(r["user"])[k],
                    start_ms=start, end_ms=start + rng.integers(0, 2 * 3_600_000, per),
                    cpus=np.asarray(r["cpus"], np.float64)[k], mem=np.asarray(r["mem"], np.float64)[k],
                    success=(rng.random(per) < 0.7).astype(np.uint8),
                    reason_code=np.where(rng.random(per) < 0.3, rng.choice([1001, 2003, 3001], per), -1))
        next_tid += per
        e = GpuEngine(pool_name=f"history-stats-{p}")
        e.state_history_seed(since, **cols)
        es.append(e)
        for mk, ck in (("user", "user"), ("tid", "task_id"), ("start", "start_ms"), ("end", "end_ms"),
                       ("cpus", "cpus"), ("mem", "mem"), ("reason", "reason_code"), ("ok", "success")):
            m[mk].append(np.asarray(cols[ck]))
        m["pidx"].append(np.full(per, p))
    table = f0 - free_bytes()
    m = {k: np.concatenate(v) for k, v in m.items()}
    f = lambda x: np.asarray(x, np.float64).view(np.int64).tolist()
    for wname, lo, hi in (("all", since, t_end + 1), ("one day", t_end - DAY_MS, t_end + 1)):
        for status in (abi.IS_SUCCESS, abi.IS_FAILED):
            f1 = free_bytes()
            for _ in range(2):   # warm-up: the carves and the first launches
                got = engine.state_history_stats(es, status, lo, hi)
            scratch = f1 - free_bytes()
            sel = np.flatnonzero((m["start"] >= lo) & (m["start"] < hi))
            mirror = {"user": m["user"][sel], "tid": m["tid"][sel], "pidx": m["pidx"][sel],
                      "start": -(m["end"][sel] - m["start"][sel]), "cpus": m["cpus"][sel], "mem": m["mem"][sel],
                      "reason": m["reason"][sel], "unknown": m["ok"][sel]}
            dev, wall, host, same = [], [], [], True
            for _ in range(a.reps):
                w0 = time.perf_counter()
                got = engine.state_history_stats(es, status, lo, hi)
                wall.append(time.perf_counter() - w0)
                st = got["stats"]
                dev.append(st["ms_h2d"] + st["ms_device"] + st["ms_d2h"])
            w0 = time.perf_counter()
            segs, lc, lm = host_instance_stats(mirror, 0, int(status == abi.IS_SUCCESS))
            host.append(time.perf_counter() - w0)
            same = len(segs) == len(got["kind"]) and all(
                (int(got["kind"][d]), int(got["user"][d]), int(got["reason"][d]), int(got["count"][d])) == w[:4]
                and f(got["total"][d]) == f(w[4]) and f(got["pct"][d]) == f(w[5]) for d, w in enumerate(segs)) and \
                [(u, f([x])) for u, x in got["leaders_cpu"]] == [(u, f([x])) for u, x in lc] and \
                [(u, f([x])) for u, x in got["leaders_mem"]] == [(u, f([x])) for u, x in lm]
            print(json.dumps({"window": wname, "status": "success" if status == abi.IS_SUCCESS else "failed",
                              "selected": int(got["count"][0]) if len(got["count"]) else 0,
                              "segments": len(got["kind"]), "device_ms": round(float(np.median(dev)), 4),
                              "wall_ms": round(1e3 * float(np.median(wall)), 4), "h2d_bytes": st["h2d_bytes"],
                              "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                              "numpy_wall_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same),
                              "table_bytes": table, "scratch_bytes_grown": scratch}), flush=True)
    # a batch of 1000 finishes over the history of handle 0: cook_state_finish_history against cook_state_finish on a
    # twin without history, alternating
    e, twin = es[0], GpuEngine(pool_name="history-twin")
    t = ts[0]["cols"]["running"]
    res = {"finish_history": [], "finish": []}
    for rep in range(a.reps + 1):
        tid = np.arange(next_tid, next_tid + 1000, dtype=np.int64)
        next_tid += 1000
        run = dict(task_id=tid, job_id=tid + 10 ** 9, user=np.asarray(t["user"])[:1000],
                   priority=np.full(1000, 50, np.int32), start_time=np.full(1000, t_end - 1000, np.int64),
                   cpus=np.asarray(t["cpus"], np.float64)[:1000], mem=np.asarray(t["mem"], np.float64)[:1000],
                   gpus=np.zeros(1000))
        for x in (e, twin):
            x.state_apply(abi.make_delta(running=abi.make_tasks(**run)))
        end = np.full(1000, t_end, np.int64)
        ok = (np.arange(1000) % 2).astype(np.uint8)
        for kind, fn in (("finish_history", lambda: e.state_finish_history(tid, end, ok, None)),
                         ("finish", lambda: twin.state_finish(tid, end, ok))):
            w0 = time.perf_counter()
            fn()
            w = time.perf_counter() - w0
            st = (e if kind == "finish_history" else twin).last_stats(abi.PHASE_STATE)
            if rep:
                res[kind].append((st["ms_h2d"] + st["ms_device"], 1e3 * w, st["h2d_bytes"], st["n_launches"]))
    for kind, v in res.items():
        print(json.dumps({"call": kind, "batch": 1000, "history_rows": int(len(m["tid"]) // H),
                          "device_ms": round(float(np.median([x[0] for x in v])), 4),
                          "wall_ms": round(float(np.median([x[1] for x in v])), 4), "h2d_bytes": v[-1][2],
                          "n_launches": v[-1][3]}), flush=True)
    twin.close()
    # one advance dropping a day
    w0 = time.perf_counter()
    e.state_history_advance(since + DAY_MS)
    w = time.perf_counter() - w0
    st = e.last_stats(abi.PHASE_STATE)
    print(json.dumps({"call": "advance", "dropped_day": True, "device_ms": round(st["ms_device"], 4),
                      "wall_ms": round(1e3 * w, 4), "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"]}),
          flush=True)
    for x in es:
        x.close()


def host_match_metrics(ids, matched, prev, thr, cpus, mem, gpus, user, facts, gmodel, dtype, dreq, dlim, U):
    """The numpy and Python restatement over the host mirror's columns of the round's rows (take order): the per-user
    counts, the left folds (np.add.accumulate is sequential), the stable sorts, the keyed folds and the dict of
    counters the reference rebuilds each cycle."""
    out = {"ucons": np.bincount(user, minlength=U), "umat": np.bincount(user[matched], minlength=U)}
    out["tot"] = (np.add.accumulate(cpus)[-1], np.add.accumulate(mem)[-1])
    N = len(ids)
    pr = [(p * N + 99) // 100 - 1 for p in (50, 95, 100)]
    oc, om = np.argsort(cpus, kind="stable"), np.argsort(mem, kind="stable")
    out["pct"] = [cpus[oc[p]] for p in pr] + [mem[om[p]] for p in pr]
    out["largest"] = (int(oc[-1]), int(om[-1]))
    keys = []
    for kind, bit, code, val in ((abi.MM_GPUS, abi.JF_GPUS, gmodel, gpus), (abi.MM_DISK_REQUEST, abi.JF_DISK_REQUEST,
                                  dtype, dreq), (abi.MM_DISK_LIMIT, abi.JF_DISK_LIMIT, dtype, dlim)):
        has = (facts & bit) != 0
        for c in np.unique(code[has]):
            keys.append((kind, int(c), float(np.add.accumulate(val[has & (code == c)])[-1])))
    out["keys"] = keys
    ms = np.zeros(N, bool)
    ms[matched] = True
    cyc = {j: prev.get(j, 0) + 1 for j, m in zip(ids.tolist(), ms.tolist()) if not m}
    out["cycles"] = cyc
    over = [(j, cyc[j]) for j in ids.tolist() if cyc.get(j, 0) > thr]
    out["too_long"], out["first"] = len(over), over[:10]
    return out


def match_metrics_prof(a):
    """cook_state_match_metrics after each match of a resident pool (C2, or config-#5 pool --c5-pool) with every
    pending job considerable and a fifth of them carrying gpus or disk facts, against the numpy and Python
    restatement over a host mirror; each answer is compared bit for bit."""
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    jobs, pc, rc, users = t["jobs"], t["cols"]["pending"], t["cols"]["running"], t["users"]
    J, U = jobs.n, users.n_users
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    e = GpuEngine(pool_name="match-metrics")
    e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**{k: np.asarray(v) for k, v in rc.items()}),
                                 pending=store.soa(np.arange(J)), pending_priority=store.prio,
                                 pending_job_id=store.jid))
    rng = np.random.default_rng(a.seed)
    facts = np.where(rng.random(J) < 0.1, abi.JF_GPUS, 0) | np.where(
        rng.random(J) < 0.1, abi.JF_DISK | abi.JF_DISK_REQUEST | abi.JF_DISK_LIMIT, 0)
    facts = facts.astype(np.uint8)
    gmodel = rng.integers(-1, 4, J).astype(np.int32)
    dtype = rng.integers(-1, 2, J).astype(np.int32)
    dreq, dlim = rng.choice([1024.0, 2048.0, 0.1], J), rng.choice([4096.0, 0.3], J)
    e.state_job_facts(store.jid, facts, gpu_model=gmodel, disk_request=dreq, disk_limit=dlim, disk_type=dtype)
    e.state_rank(users)
    pos = {int(j): i for i, j in enumerate(store.jid)}
    cols = {n: np.asarray(store.c[n] if n in store.c else np.zeros(J), np.float64) for n in ("cpus", "mem", "gpus")}
    user = np.asarray(store.c["user"], np.int64)
    prm = traces.match_params(J)
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "jobs": J,
                      "offers": t["offers"].n, "users": U}), flush=True)
    prev, dev, wall, host, same = {}, [], [], [], True
    for rep in range(a.reps + 3):
        m = e.state_match(t["offers"], users, prm)
        ids = m["considerable"]
        matched = np.flatnonzero(m["assign"] >= 0)
        dropped = matched[::10]
        kept = np.setdiff1d(matched, dropped)
        w0 = time.perf_counter()
        got = e.state_match_metrics(U, dropped, unmatched_warn_cycles=2, key_cap=64)
        w = time.perf_counter() - w0
        r = np.array([pos[int(j)] for j in ids])
        w0 = time.perf_counter()
        h = host_match_metrics(ids, kept, prev, 2, cols["cpus"][r], cols["mem"][r], cols["gpus"][r], user[r], facts[r],
                               gmodel[r], dtype[r], dreq[r], dlim[r], U)
        hw = time.perf_counter() - w0
        prev = h["cycles"]
        f = lambda x: np.asarray(x, np.float64).view(np.int64).tolist()
        same = same and got["user_considerable"].tolist() == h["ucons"].tolist() and \
            got["user_matched"].tolist() == h["umat"].tolist() and \
            f([got["total_cpus"], got["total_mem"]]) == f(h["tot"]) and f(got["pct_cpus"] + got["pct_mem"]) == f(h["pct"]) \
            and (got["rows"][1]["position"], got["rows"][2]["position"]) == h["largest"] and \
            [(k, c, f([v])) for k, c, v in got["keys"]] == [(k, c, f([v])) for k, c, v in h["keys"]] and \
            got["too_long"] == h["too_long"] and got["first"] == h["first"]
        if rep >= 3:   # the first calls carve and load the kernels
            st = got["stats"]
            dev.append(st["ms_h2d"] + st["ms_device"] + st["ms_d2h"])
            wall.append(w)
            host.append(hw)
    print(json.dumps({"considerable": int(got["considerable"]), "matched": int(got["matched"]), "keys": len(got["keys"]),
                      "too_long": got["too_long"], "device_ms": round(float(np.median(dev)), 4),
                      "wall_ms": round(1e3 * float(np.median(wall)), 4), "h2d_bytes": st["h2d_bytes"],
                      "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                      "host_restatement_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same)}),
          flush=True)
    e.close()


def host_list_jobs(mirror, user, start, end, limit):
    """get-active-jobs-by-user-and-state for waiting and running over the host mirror (one handle, no pool filter,
    every custom executor kept): [(state, job id, submit ms)], each state by job id and cut to limit."""
    out = []
    for state, m in ((abi.LJ_WAITING, mirror["pending"]), (abi.LJ_RUNNING, mirror["running"])):
        sel = m["user"] == user
        jid, sub = m["jid"][sel], m["submit"][sel]
        if state == abi.LJ_RUNNING:   # one entry per job: its greatest task id
            o = np.lexsort((-m["tid"][sel], jid))
            jid, sub = jid[o], sub[o]
            first = np.ones(len(jid), bool)
            first[1:] = jid[1:] != jid[:-1]
            jid, sub = jid[first], sub[first]
        ok = (sub >= start) & (sub < end)
        jid, sub = jid[ok], sub[ok]
        o = np.argsort(jid, kind="stable")[:limit]
        out += [(state, int(j), int(t)) for j, t in zip(jid[o], sub[o])]
    return out


def list_prof(a):
    """cook_state_list_jobs on a resident pool (C2, or config-#5 pool --c5-pool) with list facts on every job, for the
    user with the most rows and one with the fewest, both states, a 24 h window covering every row, limits
    Integer/MAX_VALUE and 150, against numpy over a host mirror; each answer is compared exactly."""
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    jobs, pc, rc = t["jobs"], t["cols"]["pending"], t["cols"]["running"]
    J = jobs.n
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    e = GpuEngine(pool_name="list")
    run = {k: np.asarray(v) for k, v in rc.items()}
    e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**run), pending=store.soa(np.arange(J)),
                                 pending_priority=store.prio, pending_job_id=store.jid))
    rng = np.random.default_rng(a.seed)
    day = 24 * 3600 * 1000
    t0 = 1_700_000_000_000
    ids = np.unique(np.concatenate([store.jid, run["job_id"]]))
    submit = t0 + rng.integers(0, day, len(ids))
    e.state_list_facts(ids, submit, np.full(len(ids), -1, np.int32), np.zeros(len(ids), np.int32))
    sub_of = dict(zip(ids.tolist(), submit.tolist()))
    mirror = {"pending": {"user": np.asarray(store.c["user"]), "jid": store.jid.copy(),
                          "submit": np.array([sub_of[int(j)] for j in store.jid], np.int64)},
              "running": {"user": run["user"], "jid": run["job_id"], "tid": run["task_id"],
                          "submit": np.array([sub_of[int(j)] for j in run["job_id"]], np.int64)}}
    counts = np.bincount(np.concatenate([mirror["pending"]["user"], mirror["running"]["user"]]))
    heavy, light = int(np.argmax(counts)), int(np.flatnonzero(counts == counts[counts > 0].min())[0])
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "pending": J,
                      "running": len(run["task_id"]), "heavy_user_rows": int(counts[heavy]),
                      "light_user_rows": int(counts[light])}), flush=True)
    for who, user in (("heavy", heavy), ("light", light)):
        for limit in ((1 << 31) - 1, 150):
            dev, wall, host, same = [], [], [], True
            for rep in range(a.reps + 3):
                w0 = time.perf_counter()
                got = engine.state_list_jobs([e], user, abi.LJ_WAITING | abi.LJ_RUNNING, t0, t0 + day, limit=limit,
                                             cap=int(counts[user]) + 1)
                w = time.perf_counter() - w0
                w0 = time.perf_counter()
                want = host_list_jobs(mirror, user, t0, t0 + day, limit)
                hw = time.perf_counter() - w0
                same = same and got["missing"] == 0 and \
                    [(int(s), int(j), int(x)) for s, j, x in zip(got["state"], got["job_id"], got["submit_ms"])] == want
                if rep >= 3:   # the first calls carve and load the kernels
                    st = got["stats"]
                    dev.append(st["ms_h2d"] + st["ms_device"] + st["ms_d2h"])
                    wall.append(w)
                    host.append(hw)
            print(json.dumps({"user": who, "rows": int(counts[user]), "limit": limit, "entries": len(got["job_id"]),
                              "device_ms": round(float(np.median(dev)), 4),
                              "wall_ms": round(1e3 * float(np.median(wall)), 4), "h2d_bytes": st["h2d_bytes"],
                              "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                              "host_restatement_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same)}),
                  flush=True)
    e.close()


def host_list_completed(m, user, state, start, end, lo, hi, limit):
    """get-completed-jobs-by-user over the host mirror of one log: each job's latest record (stamp, then row), REOPENED
    dropped, the state, window and id window on it, ascending job id cut to limit: [(job id, submit ms)]."""
    sel = np.flatnonzero((m["user"] == user) & (m["jid"] >= lo) & (m["jid"] < hi))
    o = sel[np.lexsort((-sel, -m["stamp"][sel], m["jid"][sel]))]
    first = np.ones(len(o), bool)
    first[1:] = m["jid"][o[1:]] != m["jid"][o[:-1]]
    o = o[first]
    k, s = m["kind"][o], m["submit"][o]
    ok = (k != abi.CJ_REOPENED) & (s >= start) & (s < end)
    if state != abi.LC_COMPLETED:
        ok &= k == state
    o = o[ok][:limit]
    return list(zip(m["jid"][o].tolist(), m["submit"][o].tolist()))


def list_completed_prof(a):
    """cook_state_list_completed over a synthetic log of --completed-rows records over 32 days (Zipf users as in
    traces.py; 5 % of the jobs reopened, most of those completed again; 2 % of the records sent twice), for the
    heaviest user and a light one, 24 h and 7 d windows ending at the log's end, limits Integer/MAX_VALUE and 150,
    states completed and success, against numpy over a host mirror; then one cook_state_completed_record of 1000 rows
    and one cook_state_completed_advance that drops a day."""
    rng = np.random.default_rng(a.seed)
    t_end = 1_700_000_000_000
    since = t_end - 32 * DAY_MS
    J = int(a.completed_rows / 1.1)
    submit = np.sort(rng.integers(since, t_end, J))
    jid = np.arange(1, J + 1, dtype=np.int64)          # entity ids grow with submit time
    user = traces._zipf_owner(rng, J, 1000)
    spool = np.full(J, -1, np.int32)
    cex = rng.choice(np.array([-1, 0, 1], np.int32), J, p=[0.1, 0.85, 0.05])
    done = submit + rng.integers(1000, 2 * 3_600_000, J)
    recs = [(np.arange(J), done, rng.choice(np.array([abi.CJ_SUCCESS, abi.CJ_FAILED], np.uint8), J, p=[0.7, 0.3]))]
    ro = np.flatnonzero(rng.random(J) < 0.05)           # reopened
    recs.append((ro, done[ro] + rng.integers(1, DAY_MS, len(ro)), np.full(len(ro), abi.CJ_REOPENED, np.uint8)))
    rc = ro[rng.random(len(ro)) < 0.6]                 # completed again
    recs.append((rc, done[rc] + DAY_MS + rng.integers(1, DAY_MS, len(rc)),
                 rng.choice(np.array([abi.CJ_SUCCESS, abi.CJ_FAILED], np.uint8), len(rc))))
    du = np.flatnonzero(rng.random(J) < 0.02)           # the first record sent twice
    recs.append((du, done[du], recs[0][2][du]))
    e = GpuEngine(pool_name="list-completed")
    e.state_completed_seed(since)
    m = {k: [] for k in ("jid", "stamp", "user", "submit", "kind", "cex")}
    for idx, stamp, kind in recs:   # one batch per occurrence (a job at most once per batch), in stamp order
        o = np.argsort(stamp, kind="stable")
        idx, stamp, kind = idx[o], stamp[o], kind[o]
        for c0 in range(0, len(idx), 1 << 21):
            s = slice(c0, c0 + (1 << 21))
            i = idx[s]
            e.state_completed_record(jid[i], stamp[s], user[i], submit[i], spool[i], cex[i], kind[s])
            for k, v in (("jid", jid[i]), ("stamp", stamp[s]), ("user", user[i]), ("submit", submit[i]),
                         ("kind", kind[s]), ("cex", cex[i])):
                m[k].append(v)
    m = {k: np.concatenate(v) for k, v in m.items()}
    counts = np.bincount(m["user"])
    heavy = int(np.argmax(counts))
    light = int(np.flatnonzero(counts == np.sort(counts[counts > 0])[len(counts[counts > 0]) // 10])[0])
    print(json.dumps({"card": card(), "records": len(m["jid"]), "jobs": J, "days": 32, "heavy_user_records":
                      int(counts[heavy]), "light_user_records": int(counts[light])}), flush=True)
    hour = 3_600_000
    for who, u in (("heavy", heavy), ("light", light)):
        for wname, w in (("24h", DAY_MS), ("7d", 7 * DAY_MS)):
            start, end = t_end - w, t_end
            lo, hi = int(jid[np.searchsorted(submit, start - hour)]), J + 1
            for state, sname in ((abi.LC_COMPLETED, "completed"), (abi.LC_SUCCESS, "success")):
                for limit in ((1 << 31) - 1, 150):
                    dev, wall, host, same = [], [], [], True
                    for rep in range(a.reps + 2):
                        w0 = time.perf_counter()
                        got = engine.state_list_completed([e], u, state, start, end, lo, hi, limit=limit,
                                                          cap=int(counts[u]) + 1)
                        wl = time.perf_counter() - w0
                        if rep < 2:   # the first calls carve and load the kernels
                            continue
                        st = got["stats"]
                        dev.append(st["ms_h2d"] + st["ms_device"] + st["ms_d2h"])
                        wall.append(wl)
                        if rep < 5:
                            w0 = time.perf_counter()
                            want = host_list_completed(m, u, state, start, end, lo, hi, limit)
                            host.append(time.perf_counter() - w0)
                            same = same and list(zip(got["job_id"].tolist(), got["submit_ms"].tolist())) == want
                    print(json.dumps({"user": who, "window": wname, "state": sname, "limit": limit,
                                      "entries": len(got["job_id"]), "device_ms": round(float(np.median(dev)), 4),
                                      "wall_ms": round(1e3 * float(np.median(wall)), 4), "h2d_bytes": st["h2d_bytes"],
                                      "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"],
                                      "numpy_ms": round(1e3 * float(np.median(host)), 4), "identical": bool(same)}),
                          flush=True)
    # one record of 1000 new completions, and one advance that drops a day
    res = []
    for rep in range(a.reps + 1):
        n0 = J + 1 + 1000 * rep
        nj = np.arange(n0, n0 + 1000, dtype=np.int64)
        w0 = time.perf_counter()
        e.state_completed_record(nj, np.full(1000, t_end + rep, np.int64), user[:1000], np.full(1000, t_end, np.int64),
                                 spool[:1000], cex[:1000], np.full(1000, abi.CJ_SUCCESS, np.uint8))
        wl = time.perf_counter() - w0
        st = e.last_stats(abi.PHASE_STATE)
        if rep:
            res.append((st["ms_h2d"] + st["ms_device"], 1e3 * wl, st["h2d_bytes"]))
    print(json.dumps({"call": "record", "batch": 1000, "log_rows": len(m["jid"]) + 1000 * a.reps,
                      "device_ms": round(float(np.median([x[0] for x in res])), 4),
                      "wall_ms": round(float(np.median([x[1] for x in res])), 4), "h2d_bytes": res[-1][2]}), flush=True)
    w0 = time.perf_counter()
    e.state_completed_advance(since + DAY_MS)
    wl = time.perf_counter() - w0
    st = e.last_stats(abi.PHASE_STATE)
    print(json.dumps({"call": "advance", "dropped_day": True, "device_ms": round(st["ms_device"], 4),
                      "wall_ms": round(1e3 * wl, 4), "d2h_bytes": st["d2h_bytes"], "n_launches": st["n_launches"]}),
          flush=True)
    e.close()


def requeued_soa(store, rows, host):
    """The host path cook_state_status replaces: the pending rows of failed jobs rebuilt from the host mirror with
    reserved_host -1 and the failed host appended to the novel-host list (unless -1 or already listed)."""
    soa = store.soa(rows)
    off, val = soa.col("novel_off"), soa.col("novel_host")
    lists = [val[off[i]:off[i + 1]].tolist() if off is not None else [] for i in range(len(rows))]
    for lst, h in zip(lists, host.tolist()):
        if h != -1 and h not in lst:
            lst.append(h)
    noff = np.zeros(len(rows) + 1, np.int32)
    noff[1:] = np.cumsum([len(x) for x in lists])
    nval = np.asarray([h for x in lists for h in x] or [0], np.int32)
    return _with(soa, reserved_host=np.full(len(rows), -1, np.int32), novel_off=noff, novel_host=nval)


def status_prof(a):
    """cook_state_status against the host path it replaces (requeued rows rebuilt from a host mirror, then
    cook_state_finish_history and a cook_state_apply upsert), alternated in one run on two handles holding the same
    rows (C2, or config-#5 pool --c5-pool with --pool c5): per rep, a launch of --status-batch jobs on both (with and
    without retry facts), then their failures with retries left.  Every requeued job is parked, and the two handles'
    digests must stay equal."""
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    jobs, pc = t["jobs"], t["cols"]["pending"]
    J, B = jobs.n, a.status_batch
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    print(json.dumps({"card": card(), "pool": a.pool, "jobs": J, "batch": B}), flush=True)
    res, twin = GpuEngine(pool_name="status"), GpuEngine(pool_name="twin")
    for e in (res, twin):
        e.state_apply(abi.make_delta(reset=True, pending=store.soa(np.arange(J)), pending_priority=store.prio,
                                     pending_job_id=store.jid))
    res.state_retry_config(5, [])
    res.state_retry_facts(store.jid, np.full(J, 1000, np.int32), np.zeros(J, np.uint8))
    rng = np.random.default_rng(a.seed)
    n_hosts = max(t["offers"].n, 1)
    tid = 1 << 40
    out = {"launch_facts": [], "launch_plain": [], "status": [], "host_path": []}
    order = rng.permutation(J)   # each job fails once: the host mirror's lists stay the trace's
    for rep in range(a.reps + 1):
        rows = np.sort(order[rep * B:(rep + 1) * B])
        jid, host = store.jid[rows], rng.integers(0, n_hosts, B).astype(np.int32)
        tids = np.arange(tid, tid + B, dtype=np.int64)
        tid += B
        start = np.full(B, 1_700_000_000_000, np.int64)
        end, ok, reason = start + 1000, np.zeros(B, np.uint8), np.full(B, -1, np.int32)
        for e, kind in ((res, "launch_facts"), (twin, "launch_plain"))[::1 if rep % 2 else -1]:
            t0 = time.perf_counter()
            e.state_launch(jid, tids, start, host)
            wall = time.perf_counter() - t0
            if rep:
                st = e.last_stats(abi.PHASE_STATE)
                out[kind].append((wall * 1e3, st["ms_device"], st["h2d_bytes"], st["n_launches"]))

        def host_path():
            soa = requeued_soa(store, rows, host)
            twin.state_finish_history(tids, end, ok, reason)
            twin.state_apply(abi.make_delta(pending=soa, pending_priority=store.prio[rows], pending_job_id=jid))

        for kind in (("status", "host_path") if rep % 2 else ("host_path", "status")):
            t0 = time.perf_counter()
            if kind == "status":
                oc, _ = res.state_status(tids, ok, end, reason)
                assert (oc == abi.JOB_WAITING).all()
            else:
                host_path()
            if rep:
                out[kind].append((time.perf_counter() - t0) * 1e3)
        da, db = res.state_digest(), twin.state_digest()
        assert da["pending"] == db["pending"] and da["running"] == db["running"], "the two handles differ"
    med = lambda xs, k=None: float(np.median([x[k] if k is not None else x for x in xs]))   # noqa: E731
    print(json.dumps({
        "status_wall_ms": med(out["status"]), "host_path_wall_ms": med(out["host_path"]),
        "launch_with_facts": {"wall_ms": med(out["launch_facts"], 0), "device_ms": med(out["launch_facts"], 1),
                              "h2d": out["launch_facts"][-1][2], "launches": out["launch_facts"][-1][3]},
        "launch_without_facts": {"wall_ms": med(out["launch_plain"], 0), "device_ms": med(out["launch_plain"], 1),
                                 "h2d": out["launch_plain"][-1][2], "launches": out["launch_plain"][-1][3]},
        "reps": a.reps, "identical": True}), flush=True)


def rank_quota_prof(a):
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    pc, rc0, users = t["cols"]["pending"], t["cols"]["running"], t["users"]
    jobs = t["jobs"]
    J, R = jobs.n, len(rc0["task_id"])
    print(json.dumps({"card": card(), "pool": a.pool if a.pool == "c2" else f"c5/{a.c5_pool}", "pending": J,
                      "running": R, "lib": os.environ.get("COOK_GPU_LIB", "in-tree")}), flush=True)
    pend = dict(pending=Jobs(jobs, pc["priority"], pc["job_id"]).soa(np.arange(J)), pending_priority=pc["priority"],
                pending_job_id=pc["job_id"])
    for regime in ("grid", "off"):
        run = {k: np.asarray(v).copy() for k, v in rc0.items()}
        if regime == "off":
            run["cpus"] = run["cpus"] + 0.1
            run["mem"] = run["mem"] / 3.0
        e = GpuEngine(pool_name="rank-quota")
        e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**run), **pend))
        total = e.state_usage(users.n_users)["pool"]
        q = e.state_rank(users)
        half = float(np.sum(jobs.col("cpus")[np.searchsorted(pc["job_id"], q[:len(q) // 2])]))
        pq = abi.make_pool_quota({"count": 1e18, "cpus": total[1] + half, "mem": 1e18, "gpus": 1e18})
        for kind, kw in (("no_quota", {}), ("pool_quota", dict(pool_quota=pq))):
            dev, wall = [], []
            n = 0
            for rep in range(a.reps + 1):
                w0 = time.perf_counter()
                n = len(e.state_rank(users, **kw))
                w = time.perf_counter() - w0
                st = e.last_stats(abi.PHASE_RANK)
                if rep:
                    dev.append(st["ms_device"])
                    wall.append(1e3 * w)
            print(json.dumps({"regime": regime, "kind": kind, "queue": n,
                              "ms_device_median": round(float(np.median(dev)), 3), "ms_device_min": round(min(dev), 3),
                              "wall_ms_median": round(float(np.median(wall)), 3), "wall_ms_min": round(min(wall), 3),
                              "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                              "n_launches": st["n_launches"]}), flush=True)
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pool", choices=("c2", "c5"), default="c2")
    ap.add_argument("--c5-pool", type=int, default=5)
    ap.add_argument("--rebalance", action="store_true")
    ap.add_argument("--launch", action="store_true")
    ap.add_argument("--c4-pool", type=int, default=0)
    ap.add_argument("--cycles", type=int, default=6)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--usage", action="store_true")
    ap.add_argument("--cotasks", action="store_true")
    ap.add_argument("--c3-pool", type=int, default=-1,
                    help="--cotasks: a config-#3 pool (-1: the smaller c3-shaped pool); --derived: a config-#3 pool "
                         "instead of --pool")
    ap.add_argument("--derived", action="store_true")
    ap.add_argument("--offers", action="store_true", help="live offers against the host's lease cache (C2 or --c3-pool)")
    ap.add_argument("--considerable", action="store_true")
    ap.add_argument("--audit", action="store_true")
    ap.add_argument("--user-stats", action="store_true")
    ap.add_argument("--c3-group", type=int, default=0, help="--user-stats: a quota group of config-#3 pools 0 .. N-1")
    ap.add_argument("--rank-quota", action="store_true")
    ap.add_argument("--sweeps", action="store_true", help="cook_state_sweep against numpy over a host mirror")
    ap.add_argument("--reps", type=int, default=20, help="--audit, --rank-quota, --sweeps: timed calls per kind")
    ap.add_argument("--unscheduled", action="store_true", help="cook_state_unscheduled against numpy over a host mirror")
    ap.add_argument("--user-usage", action="store_true",
                    help="cook_state_user_usage against numpy over a host mirror (--c3-group N: N config-#3 pools)")
    ap.add_argument("--instance-stats", action="store_true",
                    help="cook_state_instance_stats against numpy over a host mirror (--c3-group N: N config-#3 pools)")
    ap.add_argument("--history-stats", action="store_true",
                    help="cook_state_history_stats against numpy over a host mirror (--c3-group N: N config-#3 pools)")
    ap.add_argument("--history-rows", type=int, default=1_000_000, help="--history-stats: the finished rows in all")
    ap.add_argument("--status", action="store_true",
                    help="cook_state_status against rebuilding and re-sending the rows (C2 or --pool c5)")
    ap.add_argument("--status-batch", type=int, default=1000, help="--status: the launches and failures per rep")
    ap.add_argument("--list", action="store_true",
                    help="cook_state_list_jobs against numpy over a host mirror (C2 or --pool c5)")
    ap.add_argument("--list-completed", action="store_true",
                    help="cook_state_list_completed over a synthetic log against numpy over a host mirror")
    ap.add_argument("--completed-rows", type=int, default=10_000_000, help="--list-completed: the log's records")
    ap.add_argument("--match-metrics", action="store_true",
                    help="cook_state_match_metrics after each match against numpy over a host mirror (C2 or --pool c5)")
    a = ap.parse_args()
    if a.list_completed:
        return list_completed_prof(a)
    if a.list:
        return list_prof(a)
    if a.status:
        return status_prof(a)
    if a.match_metrics:
        return match_metrics_prof(a)
    if a.history_stats:
        return history_stats_prof(a)
    if a.instance_stats:
        return instance_stats_prof(a)
    if a.user_usage:
        return user_usage_prof(a)
    if a.unscheduled:
        return unscheduled_prof(a)
    if a.sweeps:
        return sweeps_prof(a)
    if a.rank_quota:
        return rank_quota_prof(a)
    if a.audit:
        return audit_prof(a)
    if a.user_stats:
        return user_stats_prof(a)
    if a.considerable:
        return considerable_prof(a)
    if a.rebalance:
        return rebalance(a)
    if a.usage:
        return usage(a)
    if a.cotasks:
        return cotasks_prof(a)
    if a.derived:
        return derived_prof(a)
    if a.offers:
        return offers_prof(a)
    t = traces.gen_c2() if a.pool == "c2" else traces.gen_config_pool("c5", a.c5_pool)
    jobs, pc, rc = t["jobs"], t["cols"]["pending"], t["cols"]["running"]
    J = jobs.n
    print(json.dumps({"card": card(), "pool": a.pool, "jobs": J, "offers": t["offers"].n, "running": len(rc["task_id"])}),
          flush=True)
    rng = np.random.default_rng(a.seed)
    J0 = int(J * 0.8)                       # the rest are submitted during the run
    store = Jobs(jobs, pc["priority"], pc["job_id"])
    alive = np.zeros(J, bool)
    alive[:J0] = True
    nxt = J0
    run = {k: np.asarray(v).copy() for k, v in rc.items()}
    next_tid = int(run["task_id"].max()) + 10 if len(run["task_id"]) else 10
    users, offers, groups = t["users"], t["offers"], t.get("groups")
    params = traces.match_params(J, host_lifetime_mins=t.get("host_lifetime_mins", 0))
    max_ports = int(jobs.col("ports").max()) if jobs.col("ports") is not None else 0
    # --launch: `host` is the twin resident handle that receives launches as deltas
    res, host = GpuEngine(pool_name="resident"), GpuEngine(pool_name="twin" if a.launch else "host")
    pos_of = {int(j): i for i, j in enumerate(store.jid)}
    next_jid = int(store.jid.max()) + 10

    def pend_delta(rows):
        return dict(pending=store.soa(rows), pending_priority=store.prio[rows], pending_job_id=store.jid[rows])

    init =abi.make_delta(reset=True, running=abi.make_tasks(**run), **pend_delta(np.flatnonzero(alive)))
    for e in (res, host) if a.launch else (res,):
        e.state_apply(init)
    placed = np.zeros(0, np.int64)
    placed_host = np.zeros(0, np.int32)
    for cycle in range(a.cycles):
        # ---- the batch
        launch_rows = np.array([pos_of[int(j)] for j in placed], np.int64)
        n_fin = int(len(run["task_id"]) * 0.03)
        fin = rng.choice(len(run["task_id"]), n_fin, replace=False) if n_fin else np.zeros(0, np.int64)
        fin_ids = run["task_id"][fin]
        keep = np.ones(len(run["task_id"]), bool)
        keep[fin] = False
        sc = store.c
        lt = {"user": sc["user"][launch_rows], "priority": store.prio[launch_rows],
              "start_time": np.full(len(launch_rows), 1_700_000_000_000 + cycle, np.int64),
              "task_id": next_tid + 2 * np.arange(len(launch_rows), dtype=np.int64), "job_id": store.jid[launch_rows].copy(),
              "cpus": sc["cpus"][launch_rows], "mem": sc["mem"][launch_rows], "gpus": sc["gpus"][launch_rows]}
        next_tid += 2 * len(launch_rows) + 2
        launched_ids = store.jid[launch_rows].copy()
        # as many submissions as launches + finishes: a launched job's row comes back under a new job id (same
        # shape), the finishes are made up from the rows not yet submitted
        store.jid[launch_rows] = next_jid + 2 * np.arange(len(launch_rows), dtype=np.int64)
        next_jid += 2 * len(launch_rows) + 2
        pos_of.update({int(j): int(i) for j, i in zip(store.jid[launch_rows], launch_rows)})
        n_new = min(n_fin, J - nxt)
        sub = np.concatenate([launch_rows, np.arange(nxt, nxt + n_new)]).astype(np.int64)
        nxt += n_new
        n_sub = len(sub)
        alive[sub] = True
        live = np.flatnonzero(alive & ~np.isin(np.arange(J), sub))
        chg = rng.choice(live, min(len(live), max(1, len(live) // 1000)), replace=False)
        store.prio[chg] = rng.choice(np.array([10, 50, 90], np.int32), len(chg))
        up = np.concatenate([sub, chg])
        run = {k: np.concatenate([v[keep], lt[k]]) for k, v in run.items()}
        if a.launch:
            placed, placed_host = launch_cycle(cycle, res, host, launched_ids, lt, placed_host,
                                               abi.make_delta(running_rm=fin_ids, **pend_delta(up)),
                                               (users, offers, params, groups, max_ports))
            continue
        d = abi.make_delta(running=abi.make_tasks(**lt) if len(launch_rows) else None, pending_rm=launched_ids,
                           running_rm=fin_ids, **pend_delta(up))
        w0 = time.perf_counter()
        res.state_apply(d)
        w_apply = time.perf_counter() - w0
        st_apply = res.last_stats(abi.PHASE_STATE)
        # ---- resident arm
        w0 = time.perf_counter()
        q = res.state_rank(users)
        w_rank = time.perf_counter() - w0
        rs_rank = res.last_stats(abi.PHASE_RANK)
        w0 = time.perf_counter()
        mr = res.state_match(offers, users, params, groups=groups, max_ports=max_ports)
        w_match = time.perf_counter() - w0
        # ---- host arm on the same rows
        rows = np.flatnonzero(alive)
        hj = store.soa(rows)
        hp = abi.make_tasks(user=sc["user"][rows], priority=store.prio[rows], start_time=np.full(len(rows), abi.INT64_MAX),
                            task_id=np.full(len(rows), -1, np.int64), job_id=store.jid[rows], cpus=sc["cpus"][rows],
                            mem=sc["mem"][rows], gpus=sc["gpus"][rows])
        hr = abi.make_tasks(**run)
        w0 = time.perf_counter()
        r = host.rank(hr, hp, users)
        hw_rank = time.perf_counter() - w0
        hs_rank = host.last_stats(abi.PHASE_RANK)
        w0 = time.perf_counter()
        mh = host.match(r["ranked"], hj, offers, users, params, groups=groups, max_ports=max_ports)
        hw_match = time.perf_counter() - w0
        same = (np.array_equal(q, store.jid[rows][r["ranked"]]) and
                np.array_equal(mr["considerable"], store.jid[rows][mh["considerable"]]) and
                all(np.array_equal(mr[k], mh[k]) for k in ("assign", "ports", "fail")))
        placed = mr["considerable"][mr["assign"] >= 0]

        def ms(s):
            return {k: round(s[k], 3) for k in ("ms_h2d", "ms_device", "ms_d2h")} if "ms_device" in s else \
                {k: round(s[k], 3) for k in ("ms_h2d", "ms_considerable", "ms_match", "ms_d2h")}

        print(json.dumps({
            "cycle": cycle, "pending": int(alive.sum()), "running": len(run["task_id"]),
            "batch": {"launched": len(launch_rows), "finished": n_fin, "submitted": n_sub, "reprioritised": len(chg)},
            "resident": {"apply": {**ms(st_apply), "wall_ms": round(1e3 * w_apply, 3), "h2d_bytes": st_apply["h2d_bytes"]},
                         "rank": {**ms(rs_rank), "wall_ms": round(1e3 * w_rank, 3), "h2d_bytes": rs_rank["h2d_bytes"]},
                         "match": {**ms(mr["stats"]), "wall_ms": round(1e3 * w_match, 3),
                                   "h2d_bytes": mr["stats"]["h2d_bytes"]}},
            "host": {"rank": {**ms(hs_rank), "wall_ms": round(1e3 * hw_rank, 3), "h2d_bytes": hs_rank["h2d_bytes"]},
                     "match": {**ms(mh["stats"]), "wall_ms": round(1e3 * hw_match, 3),
                               "h2d_bytes": mh["stats"]["h2d_bytes"]}},
            "identical": bool(same), "n_matched": int(mr["stats"]["n_matched"])}), flush=True)
    res.close()
    host.close()


if __name__ == "__main__":
    main()
