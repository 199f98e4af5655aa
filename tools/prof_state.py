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
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cook_b200 import abi, traces  # noqa: E402
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
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
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
    ap.add_argument("--considerable", action="store_true")
    a = ap.parse_args()
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
