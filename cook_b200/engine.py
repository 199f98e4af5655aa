"""Thin call layer over the C ABI (include/cook_gpu.h).

`GpuEngine` drives libcookgpu.so (the product).  The same call shapes are
reused by oracle/pyoracle.py for the CPU oracle so that tests can diff the two;
this module itself never touches the oracle and has no CPU fallback: if the CUDA
library is missing or no device is present, construction raises.
"""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcookgpu.so")


class CookError(RuntimeError):
    def __init__(self, code, msg=""):
        super().__init__(f"cook_gpu error {code}: {msg}")
        self.code = code


def _empty_tasks():
    z32 = np.zeros(1, np.int32)
    z64 = np.zeros(1, np.int64)
    zf = np.zeros(1, np.float64)
    t = abi.TasksSoA(n=0, user=z32, priority=z32, start_time=z64, task_id=z64, job_id=z64,
                     cpus=zf, mem=zf, gpus=zf)
    return t


class _CallShapes:
    """Argument packing shared by the GPU engine and the oracle wrapper."""

    @staticmethod
    def rank_buffers(running, pending):
        n = running.n + pending.n
        return (np.zeros(max(pending.n, 1), np.int32), C.c_int32(0),
                np.full(max(n, 1), np.nan, np.float64), np.zeros(max(n, 1), np.int32), C.c_int32(0))

    @staticmethod
    def match_buffers(params, max_ports):
        k = max(params.num_considerable, 1)
        return (np.full(k, -1, np.int32), np.full(k, -1, np.int32),
                np.full(k * max(max_ports, 1), -1, np.int32), np.zeros(k, np.uint8),
                abi.MatchStats())


def load_library(path=None):
    # COOK_GPU_LIB: A/B builds of the same library (tools/ only); never a CPU fallback
    path = path or os.environ.get("COOK_GPU_LIB", LIB_PATH)
    if not os.path.exists(path):
        raise FileNotFoundError(
            f"{path} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(path)
    lib.cook_gpu_version.restype = C.c_char_p
    for name in ("cook_gpu_init", "cook_gpu_shutdown", "cook_pool_open", "cook_pool_close",
                 "cook_last_error", "cook_rank", "cook_match", "cook_rebalance",
                 "cook_allgather_usage", "cook_last_stats", "cook_comm_unique_id", "cook_comm_init",
                 "cook_comm_destroy", "cook_exchange_usage", "cook_exchange_usage_batch", "cook_rebalance_trace",
                 "cook_match_failures", "cook_state_apply", "cook_state_rank", "cook_state_match",
                 "cook_state_rebalance", "cook_state_launch", "cook_state_patch", "cook_state_usage",
                 "cook_state_cotasks", "cook_state_match_derived", "cook_state_rebalance_derived",
                 "cook_state_considerable", "cook_state_rank_offensive"):
        getattr(lib, name).restype = C.c_int32
    for name, argtypes in abi.ARGTYPES.items():
        getattr(lib, name).argtypes = argtypes
    return lib


class GpuEngine:
    """One Cook pool bound to one GPU.  Not re-entrant (same contract as
    `(locking fenzo ...)`, scheduler/scheduler.clj:665)."""

    def __init__(self, pool_name="no-pool", dru_mode=0, device=0, lib=None):
        self.lib = lib or load_library()
        self.ctx = C.c_void_p()
        rc = self.lib.cook_gpu_init(None, C.byref(self.ctx))
        if rc != 0:
            raise CookError(rc, "cook_gpu_init failed (no CUDA device? there is no CPU fallback)")
        self.pool = C.c_void_p()
        rc = self.lib.cook_pool_open(self.ctx, pool_name.encode(), int(dru_mode), int(device),
                                     C.byref(self.pool))
        if rc != 0:
            raise CookError(rc, "cook_pool_open failed")
        self.dru_mode = dru_mode

    def close(self):
        if getattr(self, "pool", None):
            self.lib.cook_pool_close(self.pool)
            self.pool = None
        if getattr(self, "ctx", None):
            self.lib.cook_gpu_shutdown(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self, rc):
        buf = C.create_string_buffer(512)
        self.lib.cook_last_error(self.pool, buf, 512)
        raise CookError(rc, buf.value.decode(errors="replace"))

    # -- R1-R7 -------------------------------------------------------------
    def rank(self, running, pending, users, pool_quota=None, group_quota=None,
             group_usage=None, params=None):
        running = running or _empty_tasks()
        pool_quota = pool_quota or abi.make_pool_quota(None)
        group_quota = group_quota or abi.make_pool_quota(None)
        params = params or abi.RankParams(100, 0, 0.0, 0.0)
        gu = np.ascontiguousarray(group_usage if group_usage is not None else np.zeros(4), np.float64)
        ranked, n, dru, order, on = _CallShapes.rank_buffers(running, pending)
        rc = self.lib.cook_rank(self.pool, C.byref(running), C.byref(pending), C.byref(users),
                                C.byref(pool_quota), C.byref(group_quota), abi.ptr(gu, abi.P_F64),
                                C.byref(params), abi.ptr(ranked, abi.P_I32), C.byref(n),
                                abi.ptr(dru, abi.P_F64), abi.ptr(order, abi.P_I32), C.byref(on))
        if rc != 0:
            self._err(rc)
        return {"ranked": ranked[:n.value].copy(), "dru": dru[:running.n + pending.n],
                "order": order[:on.value].copy()}

    # -- M0-M6 -------------------------------------------------------------
    def match(self, ranked_idx, jobs, offers, users, params, groups=None, pool_quota=None,
              max_ports=0):
        ranked_idx = np.ascontiguousarray(ranked_idx, np.int32)
        pool_quota = pool_quota or abi.make_pool_quota(None)
        cons, assign, ports, fail, stats = _CallShapes.match_buffers(params, max_ports)
        rc = self.lib.cook_match(self.pool, abi.ptr(ranked_idx, abi.P_I32), len(ranked_idx),
                                 C.byref(jobs), C.byref(offers),
                                 C.byref(groups) if groups is not None else None,
                                 C.byref(users), C.byref(pool_quota), C.byref(params),
                                 abi.ptr(cons, abi.P_I32), abi.ptr(assign, abi.P_I32),
                                 abi.ptr(ports, abi.P_I32) if max_ports > 0 else None,
                                 int(max_ports), abi.ptr(fail, abi.P_U8), C.byref(stats))
        if rc != 0:
            self._err(rc)
        k = stats.n_considerable
        return {"considerable": cons[:k].copy(), "assign": assign[:k].copy(),
                "ports": ports[:k * max(max_ports, 1)].reshape(k, max(max_ports, 1)).copy(),
                "fail": fail[:k].copy(), "stats": stats.as_dict()}

    def match_failures(self, k_idx):
        """cook_match_failures: per requested considerable job of the LAST match on this handle, the
        per-reason host counts at the job's turn (see cook_b200.cycle.summarize_failures)."""
        k = np.ascontiguousarray(k_idx, np.int32)
        out = (abi.FailureCounts * max(len(k), 1))()
        rc = self.lib.cook_match_failures(self.pool, abi.ptr(k, abi.P_I32), len(k), out)
        if rc != 0:
            self._err(rc)
        return [{"n_vms": o.n_vms, "n_passed": o.n_passed, "n_ports": o.n_ports, "counts": list(o.counts)} for o in out[:len(k)]]

    # -- resident pool state (§8f-1) ----------------------------------------
    def state_apply(self, delta):
        """cook_state_apply: one batch of changes (abi.make_delta), all or nothing."""
        rc = self.lib.cook_state_apply(self.pool, C.byref(delta))
        if rc != 0:
            self._err(rc)
        # the live pending ids, O(delta): they size state_rank's output
        live = getattr(self, "_state_pending_ids", set())
        if delta.reset:
            live = set()
        rm = delta.col("pending_rm_job_id")
        live.difference_update(rm.tolist() if rm is not None else [])
        up = delta.col("pending_job_id")
        live.update(up.tolist() if up is not None else [])
        self._state_pending_ids = live
        # the live running ids likewise: they size state_rebalance's victims
        run = getattr(self, "_state_running_ids", set())
        if delta.reset:
            run = set()
        rm = delta.col("running_rm_task_id")
        run.difference_update(rm.tolist() if rm is not None else [])
        tid = delta.col("running").col("task_id") if delta.running.n else None
        run.update(tid.tolist() if tid is not None else [])
        self._state_running_ids = run

    def state_launch(self, job_id, task_id, start_time, hostname_id=None):
        """cook_state_launch: live pending job job_id[i] becomes running task task_id[i] (started at
        start_time[i] on hostname code hostname_id[i]; None: host unknown), its columns copied on the device."""
        jid = np.ascontiguousarray(job_id, np.int64)
        tid = np.ascontiguousarray(task_id, np.int64)
        st = np.ascontiguousarray(start_time, np.int64)
        hn = np.ascontiguousarray(hostname_id, np.int32) if hostname_id is not None else None
        if not (len(tid) == len(st) == len(jid) and (hn is None or len(hn) == len(jid))):
            raise ValueError("state_launch: job_id, task_id, start_time and hostname_id differ in length")
        rc = self.lib.cook_state_launch(self.pool, len(jid), abi.ptr(jid, abi.P_I64), abi.ptr(tid, abi.P_I64),
                                        abi.ptr(st, abi.P_I64), abi.ptr(hn, abi.P_I32) if hn is not None else None)
        if rc != 0:
            self._err(rc)
        live = getattr(self, "_state_pending_ids", set())
        live.difference_update(jid.tolist())
        self._state_pending_ids = live
        run = getattr(self, "_state_running_ids", set())
        run.update(tid.tolist())
        self._state_running_ids = run

    def state_patch(self, job_id, allowed=None, plugin_accept=None, reserved_host=None, clear_reservations=False):
        """cook_state_patch: the given match-time columns of live pending jobs, in place (None: unchanged).
        The jobs keep their place in the queue.  clear_reservations: every reservation is dropped first."""
        jid = np.ascontiguousarray(job_id, np.int64)
        cols = [np.ascontiguousarray(c, dt) if c is not None else None
                for c, dt in ((allowed, np.uint8), (plugin_accept, np.uint8), (reserved_host, np.int32))]
        if any(c is not None and len(c) != len(jid) for c in cols):
            raise ValueError("state_patch: a column's length differs from job_id's")
        al, pa, rh = cols
        rc = self.lib.cook_state_patch(self.pool, len(jid), abi.ptr(jid, abi.P_I64),
                                       abi.ptr(al, abi.P_U8) if al is not None else None,
                                       abi.ptr(pa, abi.P_U8) if pa is not None else None,
                                       abi.ptr(rh, abi.P_I32) if rh is not None else None, int(bool(clear_reservations)))
        if rc != 0:
            self._err(rc)

    def state_usage(self, n_users, hostname_id=None):
        """cook_state_usage: the running usage of the live running rows, each sum a left fold in ascending task
        id.  Returns 'user' as {count, cpus, mem, gpus} arrays of n_users (abi.make_users' `usage`), 'pool' as
        [count, cpus, mem, gpus] (one term of state_rank's group_usage) and, for the hosts of hostname_id,
        'run_cpus', 'run_mem' and 'run_count' arrays (an offer table's run_* columns)."""
        hn = np.ascontiguousarray(hostname_id if hostname_id is not None else np.zeros(0), np.int32)
        H = len(hn)
        user = np.zeros(4 * max(int(n_users), 1), np.float64)
        pool = np.zeros(4, np.float64)
        rc_, rm, rn = np.zeros(max(H, 1), np.float64), np.zeros(max(H, 1), np.float64), np.zeros(max(H, 1), np.int32)
        rc = self.lib.cook_state_usage(self.pool, int(n_users), abi.ptr(user, abi.P_F64), abi.ptr(pool, abi.P_F64), H,
                                       abi.ptr(hn, abi.P_I32) if H else None, abi.ptr(rc_, abi.P_F64),
                                       abi.ptr(rm, abi.P_F64), abi.ptr(rn, abi.P_I32))
        if rc != 0:
            self._err(rc)
        U = int(n_users)
        return {"user": {k: user[i * U:(i + 1) * U].copy() for i, k in enumerate(("count", "cpus", "mem", "gpus"))},
                "pool": pool, "run_cpus": rc_[:H].copy(), "run_mem": rm[:H].copy(), "run_count": rn[:H].copy()}

    def state_cotasks(self, n_groups, attr_col=None, hosts=None):
        """cook_state_cotasks: each group's running cotasks from the live running rows with a known host, by (group,
        task id).  Returns (cot_off, cot_hostname_id, cot_attr_val), the cot_* fields of abi.Groups; the attribute
        value is hosts' (an abi.OffersSoA or abi.HostTable) in the group's attr_col, 0 where there is none."""
        ac = np.ascontiguousarray(attr_col, np.int32) if attr_col is not None else None
        if ac is not None and len(ac) != n_groups:
            raise ValueError("state_cotasks: attr_col needs one column per group")
        hp = None
        if hosts is not None:   # the fields cook_state_cotasks reads, from an offer table or a host table
            hp = abi.HostTable(n=hosts.n, hostname_id=hosts.col("hostname_id"), n_attr_cols=hosts.n_attr_cols,
                               attr=hosts.col("attr"))
        args = (self.pool, int(n_groups), abi.ptr(ac, abi.P_I32) if ac is not None else None,
                C.byref(hp) if hp is not None else None)
        n = C.c_int32(0)
        rc = self.lib.cook_state_cotasks(*args, 0, None, None, None, C.byref(n))
        if rc != 0:
            self._err(rc)
        cap = n.value
        off = np.zeros(int(n_groups) + 1, np.int32)
        host, val = np.zeros(max(cap, 1), np.int32), np.zeros(max(cap, 1), np.int32)
        rc = self.lib.cook_state_cotasks(*args, cap, abi.ptr(off, abi.P_I32), abi.ptr(host, abi.P_I32),
                                         abi.ptr(val, abi.P_I32), C.byref(n))
        if rc != 0:
            self._err(rc)
        return off, host[:n.value], val[:n.value]

    def state_rank(self, users, pool_quota=None, group_quota=None, group_usage=None, params=None, offensive=False):
        """cook_state_rank: the live rows ranked; the queue stays on the device.  Returns its job ids.
        offensive: cook_state_rank_offensive, returns (queue job ids, the job ids the rank dropped as offensive)."""
        pool_quota = pool_quota or abi.make_pool_quota(None)
        group_quota = group_quota or abi.make_pool_quota(None)
        params = params or abi.RankParams(100, 0, 0.0, 0.0)
        gu = np.ascontiguousarray(group_usage if group_usage is not None else np.zeros(4), np.float64)
        n_live = len(getattr(self, "_state_pending_ids", ()))
        out = np.zeros(max(n_live, 1), np.int64)
        n = C.c_int32(0)
        args = (self.pool, C.byref(users), C.byref(pool_quota), C.byref(group_quota), abi.ptr(gu, abi.P_F64),
                C.byref(params), abi.ptr(out, abi.P_I64), C.byref(n))
        if not offensive:
            rc = self.lib.cook_state_rank(*args)
            if rc != 0:
                self._err(rc)
            return out[:n.value].copy()
        off = np.zeros(max(n_live, 1), np.int64)
        n_off = C.c_int32(0)
        rc = self.lib.cook_state_rank_offensive(*args, abi.ptr(off, abi.P_I64), n_live, C.byref(n_off))
        if rc != 0:
            self._err(rc)
        return out[:n.value].copy(), off[:n_off.value].copy()

    def state_considerable(self, users, params, pool_quota=None):
        """cook_state_considerable: M0 over the resident queue without a match (params: abi.ConsiderableParams).
        Returns the job ids in take order; with params.consume they leave the queue until the next state_rank."""
        pool_quota = pool_quota or abi.make_pool_quota(None)
        out = np.zeros(max(int(params.num_considerable), 1), np.int64)
        n = C.c_int32(0)
        rc = self.lib.cook_state_considerable(self.pool, C.byref(users), C.byref(pool_quota), C.byref(params),
                                              abi.ptr(out, abi.P_I64), C.byref(n))
        if rc != 0:
            self._err(rc)
        return out[:n.value].copy()

    def state_match(self, offers, users, params, groups=None, pool_quota=None, max_ports=0, derived=False):
        """cook_state_match: the resident queue (minus what left it since the rank) matched against
        `offers`.  'considerable' holds job ids.  derived: cook_state_match_derived, the users' usage_*, the
        offers' run_* and the groups' cot_* read from the resident running rows on the device (those fields of
        `users`, `offers` and `groups` are ignored)."""
        pool_quota = pool_quota or abi.make_pool_quota(None)
        k = max(params.num_considerable, 1)
        cons = np.full(k, -1, np.int64)
        _, assign, ports, fail, stats = _CallShapes.match_buffers(params, max_ports)
        fn = self.lib.cook_state_match_derived if derived else self.lib.cook_state_match
        rc = fn(self.pool, C.byref(offers),
                                       C.byref(groups) if groups is not None else None,
                                       C.byref(users), C.byref(pool_quota), C.byref(params),
                                       abi.ptr(cons, abi.P_I64), abi.ptr(assign, abi.P_I32),
                                       abi.ptr(ports, abi.P_I32) if max_ports > 0 else None,
                                       int(max_ports), abi.ptr(fail, abi.P_U8), C.byref(stats))
        if rc != 0:
            self._err(rc)
        n = stats.n_considerable
        return {"considerable": cons[:n].copy(), "assign": assign[:n].copy(),
                "ports": ports[:n * max(max_ports, 1)].reshape(n, max(max_ports, 1)).copy(),
                "fail": fail[:n].copy(), "stats": stats.as_dict()}

    def state_rebalance(self, hosts, users, params, groups=None, derived=False):
        """cook_state_rebalance: the rebalancer over the live running tasks and the first allowed jobs of the
        resident queue.  As rebalance(), plus each decision's 'job_id'; 'victims' are task ids (the task
        of the job an earlier decision e placed: -1 - e).  derived: cook_state_rebalance_derived, the groups'
        cot_* read from the resident running rows over `hosts` on the device (those fields are ignored)."""
        mp = max(params.max_preemption, 1)
        dec = (abi.Decision * mp)()
        jid = np.full(mp, -1, np.int64)
        cap = len(getattr(self, "_state_running_ids", ())) + mp
        vict = np.full(cap, -1, np.int64)
        n = C.c_int32(0)
        fn = self.lib.cook_state_rebalance_derived if derived else self.lib.cook_state_rebalance
        rc = fn(self.pool, C.byref(hosts), C.byref(groups) if groups is not None else None, C.byref(users),
                C.byref(params), dec, abi.ptr(jid, abi.P_I64), abi.ptr(vict, abi.P_I64), int(cap), C.byref(n))
        if rc != 0:
            self._err(rc)
        out = decisions_to_list(dec, vict, n.value)
        for d, j in zip(out, jid[:n.value].tolist()):
            d["job_id"] = j
        return out

    # -- B1-B6 -------------------------------------------------------------
    def rebalance(self, running, pending, pending_job_id, pending_priority, hosts, users, params,
                  groups=None):
        pj = np.ascontiguousarray(pending_job_id, np.int64)
        pp = np.ascontiguousarray(pending_priority, np.int32)
        dec = (abi.Decision * max(params.max_preemption, 1))()
        vict = np.full(running.t.n + max(params.max_preemption, 1), -1, np.int32)
        n = C.c_int32(0)
        rc = self.lib.cook_rebalance(self.pool, C.byref(running), C.byref(pending),
                                     abi.ptr(pj, abi.P_I64), abi.ptr(pp, abi.P_I32),
                                     C.byref(hosts), C.byref(groups) if groups is not None else None,
                                     C.byref(users), C.byref(params), dec,
                                     abi.ptr(vict, abi.P_I32), C.byref(n))
        if rc != 0:
            self._err(rc)
        return decisions_to_list(dec, vict, n.value)


    def rebalance_trace(self, running, pending, pending_job_id, pending_priority, hosts, users, params,
                        forced=None, forced_only=True, groups=None):
        """cook_rebalance_trace: the same walk plus the rebalancer state the reference's own tests read
        (K18 pending DRU, K21 next-state, job-below-quota).  forced: [(pending_idx, host, [victims],
        mem, cpus, gpus)] applied with next-state instead of being searched."""
        return rebalance_trace_call(
            lambda *a: self.lib.cook_rebalance_trace(self.pool, *a), self._err,
            running, pending, pending_job_id, pending_priority, hosts, users, params, forced, forced_only, groups)

    # -- phase timing / §8e exchange ----------------------------------------
    def last_stats(self, phase):
        ps = abi.PhaseStats()
        rc = self.lib.cook_last_stats(self.pool, int(phase), C.byref(ps))
        if rc != 0:
            self._err(rc)
        return ps.as_dict()

    def exchange_usage(self, n_users_pad, comm=None, world=1):
        """Per-user usage delta of the last match round on this handle, computed on the device and
        all-gathered over `comm` (a cook_comm_init handle).  Returns [world, n_users_pad, 4]."""
        n_pad = 4 * int(n_users_pad)
        out = np.zeros(world * n_pad, np.float64)
        rc = self.lib.cook_exchange_usage(self.pool, comm, int(world), n_pad, abi.ptr(out, abi.P_F64))
        if rc != 0:
            self._err(rc)
        return out.reshape(world, n_users_pad, 4)


def exchange_usage_batch(engines, n_users_pad, n_slots=None, comm=None, world=1):
    """The exchange step for ALL the pools a rank ran in the cycle: their usage deltas (slot i =
    engines[i], the slots beyond stay zero) travel in ONE all-gather (cook_exchange_usage_batch).
    Returns [world, n_slots, n_users_pad, 4]."""
    if not engines:
        raise ValueError("exchange_usage_batch: at least one handle")
    n_slots = len(engines) if n_slots is None else int(n_slots)
    n_pad = 4 * int(n_users_pad)
    out = np.zeros(world * n_slots * n_pad, np.float64)
    handles = (C.c_void_p * len(engines))(*[e.pool for e in engines])
    rc = engines[0].lib.cook_exchange_usage_batch(handles, len(engines), comm, int(world), n_pad, n_slots,
                                                  abi.ptr(out, abi.P_F64))
    if rc != 0:
        engines[0]._err(rc)
    return out.reshape(world, n_slots, n_users_pad, 4)


def comm_unique_id(lib):
    buf = (C.c_uint8 * 128)()
    rc = lib.cook_comm_unique_id(buf)
    if rc != 0:
        raise CookError(rc, "cook_comm_unique_id (is libnccl loadable?)")
    return bytes(buf)


def comm_init(lib, uid, rank, world, device):
    comm = C.c_void_p()
    buf = (C.c_uint8 * 128).from_buffer_copy(uid)
    rc = lib.cook_comm_init(buf, int(rank), int(world), int(device), C.byref(comm))
    if rc != 0:
        raise CookError(rc, "cook_comm_init")
    return comm


def rebalance_trace_call(fn, on_error, running, pending, pending_job_id, pending_priority, hosts, users, params,
                         forced, forced_only, groups):
    """Argument packing of cook_rebalance_trace (`fn` binds the handle; the test suite's CPU checker
    exports the same signature and reuses this packing)."""
    pj = np.ascontiguousarray(pending_job_id, np.int64)
    pp = np.ascontiguousarray(pending_priority, np.int32)
    mp = max(params.max_preemption, 1)
    R, P, H = running.t.n, pending.n, hosts.n
    dec = (abi.Decision * mp)()
    vict = np.full(R + mp, -1, np.int32)
    n = C.c_int32(0)
    forced = forced or []
    fdec = (abi.Decision * max(len(forced), 1))()
    fv = []
    for i, (pi, h, vs, m, c, g) in enumerate(forced):
        fdec[i] = abi.Decision(pi, h, len(fv), len(vs), 0.0, m, c, g)
        fv += list(vs)
    fv = np.array(fv + [0], np.int32)
    pdru, tdru = np.full(max(P, 1), np.nan), np.zeros(R + mp)
    alive, order, n_order = np.zeros(R + mp, np.uint8), np.zeros(R + mp, np.int32), C.c_int32(0)
    hs, sm, sc, sg = np.zeros(H, np.uint8), np.zeros(H), np.zeros(H), np.zeros(H)
    below = np.full(max(P, 1), 255, np.uint8)
    tr = abi.RebTrace(len(forced), fdec, abi.ptr(fv, abi.P_I32), abi.ptr(pdru, abi.P_F64),
                      abi.ptr(tdru, abi.P_F64), abi.ptr(alive, abi.P_U8), abi.ptr(order, abi.P_I32),
                      C.pointer(n_order), abi.ptr(hs, abi.P_U8), abi.ptr(sm, abi.P_F64),
                      abi.ptr(sc, abi.P_F64), abi.ptr(sg, abi.P_F64), 1 if forced_only else 0,
                      abi.ptr(below, abi.P_U8))
    rc = fn(C.byref(running), C.byref(pending), abi.ptr(pj, abi.P_I64), abi.ptr(pp, abi.P_I32),
            C.byref(hosts), C.byref(groups) if groups is not None else None, C.byref(users),
            C.byref(params), dec, abi.ptr(vict, abi.P_I32), C.byref(n), C.byref(tr))
    if rc != 0:
        on_error(rc)
    k = n_order.value
    return {"decisions": decisions_to_list(dec, vict, n.value), "pending_dru": pdru[:P],
            "below_quota": [bool(b) if b != 255 else None for b in below[:P]],
            "order": [int(x) for x in order[:k]], "order_dru": [float(tdru[t]) for t in order[:k]],
            "spare": {h: (float(sm[h]), float(sc[h]), float(sg[h])) for h in range(H) if hs[h]}}


def decisions_to_list(dec, vict, n):
    out = []
    for i in range(n):
        d = dec[i]
        out.append({"pending_idx": d.pending_idx, "host": d.host,
                    "victims": [int(x) for x in vict[d.victim_begin:d.victim_begin + d.victim_count]],
                    "dru": d.dru, "mem": d.mem, "cpus": d.cpus, "gpus": d.gpus})
    return out
