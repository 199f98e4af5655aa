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
    for name, argtypes in abi.ARGTYPES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = C.c_int32, argtypes
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
        # a pending upsert or removal drops a job's retry facts and parked copy, a reset all of them
        if hasattr(self, "_state_retry"):
            if delta.reset:
                for m in (self._state_retry, self._state_parked_glen, self._state_task_job):
                    m.clear()
            for c in ("pending_rm_job_id", "pending_job_id"):
                ids = delta.col(c)
                for j in (ids.tolist() if ids is not None else []):
                    self._state_retry.discard(j)
                    self._state_parked_glen.pop(j, None)
        # the live pending ids, O(delta): they size state_rank's output
        live = getattr(self, "_state_pending_ids", set())
        if delta.reset:
            live = set()
            self._state_offer_ids = set()
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
        # and the length of each live row's group list: they size state_sweep's straggler entries
        png, rng_ = self._group_lengths()
        if delta.reset:
            png.clear()
            rng_.clear()
        for j in (rm.tolist() if (rm := delta.col("pending_rm_job_id")) is not None else []):
            png.pop(j, None)
        for t in (rm.tolist() if (rm := delta.col("running_rm_task_id")) is not None else []):
            rng_.pop(t, None)
        if up is not None:
            off = delta.col("pending").col("group_off")
            png.update(zip(up.tolist(), np.diff(off).tolist() if off is not None else [0] * len(up)))
        if tid is not None:
            off = delta.col("running_group_off")
            rng_.update(zip(tid.tolist(), np.diff(off).tolist() if off is not None else [0] * len(tid)))

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
        png, rng_ = self._group_lengths()
        retry = getattr(self, "_state_retry", ())
        for j, t in zip(jid.tolist(), tid.tolist()):
            rng_[t] = png.pop(j, 0)
            if j in retry:   # the job parks: state_status may requeue it
                self._state_parked_glen[j] = rng_[t]
                self._state_task_job[t] = j

    def _group_lengths(self):
        """{job id: group list length} of the live pending rows and {task id: length} of the live running rows."""
        if not hasattr(self, "_state_group_len"):
            self._state_group_len = ({}, {})
        return self._state_group_len

    def state_task_facts(self, task_id, max_runtime_ms=None, cancelled=None, unknown=None):
        """cook_state_task_facts: the killers' facts of live running tasks (None: unchanged): the job's max-runtime in
        ms (-1: none), the cancelled flag, and whether the status is unknown rather than running."""
        tid = np.ascontiguousarray(task_id, np.int64)
        cols = [np.ascontiguousarray(c, dt) if c is not None else None
                for c, dt in ((max_runtime_ms, np.int64), (cancelled, np.uint8), (unknown, np.uint8))]
        if any(c is not None and len(c) != len(tid) for c in cols):
            raise ValueError("state_task_facts: a column's length differs from task_id's")
        mr, ca, un = cols
        rc = self.lib.cook_state_task_facts(self.pool, len(tid), abi.ptr(tid, abi.P_I64),
                                            abi.ptr(mr, abi.P_I64) if mr is not None else None,
                                            abi.ptr(ca, abi.P_U8) if ca is not None else None,
                                            abi.ptr(un, abi.P_U8) if un is not None else None)
        if rc != 0:
            self._err(rc)

    def state_task_reason(self, task_id, reason_code):
        """cook_state_task_reason: the reason code of live running tasks (the caller's :reason/code dictionary, -1:
        none), read by state_instance_stats."""
        tid = np.ascontiguousarray(task_id, np.int64)
        rc_ = np.ascontiguousarray(reason_code, np.int32)
        if len(rc_) != len(tid):
            raise ValueError("state_task_reason: reason_code differs in length from task_id")
        rc = self.lib.cook_state_task_reason(self.pool, len(tid), abi.ptr(tid, abi.P_I64), abi.ptr(rc_, abi.P_I32))
        if rc != 0:
            self._err(rc)

    def state_job_facts(self, job_id, flags=None, gpu_model=None, disk_request=None, disk_limit=None, disk_type=None):
        """cook_state_job_facts: the stats keys of live pending jobs (None: unchanged): abi.JF_* bits, the gpu model
        and disk type codes (-1: unspecified) and the disk request and limit, each read under its bit."""
        jid = np.ascontiguousarray(job_id, np.int64)
        cols = [np.ascontiguousarray(c, dt) if c is not None else None
                for c, dt in ((flags, np.uint8), (gpu_model, np.int32), (disk_request, np.float64),
                              (disk_limit, np.float64), (disk_type, np.int32))]
        if any(c is not None and len(c) != len(jid) for c in cols):
            raise ValueError("state_job_facts: a column's length differs from job_id's")
        pt = (abi.P_U8, abi.P_I32, abi.P_F64, abi.P_F64, abi.P_I32)
        rc = self.lib.cook_state_job_facts(self.pool, len(jid), abi.ptr(jid, abi.P_I64),
                                           *[abi.ptr(c, t) if c is not None else None for c, t in zip(cols, pt)])
        if rc != 0:
            self._err(rc)

    def state_list_facts(self, job_id, submit_ms=None, submit_pool=None, custom_executor=None):
        """cook_state_list_facts: the submit time (ms), submit pool code (-1: none) and custom executor (-1 nil, 0
        false, 1 true) of jobs with a live pending or running row (None: unchanged), written on every such row."""
        jid = np.ascontiguousarray(job_id, np.int64)
        cols = [np.ascontiguousarray(c, dt) if c is not None else None
                for c, dt in ((submit_ms, np.int64), (submit_pool, np.int32), (custom_executor, np.int32))]
        if any(c is not None and len(c) != len(jid) for c in cols):
            raise ValueError("state_list_facts: a column's length differs from job_id's")
        pt = (abi.P_I64, abi.P_I32, abi.P_I32)
        rc = self.lib.cook_state_list_facts(self.pool, len(jid), abi.ptr(jid, abi.P_I64),
                                            *[abi.ptr(c, t) if c is not None else None for c, t in zip(cols, pt)])
        if rc != 0:
            self._err(rc)

    def state_match_metrics(self, n_users, dropped=(), unmatched_warn_cycles=500, key_cap=64):
        """cook_state_match_metrics over the last resident match round: `dropped` are the considerable positions the
        launch-rate filter dropped.  Returns the counts by their abi.MMC_* names in lower case ('considerable',
        'matched', 'head_job_id', ...), 'total_cpus', 'total_mem', 'pct_cpus' and 'pct_mem' [50, 95, 100], 'rows'
        (head, largest by cpus, largest by mem: dicts of abi.MMR_INT and abi.MMR_AMOUNT), 'first' [(job id, cycles)]
        in take order, 'user_considerable' and 'user_matched' [n_users], 'keys' [(kind, code, total)] in ascending
        (kind, code), and 'stats' (abi.PhaseStats.as_dict()).  The call is made with key_cap keys first and, when
        more are needed, once more with the count it reports."""
        drop = np.ascontiguousarray(dropped, np.int32)
        U = int(n_users)
        ucons, umat = np.zeros(max(U, 1), np.int32), np.zeros(max(U, 1), np.int32)
        counts, amounts = np.zeros(abi.MMC_N, np.int64), np.zeros(abi.MMA_N)
        row_i, row_a = np.zeros((abi.MM_ROWS, len(abi.MMR_INT)), np.int64), np.zeros((abi.MM_ROWS, len(abi.MMR_AMOUNT)))
        fj, fc = np.zeros(abi.MM_FIRST_N, np.int64), np.zeros(abi.MM_FIRST_N, np.int32)
        st = abi.PhaseStats()
        cap = max(int(key_cap), 0)
        for _ in range(2):
            kind, code, total = np.zeros(max(cap, 1), np.int32), np.zeros(max(cap, 1), np.int32), np.zeros(max(cap, 1))
            rc = self.lib.cook_state_match_metrics(
                self.pool, U, len(drop), abi.ptr(drop, abi.P_I32) if len(drop) else None, int(unmatched_warn_cycles),
                cap, abi.ptr(counts, abi.P_I64), abi.ptr(amounts, abi.P_F64), abi.ptr(row_i, abi.P_I64),
                abi.ptr(row_a, abi.P_F64), abi.ptr(fj, abi.P_I64), abi.ptr(fc, abi.P_I32), abi.ptr(ucons, abi.P_I32),
                abi.ptr(umat, abi.P_I32), abi.ptr(kind, abi.P_I32), abi.ptr(code, abi.P_I32), abi.ptr(total, abi.P_F64),
                C.byref(st))
            if rc != abi.COOK_E_TOO_LARGE or counts[abi.MMC_KEYS] <= cap:
                break
            cap = int(counts[abi.MMC_KEYS])
        if rc != 0:
            self._err(rc)
        names = ("considerable", "matched", "head_job_id", "head_matched", "uris", "uris_position", "keys_n",
                 "too_long", "first_n")
        res = {n: int(counts[i]) for i, n in enumerate(names)}
        res["total_cpus"], res["total_mem"] = float(amounts[abi.MMA_TOTAL_CPUS]), float(amounts[abi.MMA_TOTAL_MEM])
        res["pct_cpus"] = amounts[abi.MMA_PCT_CPUS:abi.MMA_PCT_CPUS + 3].tolist()
        res["pct_mem"] = amounts[abi.MMA_PCT_MEM:abi.MMA_PCT_MEM + 3].tolist()
        res["rows"] = [dict(zip(abi.MMR_INT, map(int, row_i[r])), **dict(zip(abi.MMR_AMOUNT, map(float, row_a[r]))))
                       for r in range(abi.MM_ROWS)] if res["considerable"] else []
        res["first"] = list(zip(fj[:res["first_n"]].tolist(), fc[:res["first_n"]].tolist()))
        res["keys"] = [(int(kind[i]), int(code[i]), float(total[i])) for i in range(res["keys_n"])]
        res["user_considerable"], res["user_matched"] = ucons[:U].copy(), umat[:U].copy()
        res["stats"] = st.as_dict()
        return res

    def state_finish(self, task_id, end_time_ms=None, success=None):
        """cook_state_finish: the tasks leave as a removal delta would take them; each successful one leaves a runtime
        record per group of its list (success None: none succeeded)."""
        tid = np.ascontiguousarray(task_id, np.int64)
        end = np.ascontiguousarray(end_time_ms, np.int64) if end_time_ms is not None else None
        ok = np.ascontiguousarray(success, np.uint8) if success is not None else None
        if any(c is not None and len(c) != len(tid) for c in (end, ok)):
            raise ValueError("state_finish: end_time_ms or success differs in length from task_id")
        rc = self.lib.cook_state_finish(self.pool, len(tid), abi.ptr(tid, abi.P_I64),
                                        abi.ptr(end, abi.P_I64) if end is not None else None,
                                        abi.ptr(ok, abi.P_U8) if ok is not None else None)
        if rc != 0:
            self._err(rc)
        getattr(self, "_state_running_ids", set()).difference_update(tid.tolist())
        rng_ = self._group_lengths()[1]
        for t in tid.tolist():
            rng_.pop(t, None)
        self._forget_tasks(tid.tolist())

    def state_finish_history(self, task_id, end_time_ms, success, reason_code=None):
        """cook_state_finish_history: state_finish, and while the history is on, the rows that start at or after its
        horizon are appended to it (reason_code None: each row's reason fact)."""
        tid = np.ascontiguousarray(task_id, np.int64)
        end = np.ascontiguousarray(end_time_ms, np.int64)
        ok = np.ascontiguousarray(success, np.uint8)
        rs = np.ascontiguousarray(reason_code, np.int32) if reason_code is not None else None
        if any(c is not None and len(c) != len(tid) for c in (end, ok, rs)):
            raise ValueError("state_finish_history: a column differs in length from task_id")
        rc = self.lib.cook_state_finish_history(self.pool, len(tid), abi.ptr(tid, abi.P_I64), abi.ptr(end, abi.P_I64),
                                                abi.ptr(ok, abi.P_U8),
                                                abi.ptr(rs, abi.P_I32) if rs is not None else None)
        if rc != 0:
            self._err(rc)
        getattr(self, "_state_running_ids", set()).difference_update(tid.tolist())
        rng_ = self._group_lengths()[1]
        for t in tid.tolist():
            rng_.pop(t, None)
        self._forget_tasks(tid.tolist())

    def state_retry_config(self, mea_culpa_limit=5, reasons=()):
        """cook_state_retry_config: the global mea-culpa limit (-1: unlimited) and the reason dictionary, an iterable of
        (reason code, mea culpa, failure limit; -2: the global one, -1: unlimited)."""
        r = list(reasons)
        code = np.ascontiguousarray([x[0] for x in r], np.int32)
        mc = np.ascontiguousarray([bool(x[1]) for x in r], np.uint8)
        lim = np.ascontiguousarray([x[2] for x in r], np.int32)
        rc = self.lib.cook_state_retry_config(self.pool, int(mea_culpa_limit), len(r), abi.ptr(code, abi.P_I32),
                                              abi.ptr(mc, abi.P_U8), abi.ptr(lim, abi.P_I32))
        if rc != 0:
            self._err(rc)

    def state_retry_facts(self, job_id, max_retries, flags, done_reasons=None):
        """cook_state_retry_facts: the retry facts of jobs the handle holds: max-retries, abi.RF_* bits and, per job,
        the reason codes of its earlier done instances (-1: none; None: no done instance for any job)."""
        jid = np.ascontiguousarray(job_id, np.int64)
        mr = np.ascontiguousarray(max_retries, np.int32)
        fl = np.ascontiguousarray(flags, np.uint8)
        if not len(jid) == len(mr) == len(fl) or (done_reasons is not None and len(done_reasons) != len(jid)):
            raise ValueError("state_retry_facts: the columns differ in length")
        off = val = None
        if done_reasons is not None:
            off = np.zeros(len(jid) + 1, np.int32)
            off[1:] = np.cumsum([len(d) for d in done_reasons])
            val = np.ascontiguousarray([c for d in done_reasons for c in d] or [0], np.int32)
        rc = self.lib.cook_state_retry_facts(self.pool, len(jid), abi.ptr(jid, abi.P_I64), abi.ptr(mr, abi.P_I32),
                                             abi.ptr(fl, abi.P_U8), abi.ptr(off, abi.P_I32) if off is not None else None,
                                             abi.ptr(val, abi.P_I32) if val is not None else None)
        if rc != 0:
            self._err(rc)
        self._retry_jobs().update(jid.tolist())

    def _retry_jobs(self):
        """The job ids given retry facts (a superset of those the handle holds facts for), the parked jobs' group list
        lengths and the job of each task launched from one: what state_status needs to track a requeue."""
        if not hasattr(self, "_state_retry"):
            self._state_retry = set()
            self._state_parked_glen = {}
            self._state_task_job = {}
        return self._state_retry

    def _forget_tasks(self, tids):
        """Tasks that ended without state_status: the job loses its parked copy, and its facts unless it is a live
        pending row again (the library's rule, restated for the bookkeeping).  A job has at most one task launched
        from a parked row: a requeue needs every instance gone."""
        if not hasattr(self, "_state_retry"):
            return
        for t in tids:
            j = self._state_task_job.pop(t, None)
            if j is not None:
                self._state_parked_glen.pop(j, None)
                if j not in getattr(self, "_state_pending_ids", ()):
                    self._state_retry.discard(j)

    def state_status(self, task_id, success, end_time_ms, reason_code=None, preempted=None):
        """cook_state_status: state_finish_history plus each row's job decided in batch order; returns (outcome
        abi.JOB_* per row, attempts consumed per row).  A requeued job is a live pending row again."""
        tid = np.ascontiguousarray(task_id, np.int64)
        ok = np.ascontiguousarray(success, np.uint8)
        end = np.ascontiguousarray(end_time_ms, np.int64)
        rs = np.ascontiguousarray(reason_code, np.int32) if reason_code is not None else None
        pre = np.ascontiguousarray(preempted, np.uint8) if preempted is not None else None
        if any(c is not None and len(c) != len(tid) for c in (end, ok, rs, pre)):
            raise ValueError("state_status: a column differs in length from task_id")
        out = np.zeros(max(len(tid), 1), np.int32)
        att = np.zeros(max(len(tid), 1), np.int32)
        rc = self.lib.cook_state_status(self.pool, len(tid), abi.ptr(tid, abi.P_I64), abi.ptr(ok, abi.P_U8),
                                        abi.ptr(end, abi.P_I64), abi.ptr(rs, abi.P_I32) if rs is not None else None,
                                        abi.ptr(pre, abi.P_U8) if pre is not None else None, abi.ptr(out, abi.P_I32),
                                        abi.ptr(att, abi.P_I32))
        if rc != 0:
            self._err(rc)
        getattr(self, "_state_running_ids", set()).difference_update(tid.tolist())
        png, rng_ = self._group_lengths()
        self._retry_jobs()
        live = self._state_pending_ids = getattr(self, "_state_pending_ids", set())
        for t, o in zip(tid.tolist(), out[:len(tid)].tolist()):
            rng_.pop(t, None)
            j = self._state_task_job.pop(t, None)
            if j is None:
                continue
            if o == abi.JOB_WAITING:
                live.add(j)
                png[j] = self._state_parked_glen.pop(j, 0)
            elif o == abi.JOB_COMPLETED:
                self._state_parked_glen.pop(j, None)
                self._state_retry.discard(j)
        return out[:len(tid)].copy(), att[:len(tid)].copy()

    def state_history_seed(self, since_ms, task_id=(), user=(), start_ms=(), end_ms=(), cpus=(), mem=(), success=(),
                           reason_code=()):
        """cook_state_history_seed: the history replaced by these finished rows at horizon since_ms, and on."""
        tid = np.ascontiguousarray(task_id, np.int64)
        cols = (np.ascontiguousarray(user, np.int32), np.ascontiguousarray(start_ms, np.int64),
                np.ascontiguousarray(end_ms, np.int64), np.ascontiguousarray(cpus, np.float64),
                np.ascontiguousarray(mem, np.float64), np.ascontiguousarray(success, np.uint8),
                np.ascontiguousarray(reason_code, np.int32))
        if any(len(c) != len(tid) for c in cols):
            raise ValueError("state_history_seed: a column differs in length from task_id")
        u, st_, en, cp, me, ok, rs = cols
        rc = self.lib.cook_state_history_seed(self.pool, int(since_ms), len(tid), abi.ptr(tid, abi.P_I64),
                                              abi.ptr(u, abi.P_I32), abi.ptr(st_, abi.P_I64), abi.ptr(en, abi.P_I64),
                                              abi.ptr(cp, abi.P_F64), abi.ptr(me, abi.P_F64), abi.ptr(ok, abi.P_U8),
                                              abi.ptr(rs, abi.P_I32))
        if rc != 0:
            self._err(rc)

    def state_history_advance(self, since_ms):
        """cook_state_history_advance: the horizon raised to since_ms; the rows that start before it leave."""
        rc = self.lib.cook_state_history_advance(self.pool, int(since_ms))
        if rc != 0:
            self._err(rc)

    def _completed_cols(self, who, job_id, stamp, user, submit_ms, submit_pool, custom_executor, kind):
        cols = (np.ascontiguousarray(job_id, np.int64), np.ascontiguousarray(stamp, np.int64),
                np.ascontiguousarray(user, np.int32), np.ascontiguousarray(submit_ms, np.int64),
                np.ascontiguousarray(submit_pool, np.int32), np.ascontiguousarray(custom_executor, np.int32),
                np.ascontiguousarray(kind, np.uint8))
        if any(len(c) != len(cols[0]) for c in cols):
            raise ValueError(f"{who}: a column differs in length from job_id")
        ptrs = [abi.ptr(c, t) for c, t in zip(cols, (abi.P_I64, abi.P_I64, abi.P_I32, abi.P_I64, abi.P_I32, abi.P_I32,
                                                     abi.P_U8))]
        return len(cols[0]), ptrs

    def state_completed_seed(self, since_ms, job_id=(), stamp=(), user=(), submit_ms=(), submit_pool=(),
                             custom_executor=(), kind=()):
        """cook_state_completed_seed: the completed-job log replaced by these records (kind abi.CJ_*, custom executor
        -1 nil, 0 false, 1 true) at horizon since_ms on submit time, and on."""
        n, p = self._completed_cols("state_completed_seed", job_id, stamp, user, submit_ms, submit_pool,
                                    custom_executor, kind)
        rc = self.lib.cook_state_completed_seed(self.pool, int(since_ms), n, *p)
        if rc != 0:
            self._err(rc)

    def state_completed_record(self, job_id=(), stamp=(), user=(), submit_ms=(), submit_pool=(), custom_executor=(),
                               kind=()):
        """cook_state_completed_record: these records appended in order; those submitted before the horizon are
        skipped."""
        n, p = self._completed_cols("state_completed_record", job_id, stamp, user, submit_ms, submit_pool,
                                    custom_executor, kind)
        rc = self.lib.cook_state_completed_record(self.pool, n, *p)
        if rc != 0:
            self._err(rc)

    def state_completed_advance(self, since_ms):
        """cook_state_completed_advance: the horizon raised to since_ms; the records submitted before it leave."""
        rc = self.lib.cook_state_completed_advance(self.pool, int(since_ms))
        if rc != 0:
            self._err(rc)

    def state_group_runtimes(self, group=(), runtime_s=(), forget=()):
        """cook_state_group_runtimes: the records of the groups in `forget` leave, then (group[i], runtime_s[i]) are
        appended."""
        g = np.ascontiguousarray(group, np.int32)
        r = np.ascontiguousarray(runtime_s, np.int32)
        f = np.ascontiguousarray(forget, np.int32)
        if len(g) != len(r):
            raise ValueError("state_group_runtimes: group and runtime_s differ in length")
        rc = self.lib.cook_state_group_runtimes(self.pool, len(g), abi.ptr(g, abi.P_I32) if len(g) else None,
                                                abi.ptr(r, abi.P_I32) if len(r) else None, len(f),
                                                abi.ptr(f, abi.P_I32) if len(f) else None)
        if rc != 0:
            self._err(rc)

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

    def state_digest(self, n_buckets=0):
        """cook_state_digest: the fingerprints of the live pending rows, the live running rows and the live queue as
        (sum, xor, n) tuples, the live 'entries' per list, 'consistent' / 'first_mismatch' (an abi.AUDIT_NAMES name
        or None) of the recount, and with n_buckets 'pending_buckets' / 'running_buckets' (abi.FP_DTYPE arrays)."""
        nb = int(n_buckets)
        out = abi.StateDigest()
        pb, rb = np.zeros(max(nb, 1), abi.FP_DTYPE), np.zeros(max(nb, 1), abi.FP_DTYPE)
        fp = C.POINTER(abi.Fp)
        rc = self.lib.cook_state_digest(self.pool, nb, C.byref(out), pb.ctypes.data_as(fp) if nb else None,
                                        rb.ctypes.data_as(fp) if nb else None)
        if rc != 0:
            self._err(rc)
        return {"pending": out.pending.as_tuple(), "running": out.running.as_tuple(), "queue": out.queue.as_tuple(),
                "entries": list(out.entries), "consistent": bool(out.consistent),
                "first_mismatch": abi.AUDIT_NAMES[out.first_mismatch] if out.first_mismatch >= 0 else None,
                "pending_buckets": pb[:nb], "running_buckets": rb[:nb]}

    def state_export(self, bucket_mask=None):
        """cook_state_export: the live rows (bucket_mask: a uint8 array of a power-of-two length, the rows whose
        bucket is set) in ascending id, as the keyword arguments of abi.make_delta: pass them with reset=True to a
        fresh handle for a copy, or as they are to repair those rows."""
        mask = np.ascontiguousarray(bucket_mask, np.uint8) if bucket_mask is not None else None
        args = (self.pool, len(mask) if mask is not None else 0, abi.ptr(mask, abi.P_U8) if mask is not None else None)
        n = abi.StateSizes()
        rc = self.lib.cook_state_export(*args, None, None, C.byref(n))
        if rc != 0:
            self._err(rc)
        P, R, E = n.pending, n.running, list(n.entries)
        dt = abi._NP

        def cols(struct, rows, lists):
            kw = {}
            for name, ctype in struct._fields_:
                if name.endswith("_off"):
                    kw[name] = np.zeros(rows + 1, np.int32)
                elif name in lists:
                    kw[name] = np.zeros(max(lists[name], 1), np.int32)
                else:
                    kw[name] = np.zeros(max(rows, 1), dt[ctype])
            return kw
        pk = cols(abi.JobsRows, P, dict(novel_host=E[0], attr_col=E[1], attr_val=E[1], group_idx=E[2]))
        rk = cols(abi.TasksRows, R, {})
        prio, jid, host = np.zeros(max(P, 1), np.int32), np.zeros(max(P, 1), np.int64), np.zeros(max(R, 1), np.int32)
        goff, gidx = np.zeros(R + 1, np.int32), np.zeros(max(E[3], 1), np.int32)
        rows = abi.StateRows(pending=abi.JobsRows(**pk), pending_priority=prio, pending_job_id=jid,
                             running=abi.TasksRows(**rk), running_hostname_id=host, running_group_off=goff,
                             running_group_idx=gidx)
        got = abi.StateSizes()
        rc = self.lib.cook_state_export(*args, C.byref(n), C.byref(rows), C.byref(got))
        if rc != 0:
            self._err(rc)
        assert (got.pending, got.running, list(got.entries)) == (P, R, E)
        pk = {k: v if k.endswith("_off") or k in ("novel_host", "attr_col", "attr_val", "group_idx") else v[:P]
              for k, v in pk.items()}
        return dict(pending=abi.JobsSoA(n=P, **pk), pending_priority=prio[:P], pending_job_id=jid[:P],
                    running=abi.TasksSoA(n=R, **{k: v[:R] for k, v in rk.items()}), running_hostname_id=host[:R],
                    running_group_off=goff, running_group_idx=gidx)

    def state_queue(self):
        """cook_state_queue: the job ids cook_state_match would read now, in queue order."""
        n = C.c_int32(0)
        rc = self.lib.cook_state_queue(self.pool, 0, None, C.byref(n))
        if rc != 0:
            self._err(rc)
        out = np.zeros(max(n.value, 1), np.int64)
        rc = self.lib.cook_state_queue(self.pool, n.value, abi.ptr(out, abi.P_I64), C.byref(n))
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

    def state_offers_add(self, offers, offer_id, now_ms, single_shot=None, offer_gpus=None, hostnames=None):
        """cook_state_offers_add: one row per arriving offer (an abi.OffersSoA, not merged), stamped now_ms.
        hostnames: each row's hostname (str or bytes; "" or None for a code the handle already knows)."""
        ids = np.ascontiguousarray(offer_id, np.int64)
        ss = np.ascontiguousarray(single_shot, np.uint8) if single_shot is not None else None
        og = np.ascontiguousarray(offer_gpus, np.float64) if offer_gpus is not None else None
        blob, off = b"", None
        if hostnames is not None:
            parts = [h.encode() if isinstance(h, str) else bytes(h or b"") for h in hostnames]
            blob = b"".join(parts)
            off = np.zeros(len(parts) + 1, np.int32)
            off[1:] = np.cumsum([len(b) for b in parts])
        rc = self.lib.cook_state_offers_add(self.pool, C.byref(offers), abi.ptr(ids, abi.P_I64),
                                            abi.ptr(ss, abi.P_U8) if ss is not None else None,
                                            abi.ptr(og, abi.P_F64) if og is not None else None,
                                            blob or None, abi.ptr(off, abi.P_I32) if off is not None else None,
                                            C.c_int64(int(now_ms)))
        if rc != 0:
            self._err(rc)
        live = getattr(self, "_state_offer_ids", set())
        live.update(ids.tolist())
        self._state_offer_ids = live

    def state_match_offers(self, now_ms, incubate_ms, users, params, groups=None, pool_quota=None, max_ports=0,
                           gone_cap=None):
        """cook_state_match_offers: expiry, the merge of the live offers per hostname, the match over the resident
        queue, the consumption.  'considerable' holds job ids, 'assign' hostname codes (-1: unplaced); 'gone' lists
        (offer id, fate) in arrival order."""
        pool_quota = pool_quota or abi.make_pool_quota(None)
        k = max(params.num_considerable, 1)
        cons = np.full(k, -1, np.int64)
        _, assign, ports, fail, stats = _CallShapes.match_buffers(params, max_ports)
        live = getattr(self, "_state_offer_ids", set())
        cap = len(live) if gone_cap is None else gone_cap
        gid = np.full(max(cap, 1), -1, np.int64)
        gfate = np.zeros(max(cap, 1), np.uint8)
        ng = C.c_int32(0)
        rc = self.lib.cook_state_match_offers(self.pool, C.c_int64(int(now_ms)), C.c_int64(int(incubate_ms)),
                                              C.byref(groups) if groups is not None else None, C.byref(users),
                                              C.byref(pool_quota), C.byref(params), abi.ptr(cons, abi.P_I64),
                                              abi.ptr(assign, abi.P_I32),
                                              abi.ptr(ports, abi.P_I32) if max_ports > 0 else None, int(max_ports),
                                              abi.ptr(fail, abi.P_U8), abi.ptr(gid, abi.P_I64),
                                              abi.ptr(gfate, abi.P_U8), int(cap), C.byref(ng), C.byref(stats))
        if rc != 0:
            self._err(rc)
        n = stats.n_considerable
        gone = list(zip(gid[:ng.value].tolist(), gfate[:ng.value].tolist()))
        live.difference_update(g for g, _ in gone)
        return {"considerable": cons[:n].copy(), "assign": assign[:n].copy(),
                "ports": ports[:n * max(max_ports, 1)].reshape(n, max(max_ports, 1)).copy(),
                "fail": fail[:n].copy(), "gone": gone, "stats": stats.as_dict()}

    def state_unscheduled(self, job_id):
        """cook_state_unscheduled: per queried job id, 'status' (abi.UNSCHED_*), 'usage' [n, 4] (count, cpus, mem, gpus of
        the user's running jobs plus the job; WAITING only), 'position' (-1: neither waiting nor running), 'ahead' (a
        list per query of the job ids of the first min(position, abi.UNSCHED_AHEAD) entries ahead), 'plugin_deferred',
        and 'stats', the call's own phase statistics.  Changes nothing on the handle."""
        jid = np.ascontiguousarray(job_id, np.int64)
        n = len(jid)
        m = max(n, 1)
        status, plugin = np.zeros(m, np.uint8), np.zeros(m, np.uint8)
        usage = np.zeros((m, 4))
        pos, na = np.zeros(m, np.int32), np.zeros(m, np.int32)
        ahead = np.zeros((m, abi.UNSCHED_AHEAD), np.int64)
        st = abi.PhaseStats()
        rc = self.lib.cook_state_unscheduled(self.pool, n, abi.ptr(jid, abi.P_I64) if n else None,
                                             abi.ptr(status, abi.P_U8), abi.ptr(usage, abi.P_F64),
                                             abi.ptr(pos, abi.P_I32), abi.ptr(na, abi.P_I32),
                                             abi.ptr(ahead, abi.P_I64), abi.ptr(plugin, abi.P_U8), C.byref(st))
        if rc != 0:
            self._err(rc)
        return {"job_id": jid, "status": status[:n], "usage": usage[:n], "position": pos[:n],
                "ahead": [ahead[i, :na[i]].tolist() for i in range(n)], "ahead_raw": ahead[:n],
                "plugin_deferred": plugin[:n], "stats": st.as_dict()}

    def state_rebalance(self, hosts, users, params, groups=None, derived=False, offers=False):
        """cook_state_rebalance: the rebalancer over the live running tasks and the first allowed jobs of the
        resident queue.  As rebalance(), plus each decision's 'job_id'; 'victims' are task ids (the task
        of the job an earlier decision e placed: -1 - e).  derived: cook_state_rebalance_derived, the groups'
        cot_* read from the resident running rows over `hosts` on the device (those fields are ignored).  offers:
        cook_state_rebalance_offers, the derived call with the hosts' spare resources from the live offers."""
        mp = max(params.max_preemption, 1)
        dec = (abi.Decision * mp)()
        jid = np.full(mp, -1, np.int64)
        cap = len(getattr(self, "_state_running_ids", ())) + mp
        vict = np.full(cap, -1, np.int64)
        n = C.c_int32(0)
        fn = (self.lib.cook_state_rebalance_offers if offers else
              self.lib.cook_state_rebalance_derived if derived else self.lib.cook_state_rebalance)
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


def state_sweep(engines, now_ms, default_timeout_ms, max_timeout_ms, groups=None, lists=("linger", "cancel", "straggler")):
    """cook_state_sweep over the live running rows of `engines` (one device, the work on engines[0]'s stream).
    groups: {"kind", "quantile", "multiplier", "n_jobs"} arrays by group code (None: no group).  lists: which of
    "linger", "cancel" and "straggler" to sweep.  Returns 'linger' and 'cancel' as [(task id, engine index)],
    'straggler' as [(group, task id, engine index)] (a list not asked for: None), and 'stats' (the call's own)."""
    if not engines:
        raise ValueError("state_sweep: at least one handle")
    g = groups or {}
    G = len(g.get("kind", ()))
    kind = np.ascontiguousarray(g.get("kind", ()), np.int32)
    q = np.ascontiguousarray(g.get("quantile", ()), np.float64)
    m = np.ascontiguousarray(g.get("multiplier", ()), np.float64)
    nj = np.ascontiguousarray(g.get("n_jobs", ()), np.int32)
    if not len(kind) == len(q) == len(m) == len(nj):
        raise ValueError("state_sweep: the group columns differ in length")
    R = sum(len(getattr(e, "_state_running_ids", ())) for e in engines)
    N = sum(sum(e._group_lengths()[1].values()) for e in engines)
    out = {}
    for k, n_cols, cap in (("linger", 2, R), ("cancel", 2, R), ("straggler", 3, N)):
        if k in lists:
            cols = ([np.zeros(max(cap, 1), np.int32)] if n_cols == 3 else []) + [np.zeros(max(cap, 1), np.int64),
                                                                              np.zeros(max(cap, 1), np.int32)]
            out[k] = (cols, C.c_int32(0))
    def arg(k, i):
        if k not in out:
            return None
        a = out[k][0][i]
        return abi.ptr(a, abi.P_I64 if a.dtype == np.int64 else abi.P_I32)
    cnt = lambda k: C.byref(out[k][1]) if k in out else None
    st = abi.PhaseStats()
    handles = (C.c_void_p * len(engines))(*[e.pool for e in engines])
    rc = engines[0].lib.cook_state_sweep(
        handles, len(engines), int(now_ms), int(default_timeout_ms), int(max_timeout_ms), G,
        abi.ptr(kind, abi.P_I32) if G else None, abi.ptr(q, abi.P_F64) if G else None,
        abi.ptr(m, abi.P_F64) if G else None, abi.ptr(nj, abi.P_I32) if G else None, R, arg("linger", 0),
        arg("linger", 1), cnt("linger"), arg("cancel", 0), arg("cancel", 1), cnt("cancel"), N, arg("straggler", 0),
        arg("straggler", 1), arg("straggler", 2), cnt("straggler"), C.byref(st))
    if rc != 0:
        engines[0]._err(rc)
    res = {"stats": st.as_dict()}
    for k in ("linger", "cancel", "straggler"):
        if k not in out:
            res[k] = None
            continue
        cols, n = out[k]
        res[k] = list(zip(*[c[:n.value].tolist() for c in cols]))
    return res


def state_user_usage(engines, users=None, per_pool=False, by_group=False):
    """cook_state_user_usage over the live running rows of `engines` (one device, the work on engines[0]'s stream) for
    the user codes `users` (None: every user).  Returns the segments as numpy columns 'user', 'scope' (-1: every
    handle, else the engine index), 'group' (abi.UU_TOTAL, abi.UU_UNGROUPED or a group code), 'jobs' (int64), 'cpus',
    'mem', 'gpus', and with by_group 'list_off' and 'job_id' (the group segments' job ids, in segment order), plus
    'lists' (per segment its job ids, None for a total) and 'stats', the call's own phase statistics.  The capacities
    are sized from the engines' live running ids."""
    if not engines:
        raise ValueError("state_user_usage: at least one handle")
    q = np.ascontiguousarray(users if users is not None else (), np.int32)
    R = sum(len(getattr(e, "_state_running_ids", ())) for e in engines)
    L = (1 + bool(per_pool)) * (1 + bool(by_group))
    seg_cap, job_cap = R * L, R * (1 + bool(per_pool)) if by_group else 0
    m = max(seg_cap, 1)
    u, sc, g, off = (np.zeros(m, np.int32) for _ in range(4))
    jobs = np.zeros(m, np.int64)
    cpus, mem, gpus = np.zeros(m), np.zeros(m), np.zeros(m)
    jid = np.zeros(max(job_cap, 1), np.int64)
    n_seg, n_job = C.c_int32(0), C.c_int32(0)
    st = abi.PhaseStats()
    handles = (C.c_void_p * len(engines))(*[e.pool for e in engines])
    rc = engines[0].lib.cook_state_user_usage(
        handles, len(engines), abi.ptr(q, abi.P_I32) if users is not None else None, len(q), int(bool(per_pool)),
        int(bool(by_group)), seg_cap, abi.ptr(u, abi.P_I32), abi.ptr(sc, abi.P_I32), abi.ptr(g, abi.P_I32),
        abi.ptr(jobs, abi.P_I64), abi.ptr(cpus, abi.P_F64), abi.ptr(mem, abi.P_F64), abi.ptr(gpus, abi.P_F64),
        abi.ptr(off, abi.P_I32) if by_group else None, job_cap, abi.ptr(jid, abi.P_I64) if by_group else None,
        C.byref(n_seg), C.byref(n_job), C.byref(st))
    if rc != 0:
        engines[0]._err(rc)
    n, nj = n_seg.value, n_job.value
    out = {"user": u[:n], "scope": sc[:n], "group": g[:n], "jobs": jobs[:n], "cpus": cpus[:n], "mem": mem[:n],
           "gpus": gpus[:n], "stats": st.as_dict()}
    if by_group:
        out["list_off"], out["job_id"] = off[:n], jid[:nj]
    out["lists"] = [None if not by_group or out["group"][d] == abi.UU_TOTAL else
                    jid[off[d]:off[d] + jobs[d]].tolist() for d in range(n)]
    return out


def state_list_jobs(engines, user, states, start_ms, end_ms, job_id_lo=-(1 << 63), job_id_hi=(1 << 63) - 1,
                    pool_code=-1, handle_pool=None, include_custom_executor=True, limit=(1 << 31) - 1, cap=1024):
    """cook_state_list_jobs over the live rows of `engines` (one device, the work on engines[0]'s stream): user code
    `user`'s jobs in `states` (abi.LJ_WAITING | abi.LJ_RUNNING) submitted in [start_ms, end_ms), with job ids in
    [job_id_lo, job_id_hi), in the pool `pool_code` (-1: any; handle_pool: each engine's pool code), each state cut to
    `limit`.  Returns 'state', 'job_id', 'submit_ms' and 'pool' (the engine index) as numpy columns, waiting entries
    first, each state in ascending (job id, pool); 'missing', the rows in the window without list facts; and 'stats',
    the call's own phase statistics.  The call is made with `cap` entries first and, when more are needed, once more
    with the count it reports."""
    if not engines:
        raise ValueError("state_list_jobs: at least one handle")
    hp = np.ascontiguousarray(handle_pool if handle_pool is not None else (), np.int32)
    if handle_pool is not None and len(hp) != len(engines):
        raise ValueError("state_list_jobs: handle_pool differs in length from engines")
    handles = (C.c_void_p * len(engines))(*[e.pool for e in engines])
    n, missing = C.c_int32(0), C.c_int32(0)
    st = abi.PhaseStats()
    cap = max(int(cap), 0)
    for _ in range(2):
        m = max(cap, 1)
        state, pool = np.zeros(m, np.int32), np.zeros(m, np.int32)
        jid, sub = np.zeros(m, np.int64), np.zeros(m, np.int64)
        rc = engines[0].lib.cook_state_list_jobs(
            handles, len(engines), int(user), int(states), int(start_ms), int(end_ms), int(job_id_lo), int(job_id_hi),
            int(pool_code), abi.ptr(hp, abi.P_I32) if handle_pool is not None else None, int(bool(include_custom_executor)),
            int(limit), cap, abi.ptr(state, abi.P_I32), abi.ptr(jid, abi.P_I64), abi.ptr(sub, abi.P_I64),
            abi.ptr(pool, abi.P_I32), C.byref(n), C.byref(missing), C.byref(st))
        if rc != abi.COOK_E_TOO_LARGE or n.value <= cap:
            break
        cap = n.value
    if rc != 0:
        engines[0]._err(rc)
    k = n.value
    return {"state": state[:k], "job_id": jid[:k], "submit_ms": sub[:k], "pool": pool[:k], "missing": missing.value,
            "stats": st.as_dict()}


def state_list_completed(engines, user, state, start_ms, end_ms, job_id_lo=-(1 << 63), job_id_hi=(1 << 63) - 1,
                         pool_code=-1, handle_pool=None, include_custom_executor=True, limit=(1 << 31) - 1, cap=1024):
    """cook_state_list_completed over the completed-job logs of `engines` (on one device or several: the work runs on
    engines[0]'s stream, each other device's records of the user gathered to it): user code `user`'s jobs whose latest record is of `state` (abi.LC_SUCCESS, abi.LC_FAILED or
    abi.LC_COMPLETED), submitted in [start_ms, end_ms), with job ids in [job_id_lo, job_id_hi), in the pool `pool_code`
    (-1: any; handle_pool: each engine's pool code), cut to `limit`.  Returns 'job_id', 'submit_ms' and 'pool' (the
    engine index of the latest record) as numpy columns in ascending job id, and 'stats', the call's own phase
    statistics.  The call is made with `cap` entries first and, when more are needed, once more with the count it
    reports."""
    if not engines:
        raise ValueError("state_list_completed: at least one handle")
    hp = np.ascontiguousarray(handle_pool if handle_pool is not None else (), np.int32)
    if handle_pool is not None and len(hp) != len(engines):
        raise ValueError("state_list_completed: handle_pool differs in length from engines")
    handles = (C.c_void_p * len(engines))(*[e.pool for e in engines])
    n = C.c_int32(0)
    st = abi.PhaseStats()
    cap = max(int(cap), 0)
    for _ in range(2):
        m = max(cap, 1)
        pool = np.zeros(m, np.int32)
        jid, sub = np.zeros(m, np.int64), np.zeros(m, np.int64)
        rc = engines[0].lib.cook_state_list_completed(
            handles, len(engines), int(user), int(state), int(start_ms), int(end_ms), int(job_id_lo), int(job_id_hi),
            int(pool_code), abi.ptr(hp, abi.P_I32) if handle_pool is not None else None, int(bool(include_custom_executor)),
            int(limit), cap, abi.ptr(jid, abi.P_I64), abi.ptr(sub, abi.P_I64), abi.ptr(pool, abi.P_I32), C.byref(n),
            C.byref(st))
        if rc != abi.COOK_E_TOO_LARGE or n.value <= cap:
            break
        cap = n.value
    if rc != 0:
        engines[0]._err(rc)
    k = n.value
    return {"job_id": jid[:k], "submit_ms": sub[:k], "pool": pool[:k], "stats": st.as_dict()}


def _is_answer(engines, call, cap):
    """One cook_state_instance_stats or cook_state_history_stats call with segment capacity `cap`: call(handles,
    outputs...) -> rc.  Returns (rc, the answer, or the segments needed when rc is COOK_E_TOO_LARGE)."""
    kind, user, reason = (np.zeros(cap, np.int32) for _ in range(3))
    count = np.zeros(cap, np.int64)
    total, pct = np.zeros((cap, 3)), np.zeros((cap, 3, 5))
    lu, lt = np.zeros(2 * abi.IS_LEADERS, np.int32), np.zeros(2 * abi.IS_LEADERS)
    n_seg, n_lead = C.c_int32(0), C.c_int32(0)
    st = abi.PhaseStats()
    handles = (C.c_void_p * len(engines))(*[e.pool for e in engines])
    rc = call(handles, cap, abi.ptr(kind, abi.P_I32), abi.ptr(user, abi.P_I32), abi.ptr(reason, abi.P_I32),
              abi.ptr(count, abi.P_I64), abi.ptr(total, abi.P_F64), abi.ptr(pct, abi.P_F64), abi.ptr(lu, abi.P_I32),
              abi.ptr(lt, abi.P_F64), C.byref(n_seg), C.byref(n_lead), C.byref(st))
    if rc != 0:
        return rc, n_seg.value
    n, L = n_seg.value, n_lead.value
    lead = lambda k: [(int(lu[k * abi.IS_LEADERS + i]), float(lt[k * abi.IS_LEADERS + i])) for i in range(L)]
    return rc, {"kind": kind[:n], "user": user[:n], "reason": reason[:n], "count": count[:n], "total": total[:n],
                "pct": pct[:n], "leaders_cpu": lead(0), "leaders_mem": lead(1), "stats": st.as_dict()}


def state_instance_stats(engines, now_ms, status, start_ms, end_ms, task_id_lo=-(1 << 63), task_id_hi=(1 << 63) - 1):
    """cook_state_instance_stats over the live running rows of `engines` (on one device or several: the work runs on
    engines[0]'s stream, each other device's rows gathered to it):
    the rows of `status` (abi.IS_RUNNING or abi.IS_UNKNOWN) with task_id_lo <= task id < task_id_hi and start_ms <=
    start < end_ms.  Returns the segments as numpy columns 'kind', 'user', 'reason', 'count' (int64), 'total' [n, 3]
    and 'pct' [n, 3, 5] (metrics by abi.IS_RUN_TIME / IS_CPU / IS_MEM, percentiles 50 75 95 99 100), the leaders
    'leaders_cpu' and 'leaders_mem' as [(user, total)], and 'stats', the call's own phase statistics.  The segment
    capacity is sized from the engines' live running ids."""
    if not engines:
        raise ValueError("state_instance_stats: at least one handle")
    R = sum(len(getattr(e, "_state_running_ids", ())) for e in engines)
    rc, out = _is_answer(engines, lambda h, cap, *o: engines[0].lib.cook_state_instance_stats(
        h, len(engines), int(now_ms), int(status), int(start_ms), int(end_ms), int(task_id_lo), int(task_id_hi), cap,
        *o), 1 + 2 * R)
    if rc != 0:
        engines[0]._err(rc)
    return out


def state_history_stats(engines, status, start_ms, end_ms, task_id_lo=-(1 << 63), task_id_hi=(1 << 63) - 1,
                        seg_cap=16384):
    """cook_state_history_stats over the finished rows of `engines`' histories (on one device or several: each other
    device's selection gathered to engines[0]'s): the rows of `status`
    (abi.IS_SUCCESS or abi.IS_FAILED) with task_id_lo <= task id < task_id_hi and start_ms <= start < end_ms.  Returns
    state_instance_stats' answer shape, so cycle.instance_stats_response builds the response unchanged.  The call is
    made with seg_cap segments first and, when more are needed, once more with the count it reports."""
    if not engines:
        raise ValueError("state_history_stats: at least one handle")
    call = lambda h, cap, *o: engines[0].lib.cook_state_history_stats(
        h, len(engines), int(status), int(start_ms), int(end_ms), int(task_id_lo), int(task_id_hi), cap, *o)
    rc, out = _is_answer(engines, call, max(int(seg_cap), 1))
    if rc == abi.COOK_E_TOO_LARGE and out > seg_cap:
        rc, out = _is_answer(engines, call, out)
    if rc != 0:
        engines[0]._err(rc)
    return out


STATS_KEYS = ("running", "waiting", "starved", "waiting-under-quota")   # by abi.STATS_*
USER_COUNTS = ("total", "starved", "waiting-under-quota", "hungry", "satisfied")   # by abi.USERS_*


def state_user_stats(engines, users, quota_rest_ok=None):
    """cook_state_user_stats over the live rows of `engines` (one pool, or the pools of a quota group, on one device or
    several: the work runs on engines[0]'s stream, each other device's rows gathered to it).  quota_rest_ok: per user code, whether the user's other quota keys are all > 0
    (None: all).  Returns 'jobs' (int64), 'cpus' and 'mem' as [4, n_users] arrays by abi.STATS_*, 'member' [n_users]
    (bit s: the user is in state s), 'all' {state: (jobs, cpus, mem)} and 'users' {count name: n}, keyed by
    STATS_KEYS and USER_COUNTS, and 'stats', the call's own phase statistics (abi.PhaseStats.as_dict())."""
    if not engines:
        raise ValueError("state_user_stats: at least one handle")
    U = int(users.n_users)
    ok = np.ascontiguousarray(quota_rest_ok, np.uint8) if quota_rest_ok is not None else None
    if ok is not None and len(ok) != U:
        raise ValueError("state_user_stats: quota_rest_ok needs one flag per user")
    n = max(U, 1)
    jobs, cpus, mem = np.zeros((4, n), np.int64), np.zeros((4, n)), np.zeros((4, n))
    member = np.zeros(n, np.uint8)
    aj, ac, am = np.zeros(4, np.int64), np.zeros(4), np.zeros(4)
    counts = np.zeros(abi.USERS_N, np.int64)
    st = abi.PhaseStats()
    handles = (C.c_void_p * len(engines))(*[e.pool for e in engines])
    rc = engines[0].lib.cook_state_user_stats(
        handles, len(engines), C.byref(users), abi.ptr(ok, abi.P_U8) if ok is not None else None,
        abi.ptr(jobs, abi.P_I64), abi.ptr(cpus, abi.P_F64), abi.ptr(mem, abi.P_F64), abi.ptr(member, abi.P_U8),
        abi.ptr(aj, abi.P_I64), abi.ptr(ac, abi.P_F64), abi.ptr(am, abi.P_F64), abi.ptr(counts, abi.P_I64), C.byref(st))
    if rc != 0:
        engines[0]._err(rc)
    return {"jobs": jobs[:, :U], "cpus": cpus[:, :U], "mem": mem[:, :U], "member": member[:U],
            "all": {k: (int(aj[s]), float(ac[s]), float(am[s])) for s, k in enumerate(STATS_KEYS)},
            "users": {k: int(counts[i]) for i, k in enumerate(USER_COUNTS)}, "stats": st.as_dict()}


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
