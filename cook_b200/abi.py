"""ctypes mirror of include/cook_gpu.h.

Host-side marshalling only: every struct here is a field-for-field mirror of the
C ABI that the JVM shim (INTEGRATION.md) fills from direct ByteBuffers.  Nothing
in this module computes anything; it packs numpy columns into the SoA structs.
"""
import ctypes as C

import numpy as np

P_I32 = C.POINTER(C.c_int32)
P_I64 = C.POINTER(C.c_int64)
P_F64 = C.POINTER(C.c_double)
P_U8 = C.POINTER(C.c_uint8)

_NP = {P_I32: np.int32, P_I64: np.int64, P_F64: np.float64, P_U8: np.uint8}

COOK_OK = 0
COOK_E_BADARG = -1
COOK_E_CUDA = -2
COOK_E_NCCL = -3
COOK_E_OOM = -4
COOK_E_UNSUPPORTED_CONSTRAINT = -5
COOK_E_NO_DEVICE = -6
COOK_E_TOO_LARGE = -7

GROUP_UNIQUE, GROUP_BALANCED, GROUP_ATTR_EQUALS = 0, 1, 2
FAIL_NONE, FAIL_RESOURCES, FAIL_CONSTRAINT, FAIL_NO_OFFERS = 0, 1, 2, 3

INT64_MAX = np.iinfo(np.int64).max


class _SoA(C.Structure):
    """Base: keeps the numpy arrays referenced by pointer fields alive."""

    def __init__(self, **kw):
        super().__init__()
        self._keep = {}
        for name, ctype in self._fields_:
            if name not in kw or kw[name] is None:
                continue
            val = kw[name]
            if ctype in _NP:
                arr = np.ascontiguousarray(val, dtype=_NP[ctype])
                self._keep[name] = arr
                setattr(self, name, arr.ctypes.data_as(ctype))
            elif isinstance(val, _SoA):
                self._keep[name] = val
                setattr(self, name, val)
            else:
                setattr(self, name, val)
        unknown = set(kw) - {n for n, _ in self._fields_}
        if unknown:
            raise TypeError(f"unknown fields for {type(self).__name__}: {sorted(unknown)}")

    def col(self, name):
        """The numpy array behind a pointer field (or None)."""
        return self._keep.get(name)


class TasksSoA(_SoA):
    _fields_ = [("n", C.c_int32), ("user", P_I32), ("priority", P_I32),
                ("start_time", P_I64), ("task_id", P_I64), ("job_id", P_I64),
                ("cpus", P_F64), ("mem", P_F64), ("gpus", P_F64)]


class UserTable(_SoA):
    _fields_ = [("n_users", C.c_int32), ("name_rank", P_I32),
                ("div_mem", P_F64), ("div_cpus", P_F64), ("div_gpus", P_F64),
                ("quota_count", P_F64), ("quota_cpus", P_F64), ("quota_mem", P_F64),
                ("quota_gpus", P_F64),
                ("usage_count", P_F64), ("usage_cpus", P_F64), ("usage_mem", P_F64),
                ("usage_gpus", P_F64), ("tokens", P_I32)]


class PoolQuota(C.Structure):
    _fields_ = [("enabled", C.c_int32), ("count", C.c_double), ("cpus", C.c_double),
                ("mem", C.c_double), ("gpus", C.c_double)]


class RankParams(C.Structure):
    _fields_ = [("max_over_quota_jobs", C.c_int32), ("filter_offensive", C.c_int32),
                ("offensive_max_mem_mb", C.c_double), ("offensive_max_cpus", C.c_double)]


class JobsSoA(_SoA):
    _fields_ = [("n", C.c_int32), ("user", P_I32), ("cpus", P_F64), ("mem", P_F64),
                ("gpus", P_F64), ("ports", P_I32), ("allowed", P_U8), ("plugin_accept", P_U8),
                ("novel_off", P_I32), ("novel_host", P_I32), ("gpu_model", P_I32),
                ("disk_request", P_F64), ("disk_type", P_I32),
                ("attr_off", P_I32), ("attr_col", P_I32), ("attr_val", P_I32),
                ("est_end_ms", P_I64), ("ckpt_location", P_I32), ("reserved_host", P_I32),
                ("group_off", P_I32), ("group_idx", P_I32)]


class OffersSoA(_SoA):
    _fields_ = [("n", C.c_int32), ("hostname_id", P_I32), ("name_rank", P_I32),
                ("cpus", P_F64), ("mem", P_F64), ("run_cpus", P_F64), ("run_mem", P_F64),
                ("run_count", P_I32), ("port_off", P_I32), ("port_begin", P_I32),
                ("port_end", P_I32), ("is_k8s", P_U8), ("location", P_I32),
                ("gpu_off", P_I32), ("gpu_model", P_I32), ("gpu_count", P_F64),
                ("disk_off", P_I32), ("disk_type", P_I32), ("disk_space", P_F64),
                ("max_tasks", P_I32), ("num_tasks", P_I32), ("host_start_time", P_I64),
                ("n_attr_cols", C.c_int32), ("attr", P_I32), ("reserved", P_U8)]


class Groups(_SoA):
    _fields_ = [("n_groups", C.c_int32), ("kind", P_I32), ("attr_col", P_I32),
                ("minimum", P_I32), ("cot_off", P_I32), ("cot_hostname_id", P_I32),
                ("cot_attr_val", P_I32)]


class MatchParams(C.Structure):
    _fields_ = [("num_considerable", C.c_int32), ("enforce_rate_limit", C.c_int32),
                ("host_lifetime_mins", C.c_int32), ("fitness_kind", C.c_int32),
                ("good_enough_fitness", C.c_double), ("reuse_resident", C.c_int32),
                ("max_ctas", C.c_int32)]


class MatchStats(C.Structure):
    _fields_ = [("n_considerable", C.c_int32), ("n_matched", C.c_int32),
                ("head_matched", C.c_int32), ("n_offers_used", C.c_int32),
                ("evals", C.c_int64), ("n_fast", C.c_int64), ("n_chunk_rescan", C.c_int64),
                ("n_full_rescan", C.c_int64), ("ms_considerable", C.c_double),
                ("ms_match", C.c_double), ("ms_h2d", C.c_double), ("ms_d2h", C.c_double),
                ("ms_match_kernel", C.c_double), ("h2d_bytes", C.c_int64),
                ("d2h_bytes", C.c_int64), ("n_launches", C.c_int32), ("reserved0", C.c_int32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class PhaseStats(C.Structure):
    _fields_ = [("ms_h2d", C.c_double), ("ms_device", C.c_double), ("ms_d2h", C.c_double),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("n_launches", C.c_int32),
                ("reserved0", C.c_int32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved0"}


PHASE_RANK, PHASE_MATCH, PHASE_REBALANCE, PHASE_EXCHANGE, PHASE_STATE, PHASE_USAGE, PHASE_COTASKS = 0, 1, 2, 3, 4, 5, 6
PHASE_CONSIDERABLE = 7
PHASE_AUDIT = 8

# cook_state_user_stats: the state rows of its [4][n_users] outputs and the order of its user counts
STATS_RUNNING, STATS_WAITING, STATS_STARVED, STATS_WUQ = 0, 1, 2, 3
USERS_TOTAL, USERS_STARVED, USERS_WUQ, USERS_HUNGRY, USERS_SATISFIED, USERS_N = 0, 1, 2, 3, 4, 5

USAGE_GIVEN, USAGE_DERIVED, USAGE_LAST_MATCH = 0, 1, 2
# cook_state_sweep: a group's straggler handling
SWEEP_NONE, SWEEP_QUANTILE_DEVIATION = 0, 1
# cook_state_match_offers: why an offer left the live set
OFFER_USED, OFFER_EXPIRED, OFFER_SINGLE_SHOT = 1, 2, 3
# cook_state_unscheduled: a queried job's status, and the most job ids ahead it returns
UNSCHED_ABSENT, UNSCHED_WAITING, UNSCHED_RUNNING, UNSCHED_AHEAD = 0, 1, 2, 10
# cook_state_user_usage: a segment's group when it is the scope's total, or its jobs without a group
UU_TOTAL, UU_UNGROUPED = -2, -1
# cook_state_instance_stats (running, unknown) and cook_state_history_stats (success, failed): the statuses, the
# segment kinds, the metrics and the leaders' places
IS_RUNNING, IS_UNKNOWN, IS_SUCCESS, IS_FAILED = 0, 1, 2, 3
IS_OVERALL, IS_REASON, IS_USER_REASON = 0, 1, 2
IS_RUN_TIME, IS_CPU, IS_MEM, IS_LEADERS = 0, 1, 2, 10

# cook_state_job_facts' bits and cook_state_match_metrics' key kinds and first-ten length
JF_GPUS, JF_DISK, JF_DISK_REQUEST, JF_DISK_LIMIT, JF_URIS = 1, 2, 4, 8, 16
MM_GPUS, MM_DISK_REQUEST, MM_DISK_LIMIT = 0, 1, 2
MM_FIRST_N = 10

# cook_state_list_jobs' states
LJ_WAITING, LJ_RUNNING = 1, 2
# cook_state_completed_*: a record's kind; cook_state_list_completed: the listed state
CJ_SUCCESS, CJ_FAILED, CJ_REOPENED = 1, 2, 3
LC_SUCCESS, LC_FAILED, LC_COMPLETED = 1, 2, 3

# cook_state_retry_facts' bits and cook_state_status' outcomes
RF_DISABLE_MEA_CULPA, RF_COMPLETED = 1, 2
JOB_COMPLETED, JOB_RUNNING, JOB_WAITING, JOB_WAITING_UNRETAINED, JOB_NO_FACTS = 0, 1, 2, 3, 4

MMC_CONSIDERABLE, MMC_MATCHED, MMC_HEAD_JOB_ID, MMC_HEAD_MATCHED, MMC_URIS, MMC_URIS_POSITION, MMC_KEYS = 0, 1, 2, 3, 4, 5, 6
MMC_TOO_LONG, MMC_FIRST, MMC_N = 7, 8, 9
MMA_TOTAL_CPUS, MMA_TOTAL_MEM, MMA_PCT_CPUS, MMA_PCT_MEM, MMA_N = 0, 1, 2, 5, 8
MM_HEAD, MM_LARGEST_CPUS, MM_LARGEST_MEM, MM_ROWS = 0, 1, 2, 3
MMR_INT = ("job_id", "position", "user", "ports", "facts", "gpu_model", "disk_type")    # by COOK_MMR_*, integers
MMR_AMOUNT = ("cpus", "mem", "gpus", "disk_request", "disk_limit")                        # by COOK_MMR_*, amounts

class ConsiderableParams(C.Structure):
    """cook_considerable_params: M0 over the resident queue (cook_state_considerable)."""
    _fields_ = [("num_considerable", C.c_int32), ("enforce_rate_limit", C.c_int32), ("quota_only", C.c_int32),
                ("usage_source", C.c_int32), ("consume", C.c_int32)]


class StateDelta(_SoA):
    """cook_state_delta: one batch of changes to a handle's resident pool state."""
    _fields_ = [("reset", C.c_int32), ("pending", JobsSoA), ("pending_priority", P_I32),
                ("pending_job_id", P_I64), ("n_pending_rm", C.c_int32), ("pending_rm_job_id", P_I64),
                ("running", TasksSoA), ("n_running_rm", C.c_int32), ("running_rm_task_id", P_I64),
                ("running_hostname_id", P_I32), ("running_group_off", P_I32), ("running_group_idx", P_I32)]


def make_delta(reset=False, pending=None, pending_priority=None, pending_job_id=None, pending_rm=(),
               running=None, running_rm=(), running_hostname_id=None, running_group_off=None,
               running_group_idx=None):
    """A StateDelta; `pending` is a JobsSoA of the upserted rows, `running` a TasksSoA, `running_hostname_id`
    the hostname code of each running row (None: host unknown), `running_group_off` / `running_group_idx` the
    CSR of each running row's group list (csr(); None: empty lists)."""
    pending = pending if pending is not None else JobsSoA(n=0)
    running = running if running is not None else TasksSoA(n=0)
    prm = np.asarray(pending_rm, np.int64)
    rrm = np.asarray(running_rm, np.int64)
    return StateDelta(reset=int(bool(reset)), pending=pending, pending_priority=pending_priority,
                      pending_job_id=pending_job_id, n_pending_rm=len(prm),
                      pending_rm_job_id=prm if len(prm) else None, running=running,
                      n_running_rm=len(rrm), running_rm_task_id=rrm if len(rrm) else None,
                      running_hostname_id=running_hostname_id, running_group_off=running_group_off,
                      running_group_idx=running_group_idx)


class Fp(C.Structure):
    """cook_fp: the fingerprint of a set of rows."""
    _fields_ = [("sum", C.c_uint64), ("xr", C.c_uint64), ("n", C.c_int64)]

    def as_tuple(self):
        return (self.sum, self.xr, self.n)


FP_DTYPE = np.dtype([("sum", np.uint64), ("xr", np.uint64), ("n", np.int64)])   # a cook_fp array

# COOK_AUDIT_*: the counts cook_state_digest recounts, by index
AUDIT_NAMES = (["pending_rows", "running_rows", "entries_novel", "entries_attr", "entries_group", "entries_running_group"]
               + ["flag_" + f for f in ("gpus", "ports", "not_allowed", "not_plugin", "gpu_model", "disk", "est_end_ms",
                                        "ckpt_location", "reserved_host")]
               + ["reserved_rows", "cot_rows", "cot_entries", "max_user_pending", "max_user_running",
                  "max_group_pending", "max_group_running", "max_attr_col", "max_hostname_running"])
AUDIT_N = len(AUDIT_NAMES)


class StateDigest(C.Structure):
    """cook_state_digest_out."""
    _fields_ = [("pending", Fp), ("running", Fp), ("queue", Fp), ("entries", C.c_int64 * 4),
                ("consistent", C.c_int32), ("first_mismatch", C.c_int32)]


class JobsRows(_SoA):
    """cook_jobs_rows: cook_jobs_soa's columns, writable."""
    _fields_ = [(n, t) for n, t in JobsSoA._fields_ if n != "n"]


class TasksRows(_SoA):
    _fields_ = [(n, t) for n, t in TasksSoA._fields_ if n != "n"]


class StateRows(_SoA):
    """cook_state_rows: where cook_state_export writes the rows."""
    _fields_ = [("pending", JobsRows), ("pending_priority", P_I32), ("pending_job_id", P_I64),
                ("running", TasksRows), ("running_hostname_id", P_I32), ("running_group_off", P_I32),
                ("running_group_idx", P_I32)]


class StateSizes(C.Structure):
    """cook_state_sizes: rows per table, entries per list (novel, attr, group, running group)."""
    _fields_ = [("pending", C.c_int32), ("running", C.c_int32), ("entries", C.c_int32 * 4)]


class RunningSoA(_SoA):
    _fields_ = [("t", TasksSoA), ("host", P_I32)]


class HostTable(_SoA):
    _fields_ = [("n", C.c_int32), ("hostname_id", P_I32), ("name_rank", P_I32),
                ("has_spare", P_U8), ("spare_cpus", P_F64), ("spare_mem", P_F64),
                ("spare_gpus", P_F64), ("is_k8s", P_U8), ("location", P_I32),
                ("gpu_off", P_I32), ("gpu_model", P_I32), ("gpu_count", P_F64),
                ("disk_off", P_I32), ("disk_type", P_I32), ("disk_space", P_F64),
                ("host_start_time", P_I64), ("n_attr_cols", C.c_int32), ("attr", P_I32)]


class RebalanceParams(C.Structure):
    _fields_ = [("max_preemption", C.c_int32), ("min_dru_diff", C.c_double),
                ("safe_dru_threshold", C.c_double), ("host_lifetime_mins", C.c_int32)]


class Decision(C.Structure):
    _fields_ = [("pending_idx", C.c_int32), ("host", C.c_int32),
                ("victim_begin", C.c_int32), ("victim_count", C.c_int32),
                ("dru", C.c_double), ("mem", C.c_double), ("cpus", C.c_double),
                ("gpus", C.c_double)]


FAILC_N = 13


class FailureCounts(C.Structure):
    _fields_ = [("n_vms", C.c_int32), ("n_passed", C.c_int32), ("n_ports", C.c_int32), ("counts", C.c_int32 * FAILC_N)]


class RebTrace(C.Structure):
    """cook_reb_trace (include/cook_gpu.h): rebalancer state as the reference's own tests read it."""
    _fields_ = [("n_forced", C.c_int32), ("forced", C.POINTER(Decision)),
                ("forced_victims", P_I32), ("pending_dru", P_F64),
                ("task_dru", P_F64), ("task_alive", P_U8), ("order", P_I32),
                ("n_order", C.POINTER(C.c_int32)), ("has_spare", P_U8),
                ("spare_mem", P_F64), ("spare_cpus", P_F64), ("spare_gpus", P_F64),
                ("forced_only", C.c_int32), ("below_quota", P_U8)]


class GpuConfig(C.Structure):
    _fields_ = [("n_devices", C.c_int32), ("device_ids", P_I32)]


def ptr(arr, ctype):
    return arr.ctypes.data_as(ctype)


_H = C.c_void_p                   # an opaque handle (cook_ctx*, cook_pool*) or a void*
_P = C.POINTER
_I32 = C.c_int32
_STATE_MATCH = [_H, _P(OffersSoA), _P(Groups), _P(UserTable), _P(PoolQuota), _P(MatchParams), P_I64, P_I32, P_I32,
                _I32, P_U8, _P(MatchStats)]
_STATE_REBALANCE = [_H, _P(HostTable), _P(Groups), _P(UserTable), _P(RebalanceParams), _P(Decision), P_I64, P_I64,
                    _I32, P_I32]
_REBALANCE = [_H, _P(RunningSoA), _P(JobsSoA), P_I64, P_I32, _P(HostTable), _P(Groups), _P(UserTable),
              _P(RebalanceParams), _P(Decision), P_I32, P_I32]
_STATE_RANK = [_H, _P(UserTable), _P(PoolQuota), _P(PoolQuota), P_F64, _P(RankParams), P_I64, P_I32]
# ctypes argument types of every int32_t entry point of include/cook_gpu.h; engine.load_library sets them, and
# restype c_int32, on each.  The derived calls take exactly cook_state_match's and cook_state_rebalance's arguments.
ARGTYPES = {
    "cook_gpu_init": [_P(GpuConfig), _P(_H)],
    "cook_gpu_shutdown": [_H],
    "cook_pool_open": [_H, C.c_char_p, _I32, _I32, _P(_H)],
    "cook_pool_close": [_H],
    "cook_last_error": [_H, C.c_char_p, _I32],
    "cook_rank": [_H, _P(TasksSoA), _P(TasksSoA), _P(UserTable), _P(PoolQuota), _P(PoolQuota), P_F64, _P(RankParams),
                  P_I32, P_I32, P_F64, P_I32, P_I32],
    "cook_match": [_H, P_I32, _I32, _P(JobsSoA), _P(OffersSoA), _P(Groups), _P(UserTable), _P(PoolQuota),
                   _P(MatchParams), P_I32, P_I32, P_I32, _I32, P_U8, _P(MatchStats)],
    "cook_match_failures": [_H, P_I32, _I32, _P(FailureCounts)],
    "cook_rebalance": _REBALANCE,
    "cook_rebalance_trace": _REBALANCE + [_P(RebTrace)],
    "cook_state_apply": [_H, _P(StateDelta)],
    "cook_state_launch": [_H, _I32, P_I64, P_I64, P_I64, P_I32],
    "cook_state_patch": [_H, _I32, P_I64, P_U8, P_U8, P_I32, _I32],
    "cook_state_rank": _STATE_RANK,
    "cook_state_rank_offensive": _STATE_RANK + [P_I64, _I32, P_I32],
    "cook_state_match": _STATE_MATCH,
    "cook_state_rebalance": _STATE_REBALANCE,
    "cook_state_usage": [_H, _I32, P_F64, P_F64, _I32, P_I32, P_F64, P_F64, P_I32],
    "cook_state_cotasks": [_H, _I32, P_I32, _P(HostTable), _I32, P_I32, P_I32, P_I32, P_I32],
    "cook_state_match_derived": _STATE_MATCH,
    "cook_state_rebalance_derived": _STATE_REBALANCE,
    "cook_state_considerable": [_H, _P(UserTable), _P(PoolQuota), _P(ConsiderableParams), P_I64, P_I32],
    "cook_state_digest": [_H, _I32, _P(StateDigest), _P(Fp), _P(Fp)],
    "cook_state_counts_compare": [P_I64, P_I64, P_I32],
    "cook_state_export": [_H, _I32, P_U8, _P(StateSizes), _P(StateRows), _P(StateSizes)],
    "cook_state_queue": [_H, _I32, P_I64, P_I32],
    "cook_state_offers_add": [_H, _P(OffersSoA), P_I64, P_U8, P_F64, C.c_char_p, P_I32, C.c_int64],
    "cook_state_match_offers": [_H, C.c_int64, C.c_int64, _P(Groups), _P(UserTable), _P(PoolQuota), _P(MatchParams),
                                P_I64, P_I32, P_I32, _I32, P_U8, P_I64, P_U8, _I32, P_I32, _P(MatchStats)],
    "cook_state_rebalance_offers": _STATE_REBALANCE,
    "cook_state_user_stats": [_P(_H), _I32, _P(UserTable), P_U8, P_I64, P_F64, P_F64, P_U8, P_I64, P_F64, P_F64, P_I64,
                              _P(PhaseStats)],
    "cook_state_task_facts": [_H, _I32, P_I64, P_I64, P_U8, P_U8],
    "cook_state_task_reason": [_H, _I32, P_I64, P_I32],
    "cook_state_job_facts": [_H, _I32, P_I64, P_U8, P_I32, P_F64, P_F64, P_I32],
    "cook_state_list_facts": [_H, _I32, P_I64, P_I64, P_I32, P_I32],
    "cook_state_list_jobs": [_P(_H), _I32, _I32, _I32, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _I32, P_I32, _I32,
                             _I32, _I32, P_I32, P_I64, P_I64, P_I32, P_I32, P_I32, _P(PhaseStats)],
    "cook_state_completed_seed": [_H, C.c_int64, _I32, P_I64, P_I64, P_I32, P_I64, P_I32, P_I32, P_U8],
    "cook_state_completed_record": [_H, _I32, P_I64, P_I64, P_I32, P_I64, P_I32, P_I32, P_U8],
    "cook_state_completed_advance": [_H, C.c_int64],
    "cook_state_list_completed": [_P(_H), _I32, _I32, _I32, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _I32, P_I32,
                                  _I32, _I32, _I32, P_I64, P_I64, P_I32, P_I32, _P(PhaseStats)],
    "cook_state_match_metrics": [_H, _I32, _I32, P_I32, _I32, _I32, P_I64, P_F64, P_I64, P_F64, P_I64, P_I32, P_I32,
                                 P_I32, P_I32, P_I32, P_F64, _P(PhaseStats)],
    "cook_state_finish": [_H, _I32, P_I64, P_I64, P_U8],
    "cook_state_finish_history": [_H, _I32, P_I64, P_I64, P_U8, P_I32],
    "cook_state_retry_config": [_H, _I32, _I32, P_I32, P_U8, P_I32],
    "cook_state_retry_facts": [_H, _I32, P_I64, P_I32, P_U8, P_I32, P_I32],
    "cook_state_status": [_H, _I32, P_I64, P_U8, P_I64, P_I32, P_U8, P_I32, P_I32],
    "cook_state_history_seed": [_H, C.c_int64, _I32, P_I64, P_I32, P_I64, P_I64, P_F64, P_F64, P_U8, P_I32],
    "cook_state_history_advance": [_H, C.c_int64],
    "cook_state_group_runtimes": [_H, _I32, P_I32, P_I32, _I32, P_I32],
    "cook_state_sweep": [_P(_H), _I32, C.c_int64, C.c_int64, C.c_int64, _I32, P_I32, P_F64, P_F64, P_I32, _I32, P_I64,
                         P_I32, P_I32, P_I64, P_I32, P_I32, _I32, P_I32, P_I64, P_I32, P_I32, _P(PhaseStats)],
    "cook_state_unscheduled": [_H, _I32, P_I64, P_U8, P_F64, P_I32, P_I32, P_I64, P_U8, _P(PhaseStats)],
    "cook_state_user_usage": [_P(_H), _I32, P_I32, _I32, _I32, _I32, _I32, P_I32, P_I32, P_I32, P_I64, P_F64, P_F64,
                              P_F64, P_I32, _I32, P_I64, P_I32, P_I32, _P(PhaseStats)],
    "cook_state_instance_stats": [_P(_H), _I32, C.c_int64, _I32, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _I32,
                                  P_I32, P_I32, P_I32, P_I64, P_F64, P_F64, P_I32, P_F64, P_I32, P_I32, _P(PhaseStats)],
    "cook_state_history_stats": [_P(_H), _I32, _I32, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _I32, P_I32, P_I32,
                                 P_I32, P_I64, P_F64, P_F64, P_I32, P_F64, P_I32, P_I32, _P(PhaseStats)],
    "cook_last_stats": [_H, _I32, _P(PhaseStats)],
    "cook_allgather_usage": [_H, _H, P_F64, P_F64, C.c_int64],
    "cook_comm_unique_id": [P_U8],
    "cook_comm_init": [P_U8, _I32, _I32, _I32, _P(_H)],
    "cook_comm_destroy": [_H],
    "cook_exchange_usage": [_H, _H, _I32, _I32, P_F64],
    "cook_exchange_usage_batch": [_P(_H), _I32, _H, _I32, _I32, _I32, P_F64],
}


# ------------------------------------------------------------------ builders
def make_tasks(user, priority, start_time, task_id, job_id, cpus, mem, gpus=None):
    n = len(user)
    if gpus is None:
        gpus = np.zeros(n)
    return TasksSoA(n=n, user=user, priority=priority, start_time=start_time,
                    task_id=task_id, job_id=job_id, cpus=cpus, mem=mem, gpus=gpus)


def make_users(n_users, name_rank=None, div_mem=None, div_cpus=None, div_gpus=None,
               quota=None, usage=None, tokens=None):
    """quota/usage: dict with count/cpus/mem/gpus arrays (or scalars)."""
    big = np.finfo(np.float64).max

    def full(x, default):
        if x is None:
            return np.full(n_users, default, dtype=np.float64)
        return np.broadcast_to(np.asarray(x, dtype=np.float64), (n_users,)).copy()

    quota = quota or {}
    usage = usage or {}
    return UserTable(
        n_users=n_users,
        name_rank=np.arange(n_users, dtype=np.int32) if name_rank is None else name_rank,
        div_mem=full(div_mem, big), div_cpus=full(div_cpus, big), div_gpus=full(div_gpus, big),
        quota_count=full(quota.get("count"), big), quota_cpus=full(quota.get("cpus"), big),
        quota_mem=full(quota.get("mem"), big), quota_gpus=full(quota.get("gpus"), big),
        usage_count=full(usage.get("count"), 0.0), usage_cpus=full(usage.get("cpus"), 0.0),
        usage_mem=full(usage.get("mem"), 0.0), usage_gpus=full(usage.get("gpus"), 0.0),
        tokens=np.full(n_users, 2**31 - 1, dtype=np.int32) if tokens is None else tokens)


def make_pool_quota(q=None):
    if q is None:
        return PoolQuota(0, 0, 0, 0, 0)
    return PoolQuota(1, float(q.get("count", 0)), float(q.get("cpus", 0)),
                     float(q.get("mem", 0)), float(q.get("gpus", 0)))


def csr(lists, dtype=np.int32):
    """list of lists -> (offsets[n+1], flat)."""
    off = np.zeros(len(lists) + 1, dtype=np.int32)
    for i, l in enumerate(lists):
        off[i + 1] = off[i] + len(l)
    flat = np.array([x for l in lists for x in l], dtype=dtype)
    if flat.size == 0:
        flat = np.zeros(1, dtype=dtype)  # never dereferenced; keeps pointer non-NULL
    return off, flat
