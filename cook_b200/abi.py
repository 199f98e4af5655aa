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

USAGE_GIVEN, USAGE_DERIVED, USAGE_LAST_MATCH = 0, 1, 2


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


_STATE_MATCH = [C.c_void_p, C.POINTER(OffersSoA), C.POINTER(Groups), C.POINTER(UserTable), C.POINTER(PoolQuota),
                C.POINTER(MatchParams), P_I64, P_I32, P_I32, C.c_int32, P_U8, C.POINTER(MatchStats)]
_STATE_REBALANCE = [C.c_void_p, C.POINTER(HostTable), C.POINTER(Groups), C.POINTER(UserTable),
                    C.POINTER(RebalanceParams), C.POINTER(Decision), P_I64, P_I64, C.c_int32, C.POINTER(C.c_int32)]
# ctypes argument types of the entry points that declare them (engine.load_library sets them); the derived calls
# take exactly cook_state_match's and cook_state_rebalance's arguments
ARGTYPES = {
    "cook_state_match_derived": _STATE_MATCH,
    "cook_state_rebalance_derived": _STATE_REBALANCE,
    "cook_state_considerable": [C.c_void_p, C.POINTER(UserTable), C.POINTER(PoolQuota), C.POINTER(ConsiderableParams),
                                P_I64, P_I32],
    "cook_state_rank_offensive": [C.c_void_p, C.POINTER(UserTable), C.POINTER(PoolQuota), C.POINTER(PoolQuota), P_F64,
                                  C.POINTER(RankParams), P_I64, P_I32, P_I64, C.c_int32, P_I32],
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
