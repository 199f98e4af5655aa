"""The refusals the resident state calls share, pinned by return code and message.

Every single-handle cook_state_* call enters the same way: a NULL handle is a bare COOK_E_BADARG, and the call's own
checks then name the call in cook_last_error.  The calls that take job or task ids refuse an id given twice and an id
the handle does not hold.  None of these refusals changes the handle, so every case runs against one loaded pool: one
pending job (JOB) and one running task (TASK, of another job).
"""
import ctypes as C

import numpy as np
import pytest

from cook_b200 import abi
from cook_b200.engine import GpuEngine

JOB, TASK, TASK_JOB, UNKNOWN = 1, 10, 2, 99
BAD = abi.COOK_E_BADARG


def i64(*v):
    return abi.ptr(np.ascontiguousarray(v, np.int64), abi.P_I64)


def i32(*v):
    return abi.ptr(np.ascontiguousarray(v, np.int32), abi.P_I32)


def u8(*v):
    return abi.ptr(np.ascontiguousarray(v, np.uint8), abi.P_U8)


def f64(*v):
    return abi.ptr(np.ascontiguousarray(v, np.float64), abi.P_F64)


def _delta_pending(ids, n=None, running=None):
    k = len(ids)
    jobs = abi.JobsSoA(n=k if n is None else n, user=np.zeros(k, np.int32), cpus=np.ones(k), mem=np.ones(k))
    return abi.make_delta(pending=jobs, pending_priority=np.zeros(k, np.int32), pending_job_id=np.asarray(ids, np.int64),
                          running=running)


@pytest.fixture(scope="module")
def eng():
    e = GpuEngine()
    running = abi.make_tasks(np.zeros(1, np.int32), np.zeros(1, np.int32), np.full(1, 1000, np.int64),
                             np.full(1, TASK, np.int64), np.full(1, TASK_JOB, np.int64), np.ones(1), np.ones(1))
    e.state_apply(_delta_pending([JOB], running=running))
    yield e
    e.close()


# (call, its arguments after the handle, the expected message)
CASES = {
    "apply": [
        ("cook_state_apply", lambda: [None], "cook_state_apply: null argument"),
        ("cook_state_apply", lambda: [C.byref(_delta_pending([5], n=-1))], "cook_state_apply: bad sizes"),
        ("cook_state_apply", lambda: [C.byref(_delta_pending([5, 5]))], "cook_state_apply: job id twice in one batch"),
    ],
    "launch": [
        ("cook_state_launch", lambda: [-1, None, None, None, None], "cook_state_launch: n < 0"),
        ("cook_state_launch", lambda: [1, None, i64(20), i64(0), None],
         "cook_state_launch: null job_id, task_id or start_time"),
        ("cook_state_launch", lambda: [2, i64(JOB, JOB), i64(20, 21), i64(0, 0), None], "cook_state_launch: job id twice"),
        ("cook_state_launch", lambda: [1, i64(UNKNOWN), i64(20), i64(0), None], "cook_state_launch: unknown job id"),
    ],
    "patch": [
        ("cook_state_patch", lambda: [-1, None, None, None, None, 0], "cook_state_patch: n < 0"),
        ("cook_state_patch", lambda: [1, None, u8(1), None, None, 0], "cook_state_patch: null job_id"),
        ("cook_state_patch", lambda: [2, i64(JOB, JOB), u8(1, 1), None, None, 0], "cook_state_patch: job id twice"),
        ("cook_state_patch", lambda: [1, i64(UNKNOWN), u8(1), None, None, 0], "cook_state_patch: unknown job id"),
    ],
    "task_facts": [
        ("cook_state_task_facts", lambda: [-1, None, None, None, None], "cook_state_task_facts: n < 0"),
        ("cook_state_task_facts", lambda: [1, None, i64(5), None, None], "cook_state_task_facts: null task_id"),
        ("cook_state_task_facts", lambda: [2, i64(TASK, TASK), i64(5, 5), None, None],
         "cook_state_task_facts: task id twice"),
        ("cook_state_task_facts", lambda: [1, i64(UNKNOWN), i64(5), None, None], "cook_state_task_facts: unknown task id"),
    ],
    "task_reason": [
        ("cook_state_task_reason", lambda: [-1, None, None], "cook_state_task_reason: n < 0"),
        ("cook_state_task_reason", lambda: [1, i64(TASK), None], "cook_state_task_reason: null task_id or reason_code"),
        ("cook_state_task_reason", lambda: [2, i64(TASK, TASK), i32(0, 0)], "cook_state_task_reason: task id twice"),
        ("cook_state_task_reason", lambda: [1, i64(UNKNOWN), i32(0)], "cook_state_task_reason: unknown task id"),
    ],
    "finish": [
        ("cook_state_finish", lambda: [-1, None, None, None], "cook_state_finish: n < 0"),
        ("cook_state_finish", lambda: [1, None, None, None], "cook_state_finish: null task_id"),
        ("cook_state_finish", lambda: [2, i64(TASK, TASK), None, None], "cook_state_finish: task id twice"),
        ("cook_state_finish", lambda: [1, i64(UNKNOWN), None, None], "cook_state_finish: unknown task id"),
    ],
    "finish_history": [
        ("cook_state_finish_history", lambda: [-1, None, None, None, None], "cook_state_finish_history: n < 0"),
        ("cook_state_finish_history", lambda: [1, None, i64(2000), u8(0), None],
         "cook_state_finish_history: null task_id"),
        ("cook_state_finish_history", lambda: [2, i64(TASK, TASK), i64(2000, 2000), u8(0, 0), None],
         "cook_state_finish_history: task id twice"),
        ("cook_state_finish_history", lambda: [1, i64(UNKNOWN), i64(2000), u8(0), None],
         "cook_state_finish_history: unknown task id"),
    ],
    "status": [
        ("cook_state_status", lambda: [-1, None, None, None, None, None, None, None], "cook_state_status: n < 0"),
        ("cook_state_status", lambda: [1, i64(TASK), u8(0), i64(2000), None, None, None, i32(0)],
         "cook_state_status: null out_outcome or out_attempts"),
        ("cook_state_status", lambda: [2, i64(TASK, TASK), u8(0, 0), i64(2000, 2000), None, None, i32(0, 0), i32(0, 0)],
         "cook_state_status: task id twice"),
        ("cook_state_status", lambda: [1, i64(UNKNOWN), u8(0), i64(2000), None, None, i32(0), i32(0)],
         "cook_state_status: unknown task id"),
    ],
    "job_facts": [
        ("cook_state_job_facts", lambda: [-1, None, None, None, None, None, None], "cook_state_job_facts: n < 0"),
        ("cook_state_job_facts", lambda: [1, None, None, None, None, None, None], "cook_state_job_facts: null job_id"),
        ("cook_state_job_facts", lambda: [2, i64(JOB, JOB), None, None, None, None, None],
         "cook_state_job_facts: job id twice"),
        ("cook_state_job_facts", lambda: [1, i64(UNKNOWN), None, None, None, None, None],
         "cook_state_job_facts: unknown job id"),
    ],
    "list_facts": [
        ("cook_state_list_facts", lambda: [-1, None, None, None, None], "cook_state_list_facts: n < 0"),
        ("cook_state_list_facts", lambda: [1, None, None, None, None], "cook_state_list_facts: null job_id"),
        ("cook_state_list_facts", lambda: [2, i64(JOB, JOB), None, None, None], "cook_state_list_facts: job id twice"),
        ("cook_state_list_facts", lambda: [1, i64(UNKNOWN), None, None, None],
         "cook_state_list_facts: a job id neither live-pending nor live-running"),
    ],
    "retry_config": [
        ("cook_state_retry_config", lambda: [5, -1, None, None, None], "cook_state_retry_config: n_reasons < 0"),
        ("cook_state_retry_config", lambda: [5, 1, None, u8(0), i32(-2)], "cook_state_retry_config: null array"),
        ("cook_state_retry_config", lambda: [5, 2, i32(3, 3), u8(0, 0), i32(-2, -2)],
         "cook_state_retry_config: reason code twice"),
    ],
    "retry_facts": [
        ("cook_state_retry_facts", lambda: [-1, None, None, None, None, None], "cook_state_retry_facts: n < 0"),
        ("cook_state_retry_facts", lambda: [1, None, i32(1), u8(0), None, None],
         "cook_state_retry_facts: null job_id, max_retries or flags"),
        ("cook_state_retry_facts", lambda: [2, i64(JOB, JOB), i32(1, 1), u8(0, 0), None, None],
         "cook_state_retry_facts: job id twice"),
        ("cook_state_retry_facts", lambda: [1, i64(UNKNOWN), i32(1), u8(0), None, None],
         "cook_state_retry_facts: unknown job id"),
    ],
    "history_seed": [
        ("cook_state_history_seed", lambda: [0, -1] + [None] * 8, "cook_state_history_seed: n < 0"),
        ("cook_state_history_seed", lambda: [0, 1] + [None] * 8, "cook_state_history_seed: null argument"),
        ("cook_state_history_seed", lambda: [0, 2, i64(30, 30), i32(0, 0), i64(0, 0), i64(5, 5), f64(1, 1), f64(1, 1),
                                             u8(1, 1), i32(-1, -1)], "cook_state_history_seed: task id twice"),
    ],
    "history_advance": [
        ("cook_state_history_advance", lambda: [0], "cook_state_history_advance: history is off"),
    ],
    "group_runtimes": [
        ("cook_state_group_runtimes", lambda: [-1, None, None, 0, None], "cook_state_group_runtimes: a negative size"),
        ("cook_state_group_runtimes", lambda: [1, None, None, 0, None], "cook_state_group_runtimes: null argument"),
    ],
    "completed_seed": [
        ("cook_state_completed_seed", lambda: [0, -1] + [None] * 7, "cook_state_completed_seed: n < 0"),
        ("cook_state_completed_seed", lambda: [0, 1] + [None] * 7, "cook_state_completed_seed: null argument"),
        ("cook_state_completed_seed", lambda: [0, 2, i64(7, 7), i64(1, 1), i32(0, 0), i64(5, 5), i32(-1, -1),
                                               i32(0, 0), u8(1, 1)], "cook_state_completed_seed: job id twice"),
    ],
    "completed_record": [
        ("cook_state_completed_record", lambda: [0] + [None] * 7, "cook_state_completed_record: the log is off"),
    ],
    "completed_advance": [
        ("cook_state_completed_advance", lambda: [0], "cook_state_completed_advance: the log is off"),
    ],
    "offers_add": [
        ("cook_state_offers_add", lambda: [None, None, None, None, None, None, 0], "cook_state_offers_add: null argument"),
        ("cook_state_offers_add", lambda: [C.byref(abi.OffersSoA(n=-1)), None, None, None, None, None, 0],
         "cook_state_offers_add: bad sizes"),
    ],
    "usage": [],
}


def _last_error(e):
    buf = C.create_string_buffer(512)
    e.lib.cook_last_error(e.pool, buf, 512)
    return buf.value.decode()


@pytest.mark.gpu
@pytest.mark.parametrize("call", sorted(CASES))
def test_refusals(eng, call):
    name = "cook_state_" + call
    fn = getattr(eng.lib, name)
    # a NULL handle: a bare refusal, no handle to hold a message
    zeros = [0 if t in (C.c_int32, C.c_int64) else None for t in fn.argtypes[1:]]
    assert fn(None, *zeros) == BAD
    for fname, args, msg in CASES[call]:
        assert fname == name
        rc = fn(eng.pool, *args())
        assert (rc, _last_error(eng)) == (BAD, msg)
