"""Writes retry_golden.json: the reference's known answers on retries, transcribed as data, and hand-computed edges.

Transcribed (scheduler/test/cook/test/schema.clj, test/cook/test/tools.clj):
- reasons_attempts_consumed: test-reasons->attempts-consumed (schema.clj:195-216), all six limits.
- transitions: test-instance-update-state-with-job-state (:217-339) and test-mea-culpa-retry-on-mesos-executor-
  terminated (:109-194), each a verify-job-state-transition: the job's instances (status, reason), the updates of one
  transaction (new status or null, reason), the job's retry count and mea-culpa flag, the old and new job state.
  verify-job-state-transition's defaults: reasons :unknown, retry count 5, mea-culpa retries on.
- attempts_consumed: test-attempts-consumed (tools.clj:194-267).
The reasons are those of the schema (schema.clj:1424-1660); the test database has no :scheduler/config, so the global
mea-culpa limit is 5.

Hand-computed edges: a failure limit of exactly 0 and of -1, a nil-reason success, the novel-host list after a
preempted failure on a listed host and after a host of -1, and two instances of one job failing in one batch, in both
orders, decided one status at a time.

Run from the repository root: python tests/golden/make_retry_golden.py
"""
import json
import os

REASONS = {"unknown": {"code": 99000, "mea_culpa": False, "failure_limit": None},
           "preempted-by-rebalancer": {"code": 1002, "mea_culpa": True, "failure_limit": None},
           "mesos-executor-terminated": {"code": 99002, "mea_culpa": True, "failure_limit": 3}}

# test-reasons->attempts-consumed: A-C code 100 mea culpa, D-E 101, F nil, G 102, H-I 103 limit 1, J-K 104 limit -1
R100 = {"code": 100, "mea_culpa": True, "failure_limit": None}
R101 = {"code": 101, "mea_culpa": False, "failure_limit": None}
R102 = {"code": 102, "mea_culpa": False, "failure_limit": None}
R103 = {"code": 103, "mea_culpa": True, "failure_limit": 1}
R104 = {"code": 104, "mea_culpa": True, "failure_limit": -1}
RAC_REASONS = [R100, R100, R100, R101, R101, None, R102, R103, R103, R104, R104]
RAC = [dict(limit=0, disable=True, attempts=11), dict(limit=0, disable=False, attempts=8),
       dict(limit=1, disable=False, attempts=7), dict(limit=2, disable=False, attempts=6),
       dict(limit=3, disable=False, attempts=5), dict(limit=5, disable=False, attempts=5)]
# hand-computed: a failure limit of exactly 0 (every such failure counts), and of -1 (none does)
R0 = {"code": 105, "mea_culpa": True, "failure_limit": 0}
RAC_EDGES = [dict(reasons=[R0, R0, None], limit=5, disable=False, attempts=3),
             dict(reasons=[R104, R104, R104, R101], limit=0, disable=False, attempts=1),
             dict(reasons=[R100] * 7, limit=-1, disable=False, attempts=0),
             dict(reasons=[R100] * 7, limit=-1, disable=True, attempts=7)]

U, R, S, F = "unknown", "running", "success", "failed"


def vt(name, old, new, old_job, new_job, retry=5, old_reasons=None, new_reasons=None, disable=False):
    n = len(old)
    return dict(name=name, instances=[[s, r] for s, r in zip(old, old_reasons or ["unknown"] * n)],
                updates=[[s, r] for s, r in zip(new, new_reasons or ["unknown"] * n)], retry_count=retry,
                disable=disable, old_job_state=old_job, new_job_state=new_job)


MET = "mesos-executor-terminated"
PBR = "preempted-by-rebalancer"
T = []
for a, b, c in ((U, U, "running"), (U, R, "running"), (U, S, "completed"), (U, F, "waiting")):
    T.append(vt(f"unknown->{b}", [a], [b], "running", c))
for b, c in ((S, "completed"), (F, "waiting"), (R, "running"), (U, "running")):
    T.append(vt(f"running->{b}", [R], [b], "running", c))
for b in (S, F, R, U):
    T.append(vt(f"success->{b}", [S], [b], "completed", "completed"))
for b in (S, F, R, U):
    T.append(vt(f"failed->{b}", [F], [b], "waiting", "waiting"))
for other in (R, U):
    for b, c in ((S, "completed"), (F, "waiting"), (U, "running"), (R, "running")):
        T.append(vt(f"failed+{other}->{b}", [F, other], [None, b], "running", c))
T.append(vt("two running fail in one transaction", [R, R], [F, F], "running", "running"))
T.append(vt("two running fail in one transaction, retries 2", [R, R], [F, F], "running", "running", retry=2))
T.append(vt("out of retries, no mea-culpas", [F, F, R], [None, None, F], "running", "completed", 3,
            ["unknown"] * 3, [None, None, "unknown"]))
T.append(vt("out of retries, some mea-culpas", [F, F, F, R], [None, None, None, F], "running", "completed", 3,
            [PBR, "unknown", "unknown", "unknown"], [None, None, None, "unknown"]))
T.append(vt("retries left thanks to mea-culpas", [F, F, R], [None, None, F], "running", "waiting", 3,
            [PBR, PBR, "unknown"], [None, None, "unknown"]))
T.append(vt("retries left, no mea-culpas", [F, F, R], [None, None, F], "running", "waiting", 4,
            ["unknown"] * 3, [None, None, "unknown"]))
T.append(vt("retries left thanks to mea-culpas, edge", [F, F, R], [None, None, F], "running", "waiting", 2,
            [PBR, PBR, "unknown"], [None, None, "unknown"]))
T.append(vt("do or do not", [F, F, R], [None, None, F], "running", "completed", 1,
            [PBR, PBR, "unknown"], [None, None, "unknown"]))
T.append(vt("no mea-culpa retries when disabled", [R], [F], "running", "completed", 1, ["unknown"], [PBR],
            disable=True))
# test-mea-culpa-retry-on-mesos-executor-terminated
T.append(vt("executor terminated, disabled, retry 1", [R], [F], "running", "completed", 1, [MET], [MET], True))
T.append(vt("rebalancer, retry 2", [R], [F], "running", "waiting", 2, [PBR], [PBR]))
T.append(vt("executor terminated, disabled, retry 2", [R], [F], "running", "waiting", 2, [MET], [MET], True))
T.append(vt("executor terminated twice, disabled, retry 2", [F, R], [None, F], "running", "completed", 2,
            [MET, None], [MET, PBR], True))
for n in range(1, 4):
    T.append(vt(f"executor terminated x{n}, retry 1", [F] * (n - 1) + [R], [None] * (n - 1) + [F], "running", "waiting",
                1, [MET] * n, [MET] * n))
T.append(vt("executor terminated x4, retry 1", [F, F, F, R], [None, None, None, F], "running", "completed", 1,
            [MET] * 4, [MET] * 4))
for n in range(1, 5):
    T.append(vt(f"executor terminated x{n}, retry 2", [F] * (n - 1) + [R], [None] * (n - 1) + [F], "running",
                "waiting", 2, [MET] * n, [MET] * n))
T.append(vt("executor terminated x5, retry 2", [F] * 4 + [R], [None] * 4 + [F], "running", "completed", 2,
            [MET] * 5, [MET] * 5))

# test-attempts-consumed: (status, reason) per instance; a reason null is an instance without one
AC = [dict(name="no mea-culpa reasons", instances=[[F, "unknown"], [F, "unknown"], [R, None]], attempts=2),
      dict(name="some mea-culpa reasons", instances=[[F, "unknown"], [F, PBR], [F, PBR], [R, None]], attempts=1),
      dict(name="all mea-culpa reasons", instances=[[F, PBR], [F, PBR], [R, None]], attempts=0),
      dict(name="some nil reasons", instances=[[F, "unknown"], [F, None], [F, PBR], [R, None]], attempts=2),
      dict(name="finished running job", instances=[[S, None], [F, None], [F, PBR], [R, None]], attempts=2),
      dict(name="finished job", instances=[[S, None], [F, None], [F, PBR]], attempts=2),
      # hand-computed: a nil-reason success counts as one attempt
      dict(name="nil-reason success", instances=[[S, None]], attempts=1)]

# hand-computed novel-host lists after a requeue: (list, failed host, preempted) -> list
NOVEL = [dict(novel=[3, 7], host=5, preempted=False, after=[3, 7, 5]),
         dict(novel=[3, 7], host=7, preempted=False, after=[3, 7]),
         dict(novel=[3, 7], host=7, preempted=True, after=[3, 7]),
         dict(novel=[3, 7], host=5, preempted=True, after=[3, 7]),
         dict(novel=[3], host=-1, preempted=False, after=[3]),
         dict(novel=[], host=0, preempted=False, after=[0])]

# hand-computed: two running instances of one job fail in one batch, one status at a time, in both orders; the
# first sees the other live (running), the second decides.  Retry count 2, reasons unknown then rebalancer.
BATCH = [dict(name="unknown first", instances=[[R, "unknown"], [R, "unknown"]], order=[[0, F, "unknown"], [1, F, PBR]],
              retry_count=2, outcomes=["running", "waiting"], attempts=[1, 1], new_job_state="waiting"),
         dict(name="rebalancer first", instances=[[R, "unknown"], [R, "unknown"]], order=[[1, F, PBR], [0, F, "unknown"]],
              retry_count=2, outcomes=["running", "waiting"], attempts=[0, 1], new_job_state="waiting"),
         dict(name="both plain, retry 2", instances=[[R, "unknown"], [R, "unknown"]],
              order=[[0, F, "unknown"], [1, F, "unknown"]], retry_count=2, outcomes=["running", "completed"],
              attempts=[1, 2], new_job_state="completed"),
         dict(name="both plain, retry 2, other order", instances=[[R, "unknown"], [R, "unknown"]],
              order=[[1, F, "unknown"], [0, F, "unknown"]], retry_count=2, outcomes=["running", "completed"],
              attempts=[1, 2], new_job_state="completed")]

OUT = dict(mea_culpa_limit=5, reasons=REASONS, reasons_attempts_consumed=dict(reasons=RAC_REASONS, cases=RAC),
           reasons_attempts_edges=RAC_EDGES, transitions=T, attempts_consumed=AC, novel=NOVEL, batch=BATCH)

if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "retry_golden.json")
    with open(path, "w") as f:
        json.dump(OUT, f, indent=1)
        f.write("\n")
    print("wrote", path)
