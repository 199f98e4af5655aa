"""Writes tests/golden/unscheduled_golden.json: the known answers of the reference's unscheduled tests
(scheduler/test/cook/test/unscheduled.clj), transcribed with job ids for uuids, and hand-computed edges.

  exceed          test-how-job-would-exceed-resource-limits: three limit maps, running jobs, a job, the answer
  fenzo           test-fenzo-placement: a placement-failure summary and fenzo-failures-for-user's answer
  reasons         test-reasons: two running jobs of two instances each (instances 11-14), an uncommitted job that
                  never becomes a row (3), a waiting job (4) with two failed instances; the four checks
  queue_position  test-check-queue-position: 500 waiting jobs (1-500), 50 running jobs (501-550) of one running
                  instance each; three queries, the reference's waiting cap of 100, and the position without it
  edges           rows and queries whose answers are computed by hand here (asserted below): usage on the last bit of
                  an off-grid fold (a limit equal to it, one one ulp under it), priority ties broken by job id, 10 and
                  11 entries ahead, a running job of three rows, a job with a pending row and a running row, a
                  deferred plugin, an absent and a repeated id

Run from the repository root: python tests/golden/make_unscheduled_golden.py
"""
import json
import math
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import unscheduled_ref as U   # noqa: E402

S = 1_700_000_000_000


def run_row(tid, jid, user, start, cpus, mem, gpus=0.0, priority=50):
    return dict(task_id=tid, job_id=jid, user=user, start_time=start, cpus=cpus, mem=mem, gpus=gpus, priority=priority)


def pend_row(jid, user, cpus, mem, gpus=0.0, priority=50, plugin_accept=1):
    return dict(job_id=jid, user=user, cpus=cpus, mem=mem, gpus=gpus, priority=priority, plugin_accept=plugin_accept)


def exceed():
    quota = {"mem": 6000, "cpus": 8, "count": 5}
    running = [{"mem": 3000, "cpus": 4}, {"mem": 2000, "cpus": 2}]
    return [dict(limits=quota, running=running, job={"mem": 4000, "cpus": 4},
                 want={"mem": {"limit": 6000, "usage": 9000}, "cpus": {"limit": 8, "usage": 10}}),
            dict(limits=quota, running=running, job={"mem": 2000, "cpus": 1},
                 want={"mem": {"limit": 6000, "usage": 7000}}),
            dict(limits=dict(quota, count=2), running=running, job={"mem": 500, "cpus": 4},
                 want={"cpus": {"limit": 8, "usage": 10}, "count": {"limit": 2, "usage": 3}})]


def fenzo():
    summary = {"constraints": {"novel_host_constraint": 3}, "resources": {"mem": 14, "cpus": 8}}
    return [dict(summary=summary, want=[{"reason": "Not enough mem available.", "host_count": 14},
                                        {"reason": "Not enough cpus available.", "host_count": 8},
                                        {"reason": "Job already ran on this host.", "host_count": 3}])]


def reasons():
    run = [run_row(11, 1, 0, S + 1, 1.0, 3.0), run_row(12, 1, 0, S + 2, 1.0, 3.0),
           run_row(13, 2, 0, S + 3, 1.0, 3.1), run_row(14, 2, 0, S + 4, 1.0, 3.1)]
    pend = [pend_row(4, 0, 1.0, 3.0)]
    facts = dict(quota={"count": 2}, attempts_consumed=2, max_retries=2)
    retries = ["Job has exhausted its maximum number of retries.", {"max-retries": 2, "instance-count": 2}]
    quota = ["The job would cause you to exceed resource quotas.", {"count": {"limit": 2, "usage": 3}}]
    ahead = ["You have 2 other jobs ahead in the queue.", {"jobs": [1, 2]}]
    inv = ["The job is now under investigation. Check back in a minute for more details!", {}]
    rate = ["You are currently rate limited on how many jobs you launch per minute.", {"num-ratelimited": 3}]
    return dict(running=run, pending=pend, job=4, uncommitted=3, facts=facts, checks=[
        dict(name="not waiting", state="running", want=[["The job is running now.", {}]]),
        dict(name="waiting", want=[retries, quota, ahead, inv]),
        dict(name="rate limit enforced", enforcing_rate_limit=True, num_rate_limited=3,
             want=[retries, quota, rate, ahead, inv]),
        dict(name="rate limit not enforced", want=[retries, quota, ahead, inv])])


def queue_position():
    pend = [pend_row(j, 0, 1.0, 3.0) for j in range(1, 501)]
    run = [run_row(1001 + k, 501 + k, 0, S + k, 1.0, 3.0) for k in range(50)]
    return dict(running=run, pending=pend, cap=100, cases=[
        dict(job=502, message="You have 1 other jobs ahead in the queue.", jobs=[501], position=1),
        dict(job=1, message="You have 50 other jobs ahead in the queue.", first=501, position=50),
        dict(job=500, message="You have at least 150 other jobs ahead in the queue.", first=501, position=549)])


def edges():
    a, b, c, x = 0.1, 0.2, 0.3, 0.7
    v = ((a + b) + c) + x   # ascending task id, then the job
    assert ((c + b) + a) + x != v and (a + (b + c)) + x != v, "the fold order must show in the last bit"
    run, pend = [], []
    # user 1: three running jobs off the grid, loaded in descending task id (slot order is not task order)
    run += [run_row(112, 1102, 1, S + 12, c, 7.0 / 3.0), run_row(111, 1101, 1, S + 11, b, 5.0 / 3.0),
            run_row(110, 1100, 1, S + 10, a, 1.0 / 3.0)]
    pend += [pend_row(1103, 1, x, 1.0 / 7.0)]
    # user 2: priority ties by job id, one higher priority, a deferred plugin
    pend += [pend_row(2001, 2, 1.0, 1.0), pend_row(2002, 2, 1.0, 1.0), pend_row(2003, 2, 1.0, 1.0, priority=90),
             pend_row(2000, 2, 1.0, 1.0, plugin_accept=0)]
    # user 3: 12 waiting jobs of one priority
    pend += [pend_row(3000 + k, 3, 0.5, 512.0) for k in (5, 11, 0, 7, 3, 10, 1, 9, 2, 8, 4, 6)]
    # user 4: a running job of three rows (the newest started last), another of one row, a waiting job
    run += [run_row(40, 4000, 4, S + 50, 1.0, 10.0), run_row(41, 4000, 4, S + 5, 1.0, 10.0),
            run_row(42, 4000, 4, S + 60, 1.0, 10.0, gpus=1.0), run_row(43, 4001, 4, S + 55, 2.0, 20.0)]
    pend += [pend_row(4002, 4, 1.0, 1.0)]
    # user 5: job 5000 pending and running at once
    run += [run_row(50, 5000, 5, S + 70, 3.0, 30.0)]
    pend += [pend_row(5000, 5, 1.0, 1.0)]
    queries = [1103, 2000, 2001, 2002, 2003, 3010, 3011, 3000, 4002, 4000, 4001, 5000, 99999, 2002, 4000]
    want = {   # job id -> (status, position, ahead), by hand
        1103: (U.WAITING, 3, [1100, 1101, 1102]), 2000: (U.WAITING, 1, [2003]), 2001: (U.WAITING, 2, [2003, 2000]),
        2002: (U.WAITING, 3, [2003, 2000, 2001]), 2003: (U.WAITING, 0, []),
        3010: (U.WAITING, 10, list(range(3000, 3010))), 3011: (U.WAITING, 11, list(range(3000, 3010))),
        3000: (U.WAITING, 0, []), 4002: (U.WAITING, 2, [4001, 4000]), 4000: (U.RUNNING, 1, [4001]),
        4001: (U.RUNNING, 0, []), 5000: (U.WAITING, 1, [5000]), 99999: (U.ABSENT, -1, [])}
    usage = {1103: [4.0, v, ((1.0 / 3.0 + 5.0 / 3.0) + 7.0 / 3.0) + 1.0 / 7.0, 0.0], 4002: [3.0, 4.0, 31.0, 1.0],
             5000: [2.0, 4.0, 31.0, 0.0], 2000: [1.0, 1.0, 1.0, 0.0]}
    got = dict(zip(queries, U.answer({r["job_id"]: r for r in pend}, {r["task_id"]: r for r in run}, queries)))
    for j, (st, pos, ahead) in want.items():
        assert got[j][0] == st and got[j][2] == pos and got[j][3] == ahead, (j, got[j])
    for j, u in usage.items():
        assert list(got[j][1]) == u, (j, got[j][1], u)
    assert got[2000][4] == 1 and got[2001][4] == 0
    below = math.nextafter(v, 0.0)
    return dict(running=run, pending=pend, queries=queries,
                want={str(j): dict(status=s, position=p, ahead=a) for j, (s, p, a) in want.items()},
                usage={str(j): u for j, u in usage.items()},
                limits=dict(user=1, job=1103, equal={"cpus": v}, below={"cpus": below},
                            want_below={"cpus": {"limit": below, "usage": v}}))


def main():
    out = dict(exceed=exceed(), fenzo=fenzo(), reasons=reasons(), queue_position=queue_position(), edges=edges())
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "unscheduled_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
