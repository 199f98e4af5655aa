"""Writes tests/golden/user_usage_golden.json: the known answers of GET /usage.

"api": the reference's test-get-user-usage-no-usage and test-get-user-usage-with-some-usage
(scheduler/test/cook/test/rest/api.clj:2297-2417) transcribed step by step, with job ids for uuids and alice as user
code 0: the pools in the database, the default pool, the running jobs (pool None: none), the request and the response.

"edges": three handles (pools alpha, beta, gamma; gamma loaded without a gpus column) and hand-computed responses:
the cpus fold lies on its last bit off the grid (ascending task id differs from the reverse and from job-id order), job
100 has three running rows in alpha (the greatest task id represents it) and a fourth in beta (a second job: the same
id in two handles), job 102 is in groups [9, 7] (the list's first entry wins), bob runs nothing in alpha and gamma,
carol runs nothing at all.  Every sum below is written in the fold order.

Run from the repository root: python tests/golden/make_user_usage_golden.py
"""
import functools
import json
import os

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "user_usage_golden.json")


def u(cpus, mem, gpus, jobs):
    return {"cpus": cpus, "mem": mem, "gpus": gpus, "jobs": jobs}


Z = u(0.0, 0.0, 0.0, 0)
ZG = {"total_usage": Z, "grouped": [], "ungrouped": {"running_jobs": [], "usage": Z}}
J1 = dict(job_id=1, task_id=11, user=0, pool=None, cpus=12.0, mem=34.0, gpus=56.0)
J2 = dict(job_id=2, task_id=12, user=0, pool="baz", cpus=78.0, mem=910.0, gpus=1112.0)
J3 = dict(job_id=3, task_id=13, user=0, pool="bar", cpus=13.0, mem=14.0, gpus=15.0)
FBB = ["foo", "bar", "baz"]

API = [
    dict(pools=[], default_pool="default", jobs=[], request=dict(user=0), want={"total_usage": Z}),
    dict(pools=FBB, default_pool="default", jobs=[], request=dict(user=0),
         want={"total_usage": Z, "pools": {p: {"total_usage": Z} for p in FBB}}),
    dict(pools=[], default_pool="default", jobs=[J1], request=dict(user=0),
         want={"total_usage": u(12.0, 34.0, 56.0, 1)}),
    dict(pools=FBB, default_pool="bar", jobs=[J1], request=dict(user=0),
         want={"total_usage": u(12.0, 34.0, 56.0, 1),
               "pools": {"foo": {"total_usage": Z}, "bar": {"total_usage": u(12.0, 34.0, 56.0, 1)},
                         "baz": {"total_usage": Z}}}),
    dict(pools=FBB, default_pool="foo", jobs=[J1, J2], request=dict(user=0),
         want={"total_usage": u(12.0 + 78.0, 34.0 + 910.0, 56.0 + 1112.0, 2),
               "pools": {"foo": {"total_usage": u(12.0, 34.0, 56.0, 1)}, "bar": {"total_usage": Z},
                         "baz": {"total_usage": u(78.0, 910.0, 1112.0, 1)}}}),
    dict(pools=FBB, default_pool="baz", jobs=[J1, J2, J3], request=dict(user=0, pool="foo"), want={"total_usage": Z}),
    dict(pools=FBB, default_pool="baz", jobs=[J1, J2, J3], request=dict(user=0, pool="bar"),
         want={"total_usage": u(13.0, 14.0, 15.0, 1)}),
    dict(pools=FBB, default_pool="baz", jobs=[J1, J2, J3], request=dict(user=0, pool="baz"),
         want={"total_usage": u(12.0 + 78.0, 34.0 + 910.0, 56.0 + 1112.0, 2)}),
]


def run(t, job, user, cpus, mem, groups, gpus=0.0):
    r = dict(task_id=t, job_id=job, user=user, cpus=cpus, mem=mem, groups=groups)
    if gpus is not None:
        r["gpus"] = gpus
    return r


HANDLES = {
    "alpha": [run(1001, 100, 0, 4.0, 40.0, [8], 2.0), run(1002, 100, 0, 4.0, 40.0, [8], 2.0),
              run(1005, 100, 0, 0.3, 30.0, [7]), run(1003, 101, 0, 0.1, 10.0, [], 1.0)],
    "beta": [run(1004, 102, 0, 0.2, 20.0, [9, 7]), run(1006, 100, 0, 0.6, 60.0, []),
             run(2001, 200, 1, 2.0, 64.0, [7])],
    "gamma": [run(1007, 103, 0, 0.7, 70.0, [7], None)],   # loaded without a gpus column
}
GROUPS = {7: ["g-7", "seven"], 9: ["g-9", "nine"]}


def grp(g, jobs, usage):
    return {"group": {"uuid": GROUPS[g][0], "name": GROUPS[g][1], "running_jobs": jobs}, "usage": usage}


# alice's representatives in the fold order: 1003 (101, alpha), 1004 (102, beta), 1005 (100, alpha), 1006 (100, beta),
# 1007 (103, gamma)
ALICE = {
    "total_usage": u(0.1 + 0.2 + 0.3 + 0.6 + 0.7, 10.0 + 20.0 + 30.0 + 60.0 + 70.0, 1.0 + 0.0 + 0.0 + 0.0 + 0.0, 5),
    "grouped": [grp(7, [100, 103], u(0.3 + 0.7, 30.0 + 70.0, 0.0 + 0.0, 2)), grp(9, [102], u(0.2, 20.0, 0.0, 1))],
    "ungrouped": {"running_jobs": [101, 100], "usage": u(0.1 + 0.6, 10.0 + 60.0, 1.0 + 0.0, 2)},
    "pools": {
        "alpha": {"total_usage": u(0.1 + 0.3, 10.0 + 30.0, 1.0 + 0.0, 2), "grouped": [grp(7, [100], u(0.3, 30.0, 0.0, 1))],
                  "ungrouped": {"running_jobs": [101], "usage": u(0.1, 10.0, 1.0, 1)}},
        "beta": {"total_usage": u(0.2 + 0.6, 20.0 + 60.0, 0.0 + 0.0, 2), "grouped": [grp(9, [102], u(0.2, 20.0, 0.0, 1))],
                 "ungrouped": {"running_jobs": [100], "usage": u(0.6, 60.0, 0.0, 1)}},
        "gamma": {"total_usage": u(0.7, 70.0, 0.0, 1), "grouped": [grp(7, [103], u(0.7, 70.0, 0.0, 1))],
                  "ungrouped": {"running_jobs": [], "usage": Z}}}}
BOB = {"total_usage": u(2.0, 64.0, 0.0, 1), "grouped": [grp(7, [200], u(2.0, 64.0, 0.0, 1))],
       "ungrouped": {"running_jobs": [], "usage": Z},
       "pools": {"alpha": ZG, "beta": {"total_usage": u(2.0, 64.0, 0.0, 1), "grouped": [grp(7, [200], u(2.0, 64.0, 0.0, 1))],
                                       "ungrouped": {"running_jobs": [], "usage": Z}}, "gamma": ZG}}
CAROL = dict(ZG, pools={p: ZG for p in HANDLES})

EDGES = dict(
    handles=HANDLES, groups=GROUPS,
    cases=[
        dict(request=dict(user=0, group_breakdown=True), want=ALICE),
        dict(request=dict(user=1, group_breakdown=True), want=BOB),
        dict(request=dict(user=2, group_breakdown=True), want=CAROL),
        dict(request=dict(user=0), want={"total_usage": ALICE["total_usage"],
                                         "pools": {p: {"total_usage": v["total_usage"]} for p, v in ALICE["pools"].items()}}),
        dict(request=dict(pool="beta"), want={"users": {0: {"total_usage": ALICE["pools"]["beta"]["total_usage"]},
                                                        1: {"total_usage": BOB["pools"]["beta"]["total_usage"]}}}),
    ])


def main():
    cpus = [0.1, 0.2, 0.3, 0.6, 0.7]   # alice's cpus in ascending task id
    fold = lambda xs: functools.reduce(lambda a, b: a + b, xs, 0.0)   # not sum(): it compensates
    assert fold(cpus) != fold(cpus[::-1]) and fold(cpus) != fold([0.3, 0.6, 0.1, 0.2, 0.7])   # job-id order
    assert ALICE["total_usage"]["cpus"] == fold(cpus) == 1.9000000000000001
    json.dump({"api": API, "edges": EDGES}, open(OUT, "w"), indent=1, sort_keys=False)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
