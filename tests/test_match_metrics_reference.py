"""match_metrics_ref and cycle.match_cycle_metrics_response (CPU): the reference's test-job->resource-maps cases and
the hand-computed rounds of tests/golden/match_metrics_golden.json, jobs->resource-maps' keys, resource-maps->stats'
percentiles, last maximal rows and totals, the uris error, the log maps and the warning decision, and the unmatched
counts against PoolCycle.unmatched_cycles over the same rounds.
"""
import json
import os
from fractions import Fraction

import numpy as np

import match_metrics_ref as MR
from cook_b200 import cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                   "match_metrics_golden.json")))


def job(jid, cpus, mem, user=0, **kw):
    row = dict(job_id=jid, user=user, cpus=cpus, mem=mem, gpus=0.0, ports=0, facts=0, gpu_model=-1, disk_type=-1,
               disk_request=0.0, disk_limit=0.0)
    row.update(kw)
    return row


def test_resource_maps_keys():
    # a gpus resource of 0.0 is a key (`(if gpus ...)` is true for 0.0); no gpus resource is none
    assert MR.resource_map(job(1, 1.0, 10.0, facts=MR.JF_GPUS, gpus=0.0, gpu_model=-1)) == \
        {"cpus": 1.0, "mem": 10.0, (MR.MM_GPUS, -1): 0.0}
    assert MR.resource_map(job(1, 1.0, 10.0, gpus=2.0)) == {"cpus": 1.0, "mem": 10.0}
    # disk without a request, and without a limit
    assert MR.resource_map(job(1, 1.0, 10.0, facts=MR.JF_DISK | MR.JF_DISK_LIMIT, disk_type=3, disk_limit=5.0)) == \
        {"cpus": 1.0, "mem": 10.0, (MR.MM_DISK_LIMIT, 3): 5.0}
    assert MR.resource_map(job(1, 1.0, 10.0, facts=MR.JF_DISK | MR.JF_DISK_REQUEST, disk_type=-1,
                               disk_request=7.0)) == {"cpus": 1.0, "mem": 10.0, (MR.MM_DISK_REQUEST, -1): 7.0}


def test_uris_error():
    one = [job(1, 1.0, 1.0, facts=MR.JF_URIS), job(2, 2.0, 2.0)]
    two = [job(1, 1.0, 1.0, facts=MR.JF_URIS), job(2, 2.0, 2.0, facts=MR.JF_URIS)]
    assert MR.stats(one) != MR.ERROR and MR.stats(two) == MR.ERROR
    assert MR.answer(one, set(), {}, 500, 1)["uris_position"] == 0
    assert MR.answer(two, set(), {}, 500, 1)["uris_position"] == -1
    assert MR.answer([job(1, 1.0, 1.0)], set(), {}, 500, 1)["uris"] == 0


def test_ties_percentiles_and_fold_order():
    jobs = [job(1, 4.0, 1.0), job(2, 1.0, 9.0), job(3, 4.0, 9.0), job(4, 2.0, 3.0)]
    s = MR.stats(jobs)
    assert s["largest-by"] == {"cpus": 2, "mem": 2}   # the last maximal row in take order
    assert s["percentiles"]["cpus"] == {50: 2.0, 95: 4.0, 100: 4.0}
    a = MR.answer(jobs, {0}, {}, 500, 1)
    assert (a["largest_cpus"], a["largest_mem"]) == (2, 2)
    # a fold off the grid whose last bit depends on the order: the answer folds in take order
    xs = [0.1, 0.2, 0.3]
    left = (0.1 + 0.2) + 0.3
    assert left != 0.1 + (0.2 + 0.3)
    assert MR.answer([job(k, x, 1.0) for k, x in enumerate(xs)], set(), {}, 500, 1)["total_cpus"] == left


def test_counts_match_pool_cycle():
    """The restated counts equal PoolCycle.unmatched_cycles over the same rounds: a job leaving the considerable set
    and returning starts again at 1, and the threshold is strict (500 is not too long, 501 is)."""
    rng = np.random.default_rng(3)
    pc = cycle.PoolCycle(engine=None)
    prev = {}
    for r in range(40):
        considerable = [int(j) for j in rng.choice(30, size=20, replace=False)]
        matched = {j for j in considerable if rng.random() < 0.3}
        pc._finish(np.zeros(0, np.int32), [{"jobs": list(matched)}] if matched else [], matched, set(), True,
                   len(considerable), 20, considerable=considerable)
        prev = MR.unmatched_cycles(prev, considerable, matched)
        assert prev == pc.unmatched_cycles
    prev = {7: 499}
    jobs = [job(7, 1.0, 1.0)]
    a = MR.answer(jobs, set(), prev, 500, 1)
    assert a["cycles"] == {7: 500} and a["too_long"] == 0
    a = MR.answer(jobs, set(), a["cycles"], 500, 1)
    assert a["cycles"] == {7: 501} and a["too_long"] == 1 and a["first"] == [(7, 501)]
    assert MR.answer(jobs, {0}, a["cycles"], 500, 1)["cycles"] == {}


def test_empty_round_and_drops():
    a = MR.answer([], set(), {5: 3}, 500, 2)
    assert a["considerable"] == 0 and a["cycles"] == {} and a["head_job_id"] == -1
    jobs = [job(1, 1.0, 1.0, user=1), job(2, 1.0, 1.0)]
    a = MR.answer(jobs, {1}, {}, 500, 2)        # the head's match was dropped
    assert a["head_matched"] == 0 and a["user_considerable"] == [1, 1] and a["user_matched"] == [1, 0]
    assert a["cycles"] == {1: 1}


def _names(d):
    return {c: n for n, c in d.items()}


def test_golden_resource_maps():
    """The reference's own expected maps, through the restatement's coded keys and their names."""
    for case in GOLDEN["resource_maps"]:
        gc, dc = {}, {}
        rows = [MR.named_job(j, gc, dc) for j in case["jobs"]]
        got = [MR.named_resource_map(r, _names(gc), _names(dc)) for r in rows]
        assert got == case["want"], case["name"]


def engine_answer(a, jobs):
    """A restated answer in engine.state_match_metrics' shape."""
    out = dict(a, keys_n=len(a["keys"]), first_n=len(a["first"]), user_considerable=np.array(a["user_considerable"]),
               user_matched=np.array(a["user_matched"]))
    if a["considerable"]:
        out["rows"] = [dict(jobs[k], position=k) for k in (0, a["largest_cpus"], a["largest_mem"])]
    else:
        out["rows"] = []
    return out


def replay(case, threshold, n_users):
    """Each round of a golden case: (round, jobs, restated answer)."""
    prev = {}
    for r in MR.golden_rounds(case):
        jobs = r["jobs"]
        a = MR.answer(jobs, set(r["assigned"]) - set(r["dropped"]), prev, threshold, n_users)
        prev = a["cycles"]
        yield r, jobs, a


def check_want(a, want, jobs):
    for k, v in want.items():
        if k == "cycles":
            assert a["cycles"] == {int(j): c for j, c in v.items()}
        elif k == "keys":
            assert [list(x) for x in a["keys"]] == v
        elif k == "stats_error":
            assert (MR.stats(jobs) == MR.ERROR) == v
        elif k == "first":
            assert [list(x) for x in a["first"]] == v
        else:
            assert a[k] == v, k


def test_golden_rounds():
    for name, case in GOLDEN["rounds"].items():
        n = 0
        for r, jobs, a in replay(case, GOLDEN["threshold"], GOLDEN["n_users"]):
            if r.get("repeat"):
                continue
            check_want(a, r["want"], jobs)
            n += 1
        assert n, name


def _response(a, jobs, **kw):
    return cycle.match_cycle_metrics_response(engine_answer(a, jobs), [j["job_id"] for j in jobs], pool="p",
                                              n_offers=5, n_offers_scheduled=2, **kw)


def test_response_shapes():
    gc, dc = {}, {}
    jobs = [dict(MR.named_job(j, gc, dc), job_id=k + 1, ports=k) for k, j in
            enumerate(GOLDEN["resource_maps"][0]["jobs"])]
    gn, dn = _names(gc), _names(dc)
    a = MR.answer(jobs, {1}, {}, 500, 1)
    r = _response(a, jobs, max_considerable=2, gpu_model_name=gn.get, disk_type_name=dn.get, user_name=lambda u: "u")
    t = r["total"]
    assert r["users"] == [{"user": "u", "pool": "p", "user-considerable": 2, "user-matched": 1, "user-unmatched": 1}]
    assert t["inputs"] == {"jobs-considerable": 2, "offers": 5, "max-considerable": 2, "queue-was-full": True}
    assert t["matched"]["match-percent"] == Fraction(1, 2) and t["matched"]["head-was-matched"] is False
    assert t["unmatched"] == {"jobs-considerable": 1, "offers": 3}
    js = t["stats"]["jobs-considerable"]
    want = GOLDEN["resource_maps"][0]["want"]
    assert js["largest-by"] == {"cpus": want[1], "mem": want[1]}
    assert js["totals"] == {"cpus": 1.2 + 2.3, "mem": 79, "gpus/nvidia-tesla-k80": 2, "gpus/nvidia-tesla-p100": 4,
                            "disk/pd-ssd/request": 10, "disk/pd-ssd/limit": 20}
    assert js["percentiles"] == {"cpus": {50: 1.2, 95: 2.3, 100: 2.3}, "mem": {50: 34, 95: 45, 100: 45}}
    assert t["stats"]["head-resources"] == {"ports": 0, "cpus": 1.2, "mem": 34, "gpus": 2,
                                            "disk": {"request": 10, "limit": 20, "type": "pd-ssd"}}
    assert r["front"] == (1.2, 34) and r["warn"] is None
    # the slim zero-considerable form
    z = _response(MR.answer([], set(), {}, 500, 1), [], max_considerable=2)
    assert z == {"users": [], "warn": None, "front": (0, 0), "total": {"inputs": {"jobs-considerable": 0}, "pool": "p"}}
    # two rows with uris: the error string; one: the totals keep that row's uris
    two = [dict(j, facts=j["facts"] | MR.JF_URIS) for j in jobs]
    r2 = _response(MR.answer(two, set(), {}, 500, 1), two, max_considerable=10, gpu_model_name=gn.get,
                   disk_type_name=dn.get)
    assert r2["total"]["stats"]["jobs-considerable"] == MR.ERROR
    assert r2["total"]["inputs"]["queue-was-full"] is False
    one = [jobs[0], dict(jobs[1], facts=jobs[1]["facts"] | MR.JF_URIS)]
    r1 = _response(MR.answer(one, set(), {}, 500, 1), one, max_considerable=2, gpu_model_name=gn.get,
                   disk_type_name=dn.get, uris=lambda j: ["u%d" % j])
    assert r1["total"]["stats"]["jobs-considerable"]["totals"]["uris"] == str(["u2"])


def test_response_warning():
    """The fraction test: more than half the considerable jobs past the cycle threshold warns."""
    jobs = [job(k, 1.0, 1.0) for k in range(4)]
    prev = {0: 500, 1: 500, 2: 500}
    a = MR.answer(jobs, set(), prev, 500, 1)
    r = _response(a, jobs, max_considerable=4, job_name=lambda j: "job-%d" % j)
    assert r["warn"]["number-unmatched-too-long"] == 3 and r["warn"]["number-considerable"] == 4
    assert r["warn"]["first-ten-unmatched-too-long"] == [("job-0", 501), ("job-1", 501), ("job-2", 501)]
    a = MR.answer(jobs, set(), {0: 500, 1: 500}, 500, 1)   # exactly one half is not more than 0.5
    assert _response(a, jobs, max_considerable=4)["warn"] is None
