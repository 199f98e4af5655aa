"""CPU: unscheduled_ref against the reference's known answers (tests/golden/unscheduled_golden.json), and
cycle.unscheduled_reasons / cycle.Investigations on them, with cook_state_unscheduled's answers taken from the
restatement."""
import json
import math
import os

import numpy as np
import pytest

import unscheduled_ref as U
from cook_b200 import abi, cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "unscheduled_golden.json")))


def mirror(sc):
    return {r["job_id"]: r for r in sc["pending"]}, {r["task_id"]: r for r in sc["running"]}


@pytest.mark.parametrize("k", range(3))
def test_how_job_would_exceed_resource_limits(k):
    c = GOLDEN["exceed"][k]
    assert U.how_job_would_exceed_resource_limits(c["limits"], c["running"], c["job"]) == c["want"]


def test_fenzo_failures_for_user():
    c = GOLDEN["fenzo"][0]
    assert U.fenzo_failures_for_user(c["summary"]) == c["want"]
    assert cycle.fenzo_failures_for_user(c["summary"]) == c["want"]


def test_message_table_key_spellings():
    """A constraint name the table lacks (the matcher's underscore spelling of attribute-equals) is shown as is."""
    s = {"constraints": {"attribute_equals_host_placement_group_constraint": 2,
                         "attribute-equals-host-placement-group-constraint": 1}}
    assert [r["reason"] for r in cycle.fenzo_failures_for_user(s)] == [
        "attribute_equals_host_placement_group_constraint", "Host had a different attribute than other jobs in the group."]


def reasons_kw(sc, check):
    return dict(sc["facts"], enforcing_rate_limit=check.get("enforcing_rate_limit", False),
                num_rate_limited=check.get("num_rate_limited", 0))


@pytest.mark.parametrize("k", range(4))
def test_reasons_restatement(k):
    sc = GOLDEN["reasons"]
    check = sc["checks"][k]
    pend, run = mirror(sc)
    job = dict(pend[sc["job"]], state=check.get("state", "waiting"))
    reps = sorted(U.representatives(run).values(), key=lambda r: r["task_id"])
    got = U.reasons(job, reps, reps, list(pend.values()), **reasons_kw(sc, check))
    assert got == check["want"]


@pytest.mark.parametrize("k", range(4))
def test_reasons_through_cycle(k):
    """The same answers from cycle.unscheduled_reasons fed the restated device answer; 'not waiting' asks for a
    running job, and the uncommitted job, never a row, is absent."""
    sc = GOLDEN["reasons"]
    check = sc["checks"][k]
    pend, run = mirror(sc)
    q = [1 if check.get("state") == "running" else sc["job"]]
    a = U.engine_answer(pend, run, q)
    assert cycle.unscheduled_reasons(a, 0, **reasons_kw(sc, check)) == check["want"]
    a = U.engine_answer(pend, run, [sc["uncommitted"]])
    assert a["status"][0] == abi.UNSCHED_ABSENT
    assert cycle.unscheduled_reasons(a, 0) == [["The job already completed.", {}]]


def test_two_instances_count_once():
    sc = GOLDEN["reasons"]
    pend, run = mirror(sc)
    st, usage, pos, ahead, _ = U.answer(pend, run, [sc["job"]])[0]
    assert (st, usage[0], pos, ahead) == (U.WAITING, 3.0, 2, [1, 2])


@pytest.mark.parametrize("k", range(3))
def test_check_queue_position(k):
    sc = GOLDEN["queue_position"]
    c = sc["cases"][k]
    pend, run = mirror(sc)
    reps = list(U.representatives(run).values())
    msg, data = U.check_queue_position(c["job"], reps, sc["pending"], cap=sc["cap"])
    assert msg == c["message"]
    assert data["jobs"][:len(c.get("jobs", [c.get("first")]))] == c.get("jobs", [c.get("first")])
    # without the cap: the position the resident rows give
    st, _, pos, ahead, _ = U.answer(pend, run, [c["job"]])[0]
    assert pos == c["position"] and ahead[0] == data["jobs"][0]


def test_edges_by_hand():
    sc = GOLDEN["edges"]
    pend, run = mirror(sc)
    got = U.answer(pend, run, sc["queries"])
    for j, (st, usage, pos, ahead, _) in zip(sc["queries"], got):
        w = sc["want"][str(j)]
        assert (st, pos, ahead) == (w["status"], w["position"], w["ahead"])
        if str(j) in sc["usage"]:
            assert list(usage) == sc["usage"][str(j)]


def test_limit_on_the_last_bit():
    """A limit equal to the fold is not exceeded; one ulp under it is, with the usage reported."""
    sc = GOLDEN["edges"]
    lim = sc["limits"]
    pend, run = mirror(sc)
    a = U.engine_answer(pend, run, [lim["job"]])
    assert lim["below"]["cpus"] == math.nextafter(lim["equal"]["cpus"], 0.0)
    assert cycle.exceeded(lim["equal"], a["usage"][0]) == {}
    assert cycle.exceeded(lim["below"], a["usage"][0]) == lim["want_below"]
    r = cycle.unscheduled_reasons(a, 0, quota=lim["equal"], share=lim["below"])
    assert r[0] == ["The job would cause you to exceed resource shares.", lim["want_below"]]


def test_plugin_and_host_facts():
    sc = GOLDEN["edges"]
    pend, run = mirror(sc)
    a = U.engine_answer(pend, run, [2000, 2003])
    r = cycle.unscheduled_reasons(a, 0, plugin="cook.plugins.Demo", plugin_message="later")
    assert r[0] == ["The launch filter plugin is blocking the job launch.",
                    {"plugin": "cook.plugins.Demo", "message": "later"}]
    assert r[1] == ["You have 1 other jobs ahead in the queue.", {"jobs": [2003]}]
    r = cycle.unscheduled_reasons(a, 1, job_of=lambda j: f"uuid-{j}")
    assert r == [["The job is now under investigation. Check back in a minute for more details!", {}]]


class FakeEngine:
    def __init__(self, counts):
        self.counts, self.asked = counts, []

    def match_failures(self, ks):
        self.asked.append(list(ks))
        return [{"counts": self.counts[k]} for k in ks]


def test_investigations():
    """A marked job left unplaced gets its summary and leaves the investigation; an empty summary (ports only) keeps
    it marked; placed and unmarked jobs are not asked about."""
    inv = cycle.Investigations()
    sc = GOLDEN["edges"]
    pend, run = mirror(sc)
    a = U.engine_answer(pend, run, [2001, 2002])
    assert cycle.unscheduled_reasons(a, 0, investigations=inv)[-1][0].startswith("The job is now under investigation")
    cycle.unscheduled_reasons(a, 1, investigations=inv)
    inv.investigate(7)
    assert inv.marked == {2001, 2002, 7}
    n = abi.FAILC_N
    counts = [[0] * n, [0] * n, [0] * n, [0] * n]
    counts[1][0] = 4   # cpus (summarize_failures: resources, then constraints)
    counts[1][2 + cycle.CONSTRAINT_NAMES.index("novel_host_constraint")] = 2
    eng = FakeEngine(counts)
    match = {"considerable": np.array([5, 2001, 2002, 7]), "assign": np.array([-1, -1, -1, 3])}
    inv.record(eng, match)
    assert eng.asked == [[1, 2]]
    assert inv.summary == {2001: {"resources": {"cpus": 4}, "constraints": {"novel_host_constraint": 2}}}
    assert inv.marked == {2002, 7}
    r = cycle.unscheduled_reasons(a, 0, investigations=inv)
    assert r[-1] == ["The job couldn't be placed on any available hosts.",
                     {"reasons": [{"reason": "Not enough cpus available.", "host_count": 4},
                                  {"reason": "Job already ran on this host.", "host_count": 2}]}]
    assert 2001 in inv.marked   # asking again marks it again, as check-fenzo-placement does
