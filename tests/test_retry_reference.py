"""The plain-Python restatement of Cook's retry decision (retry_ref) against the reference's known answers and the
hand-computed edges of golden/retry_golden.json (CPU only)."""
import json
import os

import pytest

import retry_ref as RR
from cook_b200 import cycle

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "retry_golden.json")))
REASONS = GOLDEN["reasons"]


def _reason(name):
    return None if name is None else REASONS[name]


def test_reasons_attempts_consumed():
    g = GOLDEN["reasons_attempts_consumed"]
    for c in g["cases"]:
        assert RR.reasons_attempts_consumed(c["limit"], c["disable"], g["reasons"]) == c["attempts"], c


@pytest.mark.parametrize("case", GOLDEN["reasons_attempts_edges"], ids=lambda c: f"limit{c['limit']}")
def test_reasons_attempts_edges(case):
    assert RR.reasons_attempts_consumed(case["limit"], case["disable"], case["reasons"]) == case["attempts"]


@pytest.mark.parametrize("case", GOLDEN["attempts_consumed"], ids=lambda c: c["name"])
def test_attempts_consumed(case):
    inst = [dict(status=s, reason=_reason(r)) for s, r in case["instances"]]
    assert RR.attempts_consumed(inst, GOLDEN["mea_culpa_limit"]) == case["attempts"]


@pytest.mark.parametrize("case", GOLDEN["transitions"], ids=lambda c: c["name"])
def test_transitions(case):
    inst = [dict(status=s, reason=_reason(r)) for s, r in case["instances"]]
    job = dict(state=case["old_job_state"], max_retries=case["retry_count"], disable=case["disable"])
    ups = [(k, st, _reason(r)) for k, (st, r) in enumerate(case["updates"]) if st is not None]
    assert RR.transact(job, inst, ups, GOLDEN["mea_culpa_limit"]) == case["new_job_state"]
    if len(ups) == 1:   # one status: one transaction either way
        assert RR.in_order(job, inst, ups, GOLDEN["mea_culpa_limit"]) == case["new_job_state"]


@pytest.mark.parametrize("case", GOLDEN["batch"], ids=lambda c: c["name"])
def test_batch_in_order(case):
    """Two failures of one job in one batch, one status at a time: the decisions cook_state_status returns."""
    inst = [dict(status=s, reason=_reason(r)) for s, r in case["instances"]]
    job = dict(state="running", max_retries=case["retry_count"], disable=False)
    ups = [(k, st, _reason(r)) for k, st, r in case["order"]]
    assert RR.in_order(job, inst, ups, GOLDEN["mea_culpa_limit"]) == case["new_job_state"]
    reason_of = {v["code"]: v for v in REASONS.values()}
    facts = dict(max_retries=case["retry_count"], disable=False, completed=False, done=[])
    live = len(ups)
    for (k, st, r), want, want_att in zip(case["order"], case["outcomes"], case["attempts"]):
        live -= 1
        oc, att, facts = RR.decide(facts, reason_of, st == "success", REASONS[r]["code"], live > 0)
        assert (oc, att) == (want, want_att)


@pytest.mark.parametrize("case", GOLDEN["novel"], ids=lambda c: f"{c['novel']}+{c['host']}p{int(c['preempted'])}")
def test_novel_host_append(case):
    assert RR.novel_after(case["novel"], case["host"], case["preempted"]) == case["after"]
    row = dict(novel=case["novel"], reserved_host=4, cpus=1.0)
    assert RR.requeued_row(row, case["host"], case["preempted"]) == dict(row, novel=case["after"], reserved_host=-1)


def test_previous_hosts_to_avoid():
    inst = [dict(hostname="a"), dict(hostname="b", preempted=True), dict(hostname="c", preempted=False),
            dict(hostname="a", preempted=True)]
    assert RR.previous_hosts_to_avoid(inst) == {"a", "c"}


def test_decide_matches_update_state():
    """decide (the resident handle's per-status decision from facts) against job_state_after on every one-status
    transition from a live instance."""
    reason_of = {v["code"]: v for v in REASONS.values()}
    n = 0
    for case in GOLDEN["transitions"]:
        ups = [(k, st, r) for k, (st, r) in enumerate(case["updates"]) if st is not None]
        if len(ups) != 1 or ups[0][1] not in RR.DONE or case["instances"][ups[0][0]][0] not in ("running", "unknown"):
            continue
        k, st, r = ups[0]
        others = [s for j, (s, _) in enumerate(case["instances"]) if j != k]
        done = [REASONS[rr]["code"] if rr else -1 for s, rr in [case["instances"][j] for j in range(len(others) + 1)
                                                                 if j != k] if s in RR.DONE]
        facts = dict(max_retries=case["retry_count"], disable=case["disable"],
                     completed=case["old_job_state"] == "completed", done=done)
        oc, _, _ = RR.decide(facts, reason_of, st == "success", REASONS[r]["code"],
                             any(s in ("running", "unknown") for s in others))
        assert oc == case["new_job_state"], case["name"]
        n += 1
    assert n >= 20


@pytest.mark.parametrize("case", GOLDEN["attempts_consumed"], ids=lambda c: c["name"])
def test_cycle_retry_facts(case):
    """cycle.retry_facts builds the done reasons whose attempts the restatement counts as the reference does."""
    table = {k: v["code"] for k, v in REASONS.items()}
    done, completed = cycle.retry_facts([tuple(i) for i in case["instances"]], table)
    reason_of = {v["code"]: v for v in REASONS.values()}
    assert RR.reasons_attempts_consumed(GOLDEN["mea_culpa_limit"], False, [reason_of.get(c) for c in done]) == \
        case["attempts"]
    assert completed == any(s == "success" for s, _ in case["instances"])
