"""The matcher's commit hand-off at every turn residue (family 8 of match_edge_cases.py) against the oracle.

Queue entry g is commit warp g mod NCW's turn: the jobs the driver found feasible, an END entry after each block's
jobs and an EXIT entry last.  Short queues (J = 1 .. 2 NCW + 2 jobs, one block) land the END and the EXIT turn on
every owner and leave owners without a job turn; long queues (many adaptive blocks, more than 2 RING NCW turns)
take every hand[] barrier of the plain kernel through dozens of phases.

Without a GPU: the cases' inputs are what they claim and the oracle's answer equals the hand-computed one and a
plain restatement of the greedy match.  With one: cook_match equals the oracle bit for bit under each knob
setting, and the per-turn timeline of the profiling instantiation (COOK_PROF_TRACE) has the queue's structure:
every turn recorded, jobs in queue order, END entries in block order after their block's jobs, END and EXIT on
every residue, and both forms of the plain kernel's hand-off taken.  No assertion orders the clocks of two turns:
a turn's TT_DONE is read after its chain store, so the next turn may stamp TT_HAND before it.
"""
import re

import numpy as np
import pytest

import match_edge_cases as E
from test_match_edges import _same, knobs_env, oracle_claims, oracle_failures, run

CASES = E.handoff_catalogue()
ALL = [(n, od) for n in CASES for od in E.ORDERS]
ids = lambda cases: [f"{n}-{od}" for n, od in cases]
BLOCK0 = {False: 64, True: 128}   # jobs in the first block (match_run: B)

# the timeline's file, as match_run writes it: an 8-word header (magic, turn rows, block rows, words per turn row,
# resolver clocks, n_cons, matched, commit warps), the turn rows, the block rows
TRACE_MAGIC = 0x314e5254
TT_FREE, TT_LAND, TT_READY, TT_SEEN, TT_DONE, TT_FENCE, TT_INFO, TT_K, TT_EVAL, TT_DEC, TT_HAND, TT_POLL = range(12)


def read_trace(path):
    raw = np.fromfile(path, dtype=np.uint64)
    assert raw[0] == TRACE_MAGIC, "not a turn trace"
    n_turn, words = int(raw[1]), int(raw[3])
    hdr = {"n_cons": int(raw[5]), "matched": int(raw[6]), "ncw": int(raw[7])}
    return hdr, raw[8:8 + n_turn * words].reshape(n_turn, words).astype(np.int64)


def short_names(constr):
    kn = "C" if constr else "P"
    return [n for n in CASES if n.startswith(f"8-short-{kn}-")]


# ---- CPU ----------------------------------------------------------------------------------------------------
def test_handoff_catalogue():
    """Short queues J = 1 .. 2 NCW + 2 in both pools for both kernels, each in one block: END (g = J) and EXIT
    (g = J + 1) on every owner, and one to NCW - 1 owners without a job turn."""
    for constr in (False, True):
        ncw, kn = E.NCW[constr], "C" if constr else "P"
        Js = range(1, 2 * ncw + 3)
        assert set(short_names(constr)) == {f"8-short-{kn}-{p}-J{J}" for p in E.SHORT_POOLS for J in Js}
        assert max(Js) < BLOCK0[constr]
        assert {J % ncw for J in Js} == {(J + 1) % ncw for J in Js} == set(range(ncw))
        assert {ncw - min(J, ncw) for J in Js} == set(range(ncw))
        for name in short_names(constr):
            c = CASES[name]("perm")
            assert c["constr"] == constr and c["nc"] == int(name.split("J")[-1])
            assert c["knobs"] == E.HANDOFF_KNOBS
        assert {f"8-long-{kn}-{nm}" for nm in E.long_queues()} <= set(CASES)


@pytest.mark.parametrize("name,order", ALL, ids=ids(ALL))
def test_handoff_oracle_reaches(oracle, name, order):
    c = CASES[name](order)
    o = oracle_claims(oracle, c)
    placed = int((o["assign"] >= 0).sum())
    if "-short-" in name:
        pool = name.split("-")[3]
        assert placed == (c["nc"] if pool == "fit" else min(c["nc"], E.SHORT_POOLS["full"]))
    else:
        # every placement is a job turn: more than 2 RING NCW of them, in a queue of many blocks
        assert placed > 2 * E.RING * E.NCW[c["constr"]] and c["nc"] > 8 * BLOCK0[c["constr"]]
        if name.endswith("-thin"):
            assert placed < c["nc"] // 2 and (o["assign"] < 0).any()


# ---- GPU ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,order", ALL, ids=ids(ALL))
def test_handoff_equals_oracle(gpu, oracle, name, order):
    """Every knob setting: assignments, ports, placed mask and counts bit for bit, and the failure counts."""
    c = CASES[name](order)
    o = run(oracle, c)
    of = oracle_failures(oracle, c) if c["fails"] else None
    for kn in c["knobs"]:
        with knobs_env(kn):
            g = run(gpu, c, kn)
        _same(g, o)
        if of is not None:
            assert gpu.match_failures(c["fails"]) == of, kn


def _skipped(err):
    got = re.findall(r"^\[cook_prof\] skipped\s+(\d+)$", err, re.M)
    assert len(got) == 1
    return int(got[0])


def check_turns(c, o, hdr, T, skipped, ncw):
    """The timing-free structure of one run's timeline; returns its END residues, its EXIT residue and the plain
    kernel's hand-off forms (job turns learned right after a fold, job turns learned after a wait)."""
    assert hdr == {"n_cons": c["nc"], "matched": o["stats"]["n_matched"], "ncw": ncw}
    rec = np.flatnonzero(T[:, TT_DONE])
    n = int(rec.max()) + 1            # the EXIT turn records no row: it is turn n
    R = T[:n]
    assert (R[:, TT_DONE] != 0).all(), "a turn before the last one was not recorded"
    assert not T[n:].any()
    kind, blk = R[:, TT_INFO] & 0xF, R[:, TT_INFO] >> 32
    job, end = kind == 0, kind == 1
    assert (job | end).all()
    # job turns: the driver's queue in order, every job it did not skip, placed exactly as the oracle places
    gj = np.flatnonzero(job)
    k = R[job, TT_K]
    assert (np.diff(k) > 0).all() and k.min() >= 0 and k.max() < c["nc"]
    assert len(k) == c["nc"] - skipped
    assert ((R[job, TT_INFO] >> 21) & 1).tolist() == (o["assign"][k] >= 0).astype(int).tolist()
    assert set(np.flatnonzero(o["assign"] >= 0).tolist()) <= set(k.tolist())
    # END turns: blocks 0, 1, 2, ... in order, the last turn, each job turn between its block's END and the one
    # before it
    ge = np.flatnonzero(end)
    assert blk[end].tolist() == list(range(len(ge))) and end[-1]
    bj = blk[job]
    assert (bj < len(ge)).all() and (ge[bj] > gj).all()
    assert ((bj == 0) | (ge[np.maximum(bj - 1, 0)] < gj)).all()
    poll = R[job, TT_POLL]
    return dict(end=set((ge % ncw).tolist()), exit=n % ncw, n_end=len(ge), n_job=len(gj),
                midfold=int(((poll >> 32) & 1).sum()), waited=int(((poll & 0xFFFFFFFF) > 0).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("constr", [False, True])
def test_turn_trace_structure(gpu, oracle, capfd, tmp_path, constr):
    """Every short queue and every long queue once more with COOK_PROF_TRACE: equal to the oracle, each timeline
    well formed, END and EXIT turns on every owner, the long queues over many blocks and more than 2 RING NCW
    turns, and in the plain kernel both forms of the hand-off: learned right after a fold and learned after
    sleeping on hand[]."""
    ncw, kn = E.NCW[constr], "C" if constr else "P"
    names = short_names(constr) + [f"8-long-{kn}-{nm}" for nm in E.long_queues()]
    end_res, exit_res, midfold, waited = set(), set(), 0, 0
    for i, name in enumerate(names):
        c = CASES[name]("perm")
        o = run(oracle, c)
        path = tmp_path / f"turns{i}.bin"
        capfd.readouterr()
        with knobs_env({}, trace=path):
            g = run(gpu, c)
        _same(g, o)
        if c["fails"]:
            assert gpu.match_failures(c["fails"]) == oracle_failures(oracle, c), name
        hdr, T = read_trace(path)
        got = check_turns(c, o, hdr, T, _skipped(capfd.readouterr().err), ncw)
        if "-short-" in name:
            # one block: J job turns, END at g = J, EXIT at g = J + 1
            assert got["n_end"] == 1 and got["n_job"] == c["nc"] and got["exit"] == (c["nc"] + 1) % ncw, name
        else:
            assert got["n_end"] >= 8 and got["n_job"] > 2 * E.RING * ncw, (name, got)
        end_res |= got["end"]
        exit_res.add(got["exit"])
        midfold += got["midfold"]
        waited += got["waited"]
    assert end_res == exit_res == set(range(ncw)), (end_res, exit_res)
    if not constr:
        assert midfold > 0 and waited > 0, (midfold, waited)
