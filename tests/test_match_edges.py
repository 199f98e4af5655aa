"""The matcher's rare decisions against the oracle: equal-fitness ties at chunk and tile edges, fitnesses one
ulp apart, exact fits on and off the grid (cpus, mem, ports), supply confined to one or two chunks, crowded
commit turns under the pipeline's knobs, group conflicts, and the block, sparse-mode and shared-memory size
edges.  The cases are built in match_edge_cases.py.

Without a GPU: every case's inputs are valid and the oracle's answer shows what the case claims; the oracle
also equals a plain restatement of the greedy match (match_edge_cases.greedy) on every case without groups.
With one: cook_match equals the oracle bit for bit under each of the case's knob settings, the failure counts
agree, and the cases still reach their branches (public counters, and the COOK_PROF counters of the crowded
turns).
"""
import contextlib
import os
import re

import numpy as np
import pytest

import match_edge_cases as E
from cook_b200 import abi, traces

CASES = E.catalogue()
ALL = [(n, od) for n in CASES for od in E.ORDERS]
ids = lambda cases: [f"{n}-{od}" for n, od in cases]
KNOB_KEYS = ("COOK_KMIN", "COOK_LOOKAHEAD", "COOK_NSPEC", "COOK_NO_SPARSE", "COOK_NO_SMEM_STATIC", "COOK_PROF")
THRESHOLD = ("7-smem", "7-sbw", "7-gate")


@contextlib.contextmanager
def knobs_env(kn, prof=False):
    """The case's COOK_* settings for the duration of the block; the environment is restored after it."""
    saved = {k: os.environ.get(k) for k in KNOB_KEYS}
    try:
        for k in KNOB_KEYS:
            os.environ.pop(k, None)
        os.environ.update({k: v for k, v in kn.items() if k.startswith("COOK_")})
        if prof:
            os.environ["COOK_PROF"] = "1"
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def run(eng, case, kn=None):
    p = traces.match_params(case["nc"], max_ctas=(kn or {}).get("max_ctas", 0))
    return eng.match(*case["args"], p, **case["kw"])


def oracle_failures(oracle, case):
    return oracle.match_failures(*case["args"], traces.match_params(case["nc"]), case["fails"],
                                 groups=case["kw"]["groups"])


# ---- CPU: the inputs and what the oracle does with them -------------------------------------------------------
def test_catalogue():
    """Every family for both kernels where it applies; name ranks never the identity; small cases."""
    fam = {}
    for name, b in CASES.items():
        for od in E.ORDERS:
            c = b(od)
            _, jobs, offers, _ = c["args"]
            J, O = jobs.n, offers.n
            rank = offers.col("name_rank")
            assert sorted(rank.tolist()) == list(range(O)), name
            if O > 1:
                assert (rank != np.arange(O)).any(), name
            if not name.startswith(THRESHOLD):
                assert J * O <= 10 ** 8, name
            assert c["nc"] == J and all(k.startswith("COOK_") or k == "max_ctas" for kn in c["knobs"] for k in kn)
            fam.setdefault(name[0], set()).add(c["constr"])
    assert fam == {"1": {False, True}, "2": {False, True}, "3": {False, True}, "4": {False, True},
                   "5": {False, True}, "6": {True}, "7": {False, True}}
    assert E.ranks(33, "perm").tolist() != E.ranks(33, "rev").tolist()


def test_threshold_constants():
    """The shared-memory limits restated from the struct sizes (see match_edge_cases) and the catalogue's cases
    on either side of them."""
    ev_base = (49216 + 127) // 128 * 128
    fits_static = lambda O: ev_base + 32 * O + 8324 <= 224 * 1024
    res = lambda O, constr: 160224 + (16 * -(-O // 32) if constr else 0)
    fits_latest = lambda O, constr: res(O, constr) + 4 * O <= 200 * 1024
    assert fits_static(E.SMEM_STATIC_O) and not fits_static(E.SMEM_STATIC_O + 1)
    for constr in (False, True):
        O = E.LATEST_O[constr]
        assert fits_latest(O, constr) and not fits_latest(O + 1, constr)
    assert -(-E.SBW_O // 32) == 1024 and -(-(E.SBW_O + 1) // 32) == 1025
    for O in (E.SMEM_STATIC_O, E.SMEM_STATIC_O + 1, E.LATEST_O[False], E.LATEST_O[False] + 1):
        assert f"7-smem-P-O{O}" in CASES
    for O in (E.SBW_O, E.SBW_O + 1, E.LATEST_O[True], E.LATEST_O[True] + 1):
        assert f"7-sbw-C-O{O}" in CASES or f"7-smem-C-O{O}" in CASES


@pytest.mark.parametrize("name,order", ALL, ids=ids(ALL))
def test_oracle_reaches(oracle, name, order):
    """The oracle's answer equals the hand-computed one, and the plain greedy restatement (cases without groups)."""
    c = CASES[name](order)
    o = oracle.match(*c["args"], traces.match_params(c["nc"]), **c["kw"])
    cl = c["claims"]
    assert o["considerable"].tolist() == list(range(c["nc"]))
    if "want" in cl:
        assert o["assign"].tolist() == cl["want"]
    if c["kw"]["groups"] is None:
        assign, ports = E.greedy(c)
        assert o["assign"].tolist() == assign.tolist()
        if c["kw"]["max_ports"]:
            mp = c["kw"]["max_ports"]
            assert o["ports"].tolist() == [p + [-1] * (mp - len(p)) for p in ports]
    assert o["stats"]["n_matched"] == int((o["assign"] >= 0).sum())
    assert ((o["fail"] == abi.FAIL_NONE) == (o["assign"] >= 0)).all()


def _fit_all(c, j, assign_before=()):
    """Fitness of job j on every VM after the placements `assign_before` (job, vm) of the same cycle."""
    _, jobs, offers, _ = c["args"]
    lc, lm, rc, rm = (offers.col(k) for k in ("cpus", "mem", "run_cpus", "run_mem"))
    ac, am = np.zeros(len(lc)), np.zeros(len(lc))
    for k, v in assign_before:
        ac[v] = ac[v] + jobs.col("cpus")[k]
        am[v] = am[v] + jobs.col("mem")[k]
    cj, mj = jobs.col("cpus")[j], jobs.col("mem")[j]
    no = (ac + cj > lc) | (am + mj > lm)
    return np.where(no, 0.0, (((cj + ac) + rc) / (lc + rc) + ((mj + am) + rm) / (lm + rm)) / 2.0)


@pytest.mark.parametrize("order", E.ORDERS)
def test_ties_go_to_the_lowest_name(oracle, order):
    """Among at least two bit-equal fitnesses the lowest name rank wins, which is neither the lowest input index
    nor the lowest index of the rank column's reverse."""
    for O in E.TIE_O[1:] + (4096,):
        c = E.ties(O, order, False)
        f = _fit_all(c, 0)
        best = np.flatnonzero(f == f.max())
        assert len(best) == O >= 2 and f.max() == c["claims"]["f0"]
        o = oracle.match(*c["args"], traces.match_params(c["nc"]))
        rank = c["rank"]
        assert o["assign"][0] == best[np.argmin(rank[best])] != 0
    # more tied jobs than 32 chunks x TOPK row entries
    c = E.ties(4096, order, False)
    assert c["nc"] > 32 * E.TOPK and all(v >= 0 for v in c["claims"]["want"])


@pytest.mark.parametrize("constr", [False, True])
@pytest.mark.parametrize("order", E.ORDERS)
def test_one_ulp_better_wins_despite_its_name(oracle, order, constr):
    c = E.ulp_pairs("ulp", order, constr)
    cl = c["claims"]
    assert cl["fb"] == np.nextafter(cl["fa"], np.inf)
    f = _fit_all(c, 0)
    b = cl["b_vms"]
    assert set(np.flatnonzero(f == f.max())) == set(b)
    assert min(c["rank"][b]) > max(np.delete(c["rank"], b))       # every better VM has a higher name
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    assert o["assign"][0] in b and o["assign"][len(b)] not in b


@pytest.mark.parametrize("order", E.ORDERS)
def test_bit_equal_after_rounding(oracle, order):
    """Different inputs, the same fitness bits: a plain tie, broken by name rank across both kinds of VM."""
    c = E.ulp_pairs("equal", order, False)
    _, _, offers, _ = c["args"]
    f = _fit_all(c, 0)
    assert len(set(f.tolist())) == 1
    assert len({(a, b) for a, b in zip(offers.col("mem"), offers.col("run_mem"))}) == 2
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    b = set(c["claims"]["b_vms"])
    kinds = [v in b for v in o["assign"][:-1]]
    assert kinds[0] != kinds[1] and sorted(c["rank"][o["assign"][:-1]]) == list(c["rank"][o["assign"][:-1]])


@pytest.mark.parametrize("res,regime", [("cpus", "grid"), ("cpus", "off"), ("mem", "grid"), ("mem", "off"),
                                        ("ports", "grid")])
def test_exact_fit_is_placed_and_its_twin_is_not(oracle, res, regime):
    got = {}
    for edge in ("exact", "ulp"):
        c = E.exact_fit(res, regime, edge, "perm", True)
        o = oracle.match(*c["args"], traces.match_params(c["nc"]), **c["kw"])
        T = c["claims"]["want"][0]
        assert o["assign"][:2].tolist() == [T, T]
        got[edge] = int(o["assign"][2])
        if res != "ports":
            L, (a, b, x) = c["claims"]["amounts"]
            acc = (0.0 + a) + b
            assert (acc + x <= L) == (edge == "exact")
        else:
            assert o["ports"].tolist()[2][:4 if edge == "exact" else 5] == c["claims"]["ports"][2]
    assert got["exact"] == T != got["ulp"] >= 0
    if res != "ports":
        L, a, b, x = E.exact_amounts(regime)
        xu = float(np.nextafter(x, np.inf))
        assert (0.0 + a) + b + x <= L < (0.0 + a) + b + xu
        # off the grid another association of the same three requests lets the twin fit
        assert (a + (b + xu) <= L) == (regime == "off")


@pytest.mark.parametrize("constr", [False, True])
@pytest.mark.parametrize("chunks", [[11], [3, 30]])
def test_single_chunk_places_more_than_a_row(oracle, chunks, constr):
    c = E.single_chunk(chunks, "perm", constr)
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    v = c["rank"][o["assign"]]
    assert (o["assign"] >= 0).all() and set((v % 32).tolist()) == set(chunks)
    for ch in chunks:
        assert (v % 32 == ch).sum() > E.TOPK


@pytest.mark.parametrize("per_vm", [1, 2])
def test_crowded_fills_best_first(oracle, per_vm):
    """Every placement takes the best VM left: each one supersedes the top of every later job's list."""
    c = E.crowded(per_vm, "perm", False)
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    a = o["assign"]
    assert (a >= 0).all()
    for k in range(0, len(a) - per_vm, per_vm):
        f = _fit_all(c, k, [(i, int(a[i])) for i in range(k)])
        assert f[a[k]] == f.max() and (f == f.max()).sum() == 1
    assert len(set(a.tolist())) == len(a) // per_vm


@pytest.mark.parametrize("order", E.ORDERS)
def test_group_conflicts(oracle, order):
    c = E.group_conflicts(order)
    o = oracle.match(*c["args"], traces.match_params(c["nc"]), **c["kw"])
    a, cl = o["assign"], c["claims"]
    uq, bal, eq = cl["members"]
    assert (a >= 0).all()
    assert a[uq].tolist() == cl["unique"]                        # distinct hosts, best-named first
    vals = cl["attr"][a[bal]]
    counts = np.bincount(vals, minlength=4)[1:]
    assert counts.max() - counts.min() <= 1
    assert len(set(cl["attr"][a[eq]].tolist())) == 1
    # without the groups the members would stack on the touched VMs
    f = _fit_all(c, uq[1], [(uq[0], int(a[uq[0]]))])
    assert np.argmax(f) == a[uq[0]]


@pytest.mark.parametrize("constr", [False, True])
def test_queue_turns_hopeless_mid_block(oracle, constr):
    c = E.hopeless("perm", constr)
    O = c["args"][2].n
    B = 128 if constr else 64
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    placed = np.flatnonzero(o["assign"] >= 0)
    assert placed.tolist() == list(range(O)) and B < O < 2 * B and c["nc"] > 2 * B


@pytest.mark.parametrize("constr", [False, True])
@pytest.mark.parametrize("live", [E.SL_MAX, E.SL_MAX + 1])
def test_sparse_edge_live_counts(oracle, live, constr):
    """After block 0 the supply chunk has exactly `live` VMs left, and block 2 exists."""
    c = E.sparse_edge(live, "perm", constr)
    _, jobs, offers, _ = c["args"]
    B = c["claims"]["B"]
    fits = (offers.col("cpus") >= jobs.col("cpus").min()) & (offers.col("mem") >= jobs.col("mem").min())
    per_chunk = np.bincount(c["rank"][fits] % 32, minlength=32)
    assert per_chunk.max() == B + live == per_chunk.sum() and c["nc"] > 3 * B
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    a = o["assign"]
    assert (a[:B] >= 0).all() and (a >= 0).sum() == B + live


@pytest.mark.parametrize("O", [E.SBW_O, E.SBW_O + 1])
def test_sbw_edge_is_sparse_shaped(oracle, O):
    """At most SL_MAX live VMs in every chunk, live VMs in the last tile of the 1024 verdict words (and in tile
    1024 past them at 32769), and the oracle places one job on each."""
    c = E.sbw_edge(O, "perm")
    _, jobs, offers, _ = c["args"]
    fits = offers.col("cpus") >= jobs.col("cpus").min()
    r = c["rank"][fits]
    assert np.bincount(r % 32, minlength=32).max() <= E.SL_MAX
    assert (r // 32 == 1023).any() and ((r // 32 == 1024).any() == (O > E.SBW_O))
    assert -(-O // 32) == (1024 if O == E.SBW_O else 1025)
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    assert (o["assign"] >= 0).sum() == fits.sum() < c["nc"]


@pytest.mark.parametrize("constr", [False, True])
@pytest.mark.parametrize("side", ["low", "high"])
def test_winner_ties_with_the_bound(oracle, side, constr):
    """For Y, the T an X changed and an untouched U fit bit for bit equally; the lower name takes Y: the T when
    the T's rank below every U's, else the next untouched U (the bound of a set computed before X and F)."""
    c = E.bound_tie(side, "perm", constr)
    cl = c["claims"]
    assert cl["f_t"] == cl["f_u"]
    o = oracle.match(*c["args"], traces.match_params(c["nc"]))
    a = o["assign"]
    rank = c["rank"]
    for i in range(0, len(a), 3):
        t = a[i]
        assert t in cl["ts"] and a[i + 1] in cl["us"]
        f = _fit_all(c, i + 2, [(k, int(a[k])) for k in range(i + 2)])
        tied = np.flatnonzero(f == f.max())
        assert f.max() == cl["f_t"] and t in tied and len(tied) >= 2
        assert a[i + 2] == tied[np.argmin(rank[tied])]
        assert (a[i + 2] == t) == (side == "low")


# ---- GPU: the kernel against the oracle -----------------------------------------------------------------------
def _same(g, o):
    assert np.array_equal(g["considerable"], o["considerable"])
    assert np.array_equal(g["assign"], o["assign"])
    assert np.array_equal(g["ports"], o["ports"])
    assert np.array_equal(g["fail"] == abi.FAIL_NONE, o["fail"] == abi.FAIL_NONE)
    assert g["stats"]["n_matched"] == o["stats"]["n_matched"]


@pytest.mark.gpu
@pytest.mark.parametrize("name,order", ALL, ids=ids(ALL))
def test_match_equals_oracle(gpu, oracle, name, order):
    """Every knob setting of the case: assignments, ports, placed mask and counts bit for bit; failure counts at
    the case's turns; families 4 and 6 still reach the chunk re-scan and the group full scan."""
    c = CASES[name](order)
    o = run(oracle, c)
    of = oracle_failures(oracle, c) if c["fails"] else None
    full = 0
    for kn in c["knobs"]:
        with knobs_env(kn):
            g = run(gpu, c, kn)
        _same(g, o)
        if of is not None:
            assert gpu.match_failures(c["fails"]) == of, kn
        if name.startswith("4-"):
            assert g["stats"]["n_chunk_rescan"] > 0, kn
        full += g["stats"]["n_full_rescan"]
    if name.startswith("6-"):
        assert full > 0


PROF_NAMES = ("fallbacks", "z_takes", "relooks", "trunc_specs", "chunk_rescan")


def _prof(err):
    out = {}
    for k in PROF_NAMES:
        got = re.findall(rf"^\[cook_prof\] {k}\s+(\d+)$", err, re.M)
        assert len(got) == 1, k
        out[k] = int(got[0])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("constr", [False, True])
def test_crowded_turns_reach_every_outcome(gpu, oracle, capfd, constr):
    """The crowded and swapped-bound cases once more with COOK_PROF=1 (the profiling instantiation of the kernel): equal to the
    oracle, and exact recomputations, bounds taken directly and relooks each happen under some knob setting."""
    seen = {k: 0 for k in PROF_NAMES}
    for name in [n for n in CASES if n.startswith("5-") and (n.split("-")[2] == "C") == constr]:
        c = CASES[name]("perm")
        o = run(oracle, c)
        for kn in c["knobs"]:
            capfd.readouterr()
            with knobs_env(kn, prof=True):
                g = run(gpu, c, kn)
            _same(g, o)
            got = _prof(capfd.readouterr().err)
            for k in PROF_NAMES:
                seen[k] += got[k]
    assert seen["fallbacks"] > 0 and seen["z_takes"] > 0 and seen["relooks"] > 0, seen
