"""CPU tests: the plain restatements of dru/sorted-merge in merge_ref.py against both forms of the oracle on
tables with runs of equal scores inside a user's list, and the property LessMerge's run rule rests on: a
user's run of equal consecutive scores is emitted contiguously."""
import numpy as np
import pytest

import merge_ref as M
from oracle.pyoracle import OracleEngine

TABLES = M.tie_tables()


def test_hand_case():
    t = M.hand_case()
    assert t["merge"] == [0, 1, 2, 3]                    # a1 a2 b1 b2
    assert M.heap_merge(t["lists"], lambda p: t["dru"][p]) == [0, 1, 2, 3]


def _oracle_rank(lib, t, naive):
    pending, users, params, pos = M.table_ranking(t)
    eng = OracleEngine(dru_mode=t["mode"], lib=lib)
    eng.set_naive_merge(naive)
    try:
        r = eng.rank(None, pending, users, params=params)
    finally:
        eng.set_naive_merge(0)
    return r, pos


@pytest.mark.parametrize("name", list(TABLES))
def test_merge_ref_equals_both_oracle_forms(oracle, name):
    t = TABLES[name]
    score = lambda p: t["dru"][p]
    assert t["merge"] == M.heap_merge(t["lists"], score)
    for naive in (1, 0):
        r, pos = _oracle_rank(oracle.lib, t, naive)
        assert np.array_equal(pos[r["order"]], t["merge"]), naive      # order as positions
        assert np.array_equal(r["dru"], t["dru"][pos], equal_nan=True)


def _runs(t):
    """Every run of equal consecutive kept scores in a user's list, as a list of positions (length >= 2)."""
    out = []
    for lst in t["lists"]:
        run = lst[:1]
        for p in lst[1:]:
            if t["dru"][p] == t["dru"][run[-1]]:
                run.append(p)
            else:
                if len(run) > 1:
                    out.append(run)
                run = [p]
        if len(run) > 1:
            out.append(run)
    return out


@pytest.mark.parametrize("name", list(TABLES))
def test_runs_are_emitted_contiguously(oracle, name):
    t = TABLES[name]
    r, pos = _oracle_rank(oracle.lib, t, 1)
    at = np.empty(len(t["dru"]), np.int64)
    at[pos[r["order"]]] = np.arange(len(r["order"]))
    runs = _runs(t)
    assert runs or name in ("inf_default", "inf_default_perm") or name.startswith("random")
    for run in runs:
        assert np.array_equal(at[run], at[run[0]] + np.arange(len(run))), run


def test_tables_have_the_chosen_runs():
    """The hand-built tables really hold runs across users with equal scores, cut tails and +inf."""
    s = TABLES["structured"]
    assert len(_runs(s)) >= 8 and len(s["cut"]) == 5
    assert np.unique(s["dru"][~np.isnan(s["dru"])]).tolist() == [0.0, 1.0, 2.0, 3.0]
    d = TABLES["inf_default"]
    assert np.isinf(d["dru"]).sum() == 10 and len(_runs(d)) == 4
    assert not np.array_equal(TABLES["structured_perm"]["perm"], np.arange(12))
