"""CPU: the grid rule behind the parallel scans of cook_b200/csrc/fold.cuh is sufficient, the
off-grid and large inputs of the GPU fold tests really depend on the association, and the fold
harness compiles for sm_90a."""
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import fold_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))


def _random_association(xs, rng):
    """Sum of xs under a random binary tree over a random permutation."""
    items = [float(x) for x in xs]
    rng.shuffle(items)
    while len(items) > 1:
        i = rng.randrange(len(items) - 1)
        items[i:i + 2] = [items[i] + items[i + 1]]
    return items[0]


def _cases_inside(rng):
    """(addends, start) that the rule accepts, at and just inside its boundary."""
    g = R.GRID
    out = []
    for n in (7, 8, 31, 64, 200):          # 2^43 / (n + 1) <= 2^40
        m = 2.0 ** 43 / (n + 1) - 1.0           # (n + 1) * m just below 2^43
        m = np.floor(m / g) * g
        xs = [m - g * rng.randrange(0, 1024) for _ in range(n)]
        out.append((xs, 0.0))
        out.append((xs[:-1], m))                  # the start value takes one addend's place
    out.append(([R.VMAX] * 6, 0.0))               # 7 * 2^40 < 2^43
    out.append(([g] * 3 + [R.VMAX] * 3, g * 3))
    out.append(([3 * g, 5 * g, 1.0 - g, 2.0 ** 30 + g] * 8, 7 * g))
    return out


def test_rule_accepts_the_inside_cases():
    rng = random.Random(1)
    for xs, start in _cases_inside(rng):
        assert R.grid_exact(R.grid_flag(xs), len(xs), start), (len(xs), start)


def test_every_association_equals_fsum_where_the_rule_holds():
    """Soundness: where the rule says yes, random permutations and pairings, the left fold, the
    reversed and the pairwise sums all give fsum's bits, prefix by prefix."""
    rng = random.Random(2)
    for xs, start in _cases_inside(rng):
        want = R.exact_sum(xs, start)
        assert R.left_total(xs, start) == want
        assert R.reversed_sum(xs, start) == want
        assert start + R.pairwise_sum(xs) == want
        for _ in range(200):
            assert _random_association(list(xs) + [start], rng) == want
        for k in range(1, len(xs) + 1):
            assert R.left_fold(xs, start)[k - 1] == R.exact_sum(xs[:k], start)


def _differs_somewhere(xs, start, rng, tries=3000):
    want = R.left_total(xs, start)
    if R.reversed_sum(xs, start) != want or start + R.pairwise_sum(xs) != want:
        return True
    return any(_random_association(list(xs) + [start], rng) != want for _ in range(tries))


def test_associations_differ_outside_the_rule():
    """The rule is sufficient, not exact: with (n + 1) in the bound, n addends at (n + 1) * m == 2^43
    still sum exactly.  Differences appear once the totals pass 2^43, or once an addend or the start
    value leaves the 2^-10 grid; each case below shows an association with other bits."""
    rng = random.Random(3)
    g = R.GRID
    # magnitude: (n + 1) * m at 2^44 with 2^-10 parts rounds somewhere
    xs = [2.0 ** 42 + g * k for k in (1, 3, 5)] + [g * 7, g]
    assert not R.grid_exact(R.grid_flag(xs), len(xs))
    assert _differs_somewhere(xs, 0.0, rng)
    # at the boundary (n + 1) * m == 2^43 the rule already says no; six more addends push the totals
    # past 2^43, where the 2^-10 parts round
    n = 7
    m = 2.0 ** 43 / (n + 1)
    xs = [m] + [m - g * (2 * k + 1) for k in range(n - 1)]
    assert not R.grid_exact(R.grid_flag(xs), n)
    assert R.grid_exact(R.grid_flag(xs[1:]), n - 1)
    assert _differs_somewhere(xs + [m - g * (6 * k + 3) for k in range(6)], 0.0, rng)
    # the grid: 2^-11 parts, every sum below 2^43
    xs = [2.0 ** 41 + 2.0 ** -11, 2.0 ** -11, 2.0 ** 41, 2.0 ** -11]
    assert R.grid_flag(xs)[0] == 1
    assert _differs_somewhere(xs, 0.0, rng)
    # the start value: off the grid while the addends are on it
    xs = [2.0 ** 40 - g, g, 3 * g, 2.0 ** 40, 5 * g]
    assert R.grid_exact(R.grid_flag(xs), len(xs), 0.0)
    assert not R.grid_exact(R.grid_flag(xs), len(xs), 0.1)
    assert not R.grid_exact(R.grid_flag(xs), len(xs), 2.0 ** 41 + 0.1)
    assert _differs_somewhere(xs, 2.0 ** 41 + 0.1, rng)


def test_rule_restatement_on_the_boundary_table():
    """The Python rule itself, value by value (the GPU test compares the device against it)."""
    ok = R.grid_value_ok
    assert ok(0.0) and ok(-0.0) and ok(2.0 ** -10) and ok(2.0 ** 40)
    assert not ok(2.0 ** -11) and not ok(3 * 2.0 ** -11) and not ok(np.nextafter(2.0 ** 40, np.inf))
    assert not any(ok(v) for v in (float("nan"), float("inf"), -(2.0 ** -10), 0.1))
    f = R.grid_flag([3.0, 1.0])
    n0 = int(2.0 ** 43 // 3.0) - 1
    assert R.grid_exact(f, n0 - 1) and not R.grid_exact(f, n0 + 1)
    f = R.grid_flag([0.25])                       # m < 1: the bound uses max(m, 1)
    assert R.grid_exact(f, 2 ** 43 - 2) and not R.grid_exact(f, 2 ** 43 - 1)
    assert R.grid_exact(f, 0, 2.0 ** 43 - 2.0 ** -10 - 1.0) is False   # start past 2^40
    assert R.grid_exact(f, 3, 2.0 ** 40) and not R.grid_exact(f, 3, 2.0 ** -11)


@pytest.mark.parametrize("regime,offset", [("off", 0.0), ("mixed", 0.0), ("grid", 1 / 3), ("mixed", 1 / 3)])
def test_below_quota_folds_are_association_sensitive(regime, offset):
    """The job-below-quota folds of test_job_below_quota_fold: off the grid (amounts or the pending
    request) or past 2^43, some lead job's fold differs from its reversed or pairwise sum, so with the
    quota on the left fold's last bit a kernel that summed in another order would flip an answer.  On the
    grid every fold is exact."""
    r = R.fold_rebalance(regime, 11, lead_mem_offset=offset)
    folds = [R.below_quota_mem(r, p) for p in range(len(r["lead"]))]
    assert any(R.association_sensitive(xs) for xs in folds)
    g = R.fold_rebalance("grid", 11)
    for p in range(len(g["lead"])):
        xs = R.below_quota_mem(g, p)
        assert R.left_total(xs) == R.exact_sum(xs) and not R.association_sensitive(xs)


@pytest.mark.parametrize("regime", ["off", "mixed"])
def test_path_traces_are_association_sensitive(regime):
    """The off-grid and large-value traces of test_fold_paths: in some user's running sum (a DRU
    score), the left fold differs from the reversed or pairwise sum of the same prefix, so a kernel
    that summed in another order would fail them."""
    t = R.fold_pool(regime, 7)
    c = t["cols"]
    user = np.concatenate([c["run"]["user"], c["pend"]["user"]])
    for col in ("mem",):
        amt = np.concatenate([c["run"][col], c["pend"][col]])
        assert R.segments_sensitive(amt, user)
    r = R.fold_rebalance(regime, 11)
    assert R.segments_sensitive(r["run"]["mem"], r["run"]["user"])


def test_primitive_inputs_are_association_sensitive():
    """The 'off' and 'wild' values of test_fold_primitives fold differently in another order."""
    import test_fold_primitives as P
    rng = np.random.default_rng(5)
    for kind in ("off", "wild"):
        xs = list(P._values(rng, kind, 129))
        assert R.association_sensitive(xs, 0.7)


def test_grid_traces_take_the_exact_path():
    t = R.fold_pool("grid", 7)
    c = t["cols"]
    cpus = np.concatenate([c["run"]["cpus"], c["pend"]["cpus"]])
    mem = np.concatenate([c["run"]["mem"], c["pend"]["mem"]])
    assert R.grid_exact(R.grid_flag(cpus, mem, None), len(cpus))
    assert sum(c["counts"]) < 30_000
    starts = np.concatenate([[0], np.cumsum(c["counts"])])
    assert R.OS_TILE in starts and R.LONG_USER > 2 * R.OS_TILE
    for k in (1, 31, 32, 33, 127, 128, 129):
        assert k in c["counts"]


def test_fold_probe_compiles_for_sm_90a(tmp_path):
    """tests/fold_probe.cu builds with the product's nvcc flags (skipped where nvcc is absent)."""
    import __graft_entry__ as g
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which("nvcc")):
        pytest.skip("nvcc not installed")
    out = tmp_path / "libfoldprobe.so"
    subprocess.check_call([nvcc] + g.NVCC_FLAGS + ["-o", str(out), os.path.join(HERE, "fold_probe.cu")])
    assert out.stat().st_size > 0
