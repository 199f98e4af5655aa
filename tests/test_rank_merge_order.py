"""-m gpu: cook_rank's merge order where a user's score repeats, against the oracle in both forms of
dru/sorted-merge (the literal re-sort and the heap).

In GPU mode a task's score is the user's cumulative gpus over its gpu share, so every task with gpus = 0
repeats the score of the task before it; in default mode a user with a zero share scores +inf on every
task.  Sizes sit at the sort's edges (one 2048-wide tile, one merge pass, an odd number of runs)."""
import numpy as np
import pytest

import merge_ref as M
from cook_b200 import abi, traces
from cook_b200.engine import GpuEngine
from oracle.pyoracle import OracleEngine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    g = {m: GpuEngine(pool_name=f"merge-order-{m}", dru_mode=m) for m in (0, 1)}
    yield g
    for e in g.values():
        e.close()


@pytest.fixture(scope="module")
def oracles(oracle):
    return {m: OracleEngine(dru_mode=m, lib=oracle.lib) for m in (0, 1)}


def _with_gpus(cols, rng, frac_zero, off_grid):
    n = len(cols["user"])
    g = np.where(rng.random(n) < frac_zero, 0.0, rng.choice([1.0, 2.0, 4.0, 8.0], n))
    cpus = cols["cpus"] + 0.1 if off_grid else cols["cpus"]
    return abi.make_tasks(**dict(cols, gpus=g, cpus=cpus))


def gpu_pool(seed, n_total, n_users, frac_zero, running_frac=0.25, off_grid=False):
    """gen_pool's shape in GPU mode: gpus 0 with probability frac_zero (else 1, 2, 4 or 8), running tasks
    too, gpu shares 1 .. 16.  off_grid: cpus 0.1 above gen_pool's, so the scores come from the per-user
    serial fold instead of the order-wide scans (each path writes the merge comparator's run starts)."""
    n_run = int(n_total * running_frac)
    t = traces.gen_pool(seed, n_total - n_run, 10, n_users, n_run)
    rng = np.random.default_rng(seed + 7)
    t["running"] = _with_gpus(t["cols"]["running"], rng, frac_zero, off_grid)
    t["pending"] = _with_gpus(t["cols"]["pending"], rng, frac_zero, off_grid)
    t["div_gpus"] = rng.integers(1, 17, n_users).astype(np.float64)
    t["users"] = abi.make_users(n_users, name_rank=t["cols"]["name_rank"], div_gpus=t["div_gpus"])
    return t


def _rank_all(gpu, ora, t, **kw):
    """The oracle's two forms must agree; then cook_rank must give their order, queue and scores."""
    args = (t["running"], t["pending"], t["users"])
    ora.lib.oracle_set_naive_merge(1)
    try:
        naive = ora.rank(*args, **kw)
    finally:
        ora.lib.oracle_set_naive_merge(0)
    heap = ora.rank(*args, **kw)
    for k in ("order", "ranked"):
        assert np.array_equal(naive[k], heap[k]), k
    got = gpu.rank(*args, **kw)
    assert len(got["order"]) == len(heap["order"])
    diff = np.flatnonzero(got["order"] != heap["order"])
    assert len(diff) == 0, f"order differs at {len(diff)} positions, first {diff[0]}"
    assert np.array_equal(got["ranked"], heap["ranked"])
    assert _same_scores(got["dru"], heap["dru"])
    return got, heap


def _same_scores(a, b):
    """Bit for bit, the cut tasks (NaN) at the same places."""
    cut = np.isnan(a)
    return np.array_equal(cut, np.isnan(b)) and np.array_equal(a[~cut].view(np.int64), b[~cut].view(np.int64))


SIZES = [2047, 2048, 2049, 4097, 3 * 2048 + 1]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("n_users", [1, 7, 1000])
@pytest.mark.parametrize("frac_zero", [0.0, 0.3, 0.7, 1.0])
def test_gpu_mode_merge_order(engines, oracles, n, n_users, frac_zero):
    t = gpu_pool(n + n_users + int(10 * frac_zero), n, n_users, frac_zero)
    got, _ = _rank_all(engines[1], oracles[1], t)
    d = got["dru"][got["order"]]
    assert np.all(np.diff(d) >= 0)


@pytest.mark.parametrize("n", [2049, 3 * 2048 + 1])
@pytest.mark.parametrize("n_users", [7, 1000])
@pytest.mark.parametrize("frac_zero", [0.3, 1.0])
def test_gpu_mode_merge_order_off_grid(engines, oracles, n, n_users, frac_zero):
    t = gpu_pool(n + n_users + 3, n, n_users, frac_zero, off_grid=True)
    _rank_all(engines[1], oracles[1], t)


@pytest.mark.parametrize("frac_zero", [0.7, 1.0])
def test_gpu_mode_merge_order_100k(engines, oracles, frac_zero):
    t = gpu_pool(41, 100_000, 50, frac_zero)
    _rank_all(engines[1], oracles[1], t)


@pytest.mark.parametrize("n,n_users", [(2049, 7), (3 * 2048 + 1, 200), (4097, 1000)])
@pytest.mark.parametrize("frac_zero", [0.3, 0.7])
@pytest.mark.parametrize("max_over", [0, 3])
def test_gpu_mode_cut_tails_and_quotas(engines, oracles, n, n_users, frac_zero, max_over):
    """Binding user quotas leave over-quota (NaN) tails right after runs; the pool and quota-group filters
    then walk the merged queue."""
    _cut_tails_and_quotas(engines, oracles, n, n_users, frac_zero, max_over, False)


@pytest.mark.parametrize("n,n_users", [(2049, 7), (4097, 1000)])
@pytest.mark.parametrize("max_over", [0, 3])
def test_gpu_mode_cut_tails_and_quotas_off_grid(engines, oracles, n, n_users, max_over):
    _cut_tails_and_quotas(engines, oracles, n, n_users, 0.7, max_over, True)


def _cut_tails_and_quotas(engines, oracles, n, n_users, frac_zero, max_over, off_grid):
    t = gpu_pool(n + 3 * n_users + max_over, n, n_users, frac_zero, off_grid=off_grid)
    rng = np.random.default_rng(n_users + max_over)
    quota = {"count": rng.integers(2, 40, n_users).astype(np.float64),
             "gpus": rng.integers(0, 30, n_users).astype(np.float64)}
    t["users"] = abi.make_users(n_users, name_rank=t["cols"]["name_rank"], div_gpus=t["div_gpus"], quota=quota)
    n_pend = t["pending"].n
    kw = dict(params=abi.RankParams(max_over, 0, 0.0, 0.0),
              pool_quota=abi.make_pool_quota({"count": n // 2, "cpus": 1e9, "mem": 1e12, "gpus": 2.0 * n_pend}),
              group_quota=abi.make_pool_quota({"count": n // 3, "cpus": 1e9, "mem": 1e12, "gpus": 1.5 * n_pend}),
              group_usage=np.array([5.0, 10.0, 4096.0, 3.0]))
    got, _ = _rank_all(engines[1], oracles[1], t, **kw)
    cut = np.isnan(got["dru"])
    assert cut.any() and not cut.all()
    assert 0 < len(got["ranked"]) < n_pend


@pytest.mark.parametrize("n,n_users", [(2049, 7), (3 * 2048 + 1, 200), (4097, 1000)])
def test_default_mode_zero_shares(engines, oracles, n, n_users):
    """Default mode, users with a zero share (+inf on every task) and users with a zero mem share whose
    tasks without mem score finite until the first one with mem, beside ordinary users."""
    _zero_shares(engines, oracles, n, n_users, False)


@pytest.mark.parametrize("n,n_users", [(2049, 7), (3 * 2048 + 1, 200), (4097, 1000)])
def test_default_mode_zero_shares_off_grid(engines, oracles, n, n_users):
    _zero_shares(engines, oracles, n, n_users, True)


def _zero_shares(engines, oracles, n, n_users, off_grid):
    t = traces.gen_pool(n + n_users, n - n // 4, 10, n_users, n // 4)
    rng = np.random.default_rng(n)
    for side in ("running", "pending"):
        cols = t["cols"][side]
        cpus = cols["cpus"] + 0.1 if off_grid else cols["cpus"]
        t[side] = abi.make_tasks(**dict(cols, cpus=cpus,
                                        mem=np.where(rng.random(len(cols["mem"])) < 0.3, 0.0, cols["mem"])))
    kind = rng.choice(3, n_users, p=[0.5, 0.3, 0.2])          # ordinary, zero share, zero mem share
    kind[0], kind[-1] = 1, 2
    div_cpus = np.where(kind == 1, 0.0, t["cols"]["div_cpus"])
    div_mem = np.where(kind > 0, 0.0, t["cols"]["div_mem"])
    t["users"] = abi.make_users(n_users, name_rank=t["cols"]["name_rank"], div_cpus=div_cpus, div_mem=div_mem)
    got, _ = _rank_all(engines[0], oracles[0], t)
    inf = np.isinf(got["dru"])
    assert inf.sum() > 1 and not np.isnan(got["dru"]).any()


@pytest.mark.parametrize("name", list(M.tie_tables()))
def test_tie_tables_through_cook_rank(engines, oracles, name):
    """The hand-built tables of merge_ref.py, ranked from shuffled task columns."""
    t = M.tie_tables()[name]
    pending, users, params, pos = M.table_ranking(t)
    got = engines[t["mode"]].rank(None, pending, users, params=params)
    assert np.array_equal(pos[got["order"]], t["merge"])
    assert np.array_equal(got["dru"], t["dru"][pos], equal_nan=True)


@pytest.mark.parametrize("name", [k for k, t in M.tie_tables().items() if t["mode"] == 1])
def test_tie_tables_through_cook_rank_off_grid(engines, oracles, name):
    t = M.tie_tables()[name]
    pending, users, params, pos = M.table_ranking(t, off_grid=True)
    got = engines[1].rank(None, pending, users, params=params)
    assert np.array_equal(pos[got["order"]], t["merge"])
    assert np.array_equal(got["dru"], t["dru"][pos], equal_nan=True)


def test_rank_then_match_gpu_mode_pool(engines, oracles):
    """A config-#3 pool where 98 % of the jobs ask for no GPU, ranked in GPU mode and matched."""
    t = traces.gen_c3_pool(51, 4000, 250, 60, 800, frac_gpu_jobs=0.02)
    rng = np.random.default_rng(52)
    t["pending"] = abi.make_tasks(**dict(t["cols"]["pending"], gpus=t["jobs"].col("gpus")))
    nr = t["running"].n
    t["running"] = abi.make_tasks(**dict(t["cols"]["running"],
                                         gpus=np.where(rng.random(nr) < 0.02, rng.choice([1.0, 2.0], nr), 0.0)))
    t["div_gpus"] = rng.integers(1, 17, 60).astype(np.float64)
    u = t["users"]
    t["users"] = abi.make_users(60, name_rank=t["cols"]["name_rank"], div_mem=t["cols"]["div_mem"],
                                div_cpus=t["cols"]["div_cpus"], div_gpus=t["div_gpus"],
                                usage={k: u.col("usage_" + k) for k in ("count", "cpus", "mem", "gpus")})
    got, want = _rank_all(engines[1], oracles[1], t)
    prm = traces.match_params(len(want["ranked"]), host_lifetime_mins=t["host_lifetime_mins"])
    mg = engines[1].match(got["ranked"], t["jobs"], t["offers"], t["users"], prm, groups=t["groups"], max_ports=2)
    mo = oracles[1].match(want["ranked"], t["jobs"], t["offers"], t["users"], prm, groups=t["groups"], max_ports=2)
    for k in ("considerable", "assign", "ports"):
        assert np.array_equal(mg[k], mo[k]), k
    assert np.array_equal(mg["fail"] == 0, mo["fail"] == 0)
    for k in ("n_considerable", "n_matched", "head_matched", "n_offers_used", "evals"):
        assert mg["stats"][k] == mo["stats"][k], k
    assert mg["stats"]["n_matched"] > 0
