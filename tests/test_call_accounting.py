"""-m gpu: what a phase call reports about itself, and each phase's buffers sized on a fresh handle.

  h2d_bytes    the bytes of the host columns the call reads, summed here from the arrays the test built,
               once with every optional column (constraints, CSR lists, groups, ports) and once without;
  n_launches   the kernels a call launches: rank and match below one sort tile and past two merge passes,
               the rebalancer with and without running tasks;
  sizing       arenas only grow, so an earlier, larger call hides a buffer list that falls short: each case
               runs on a fresh handle, with inputs where one optional list dominates the call's buffers
               (very long novel-host lists, many port ranges, groups of tens of thousands of cotasks, a
               traced rebalance with forced decisions), and must match the oracle.
"""
import numpy as np
import pytest

from cook_b200 import abi, traces
from cook_b200.engine import GpuEngine
from test_constraint_paths import _groups, rebalance_case

pytestmark = pytest.mark.gpu

USER_RANK = ("name_rank", "div_mem", "div_cpus", "div_gpus", "quota_count", "quota_cpus", "quota_mem", "quota_gpus")
USER_MATCH = ("quota_count", "quota_cpus", "quota_mem", "quota_gpus", "usage_count", "usage_cpus", "usage_mem",
              "usage_gpus", "tokens")
USER_REB = ("name_rank", "div_mem", "div_cpus", "quota_count", "quota_cpus", "quota_mem", "quota_gpus")
PENDING_NOT_REB = ("allowed", "plugin_accept", "ports", "reserved_host")   # match-only job columns


def _nbytes(soa, names=None, skip=()):
    """Bytes of the arrays behind soa's pointer fields (only `names`, if given; never `skip`)."""
    names = names or [n for n, _ in soa._fields_]
    return sum(soa.col(n).nbytes for n in names
               if n not in skip and isinstance(soa.col(n), np.ndarray))


def _with(soa, **kw):
    """A copy of soa with some columns replaced (None drops one)."""
    f = {}
    for n, ctype in soa._fields_:
        if isinstance(soa.col(n), (np.ndarray, abi._SoA)):
            f[n] = soa.col(n)
        elif ctype not in abi._NP:
            f[n] = getattr(soa, n)
    f.update(kw)
    return type(soa)(**f)


def _fresh(fn):
    eng = GpuEngine(pool_name="accounting")
    try:
        return fn(eng)
    finally:
        eng.close()


# ---- h2d_bytes -------------------------------------------------------------------------------------
def _rank_h2d(gpu, running, pending, users):
    gpu.rank(running, pending, users)
    want = _nbytes(pending) + _nbytes(users, USER_RANK) + (_nbytes(running) if running is not None else 0)
    assert gpu.last_stats(abi.PHASE_RANK)["h2d_bytes"] == want


def test_rank_h2d_bytes(gpu):
    t = traces.gen_pool(91, 3000, 100, 40, 800)
    _rank_h2d(gpu, t["running"], t["pending"], t["users"])
    # no running tasks, and a user table without the columns rank does not read
    users = _with(t["users"], usage_count=None, usage_cpus=None, usage_mem=None, usage_gpus=None, tokens=None)
    _rank_h2d(gpu, None, t["pending"], users)


def _match_h2d(gpu, ranked, jobs, offers, users, groups):
    prm = traces.match_params(jobs.n)
    m = gpu.match(ranked, jobs, offers, users, prm, groups=groups, max_ports=2)
    want = ranked.nbytes + _nbytes(jobs) + _nbytes(offers) + _nbytes(users, USER_MATCH)
    if groups is not None:
        want += _nbytes(groups) + 4 * (groups.n_groups + 1)   # and the offsets of each group's placed list
    assert m["stats"]["h2d_bytes"] == gpu.last_stats(abi.PHASE_MATCH)["h2d_bytes"] == want
    return m


def test_match_h2d_bytes(gpu):
    t = traces.gen_c3_pool(92, 3000, 200, 30, 600)
    ranked = gpu.rank(t["running"], t["pending"], t["users"])["ranked"]
    j, o = t["jobs"], t["offers"]
    assert all(j.col(c) is not None for c in ("novel_off", "attr_off", "group_off", "ports", "est_end_ms"))
    assert all(o.col(c) is not None for c in ("port_off", "gpu_off", "disk_off", "attr", "reserved"))
    _match_h2d(gpu, ranked, j, o, t["users"], t["groups"])
    # the columns every match reads, nothing else
    jobs = abi.JobsSoA(n=j.n, user=j.col("user"), cpus=j.col("cpus"), mem=j.col("mem"))
    offers = abi.OffersSoA(n=o.n, name_rank=o.col("name_rank"), cpus=o.col("cpus"), mem=o.col("mem"),
                           run_cpus=o.col("run_cpus"), run_mem=o.col("run_mem"))
    _match_h2d(gpu, ranked, jobs, offers, t["users"], None)


def _reb_h2d(gpu, r):
    gpu.rebalance(r["running"], r["pending"], r["pending_job_id"], r["pending_priority"], r["hosts"], r["users"],
                  r["params"], groups=r["groups"])
    pend_skip = PENDING_NOT_REB + (() if r["groups"] is not None else ("group_off", "group_idx"))
    want = (_nbytes(r["running"].col("t")) + r["running"].col("host").nbytes + _nbytes(r["users"], USER_REB) +
            _nbytes(r["hosts"]) + _nbytes(r["pending"], skip=pend_skip) +
            np.asarray(r["pending_job_id"], np.int64).nbytes + np.asarray(r["pending_priority"], np.int32).nbytes)
    if r["groups"] is not None:
        want += _nbytes(r["groups"])
    assert gpu.last_stats(abi.PHASE_REBALANCE)["h2d_bytes"] == want


def test_rebalance_h2d_bytes(gpu):
    r = traces.gen_rebalance(93, 4000, 300, 200, 60, constraints=True)
    assert r["groups"] is not None and r["pending"].col("novel_off") is not None
    _reb_h2d(gpu, r)
    r = traces.gen_rebalance(94, 4000, 300, 200, 60, constraints=False)
    t, h = r["running"].col("t"), r["hosts"]
    r["running"] = abi.RunningSoA(t=_with(t, gpus=None), host=r["running"].col("host"))
    r["hosts"] = abi.HostTable(n=h.n, hostname_id=h.col("hostname_id"), name_rank=h.col("name_rank"))
    _reb_h2d(gpu, r)


# ---- n_launches ------------------------------------------------------------------------------------
# one sort tile is 2048 indices: 1500 sort in the tile pass alone, 6000 take two merge passes
@pytest.mark.parametrize("n,want", [(1500, 15), (6000, 19)])
def test_rank_launches(gpu, n, want):
    t = traces.gen_pool(95, n - 500, 100, 40, 500)
    gpu.rank(t["running"], t["pending"], t["users"])
    assert gpu.last_stats(abi.PHASE_RANK)["n_launches"] == want


@pytest.mark.parametrize("n,want", [(1500, 14), (6000, 16)])
def test_match_launches(gpu, n, want):
    t = traces.gen_pool(96, n, 300, 40, 500)
    ranked = np.arange(n, dtype=np.int32)
    m = gpu.match(ranked, t["jobs"], t["offers"], t["users"], traces.match_params(n))
    assert m["stats"]["n_considerable"] > 0
    assert m["stats"]["n_launches"] == gpu.last_stats(abi.PHASE_MATCH)["n_launches"] == want


@pytest.mark.parametrize("n_running,want", [(0, 2), (1000, 13)])
def test_rebalance_launches(gpu, n_running, want):
    r = traces.gen_rebalance(97, max(n_running, 1), 200, 100, 40, constraints=False)
    if n_running == 0:
        t = r["running"].col("t")
        r["running"] = abi.RunningSoA(t=abi.make_tasks(*(t.col(c)[:0] for c in ("user", "priority", "start_time",
                                                                                 "task_id", "job_id", "cpus", "mem"))),
                                      host=np.zeros(0, np.int32))
    gpu.rebalance(r["running"], r["pending"], r["pending_job_id"], r["pending_priority"], r["hosts"], r["users"],
                  r["params"])
    assert gpu.last_stats(abi.PHASE_REBALANCE)["n_launches"] == want


# ---- sizing on a fresh handle -------------------------------------------------------------------------
def _match_case(oracle, jobs, offers, users, groups=None, max_ports=0, lifetime=0):
    ranked = np.arange(jobs.n, dtype=np.int32)
    prm = traces.match_params(jobs.n, host_lifetime_mins=lifetime)
    mg = _fresh(lambda e: e.match(ranked, jobs, offers, users, prm, groups=groups, max_ports=max_ports))
    mo = oracle.match(ranked, jobs, offers, users, prm, groups=groups, max_ports=max_ports)
    assert np.array_equal(mg["considerable"], mo["considerable"])
    assert np.array_equal(mg["assign"], mo["assign"])
    assert np.array_equal(mg["ports"], mo["ports"])
    assert mg["stats"]["n_matched"] == mo["stats"]["n_matched"] > 0
    return mg


def test_fresh_handle_long_novel_host_lists(oracle):
    """Four jobs with 300k novel hosts each (4.8 MB, more than the matcher's scratch), one of them
    listing every offer but the last."""
    t = traces.gen_pool(98, 400, 32, 10, 50)
    rng = np.random.default_rng(98)
    lists = [[] for _ in range(400)]
    for j in (0, 1, 2):
        lists[j] = list(rng.integers(1000, 10**6, 300_000))
    lists[3] = list(rng.integers(1000, 10**6, 300_000 - 31)) + list(range(31))
    off, host = abi.csr(lists)
    jobs = _with(t["jobs"], novel_off=off, novel_host=host)
    offers = _with(t["offers"], hostname_id=np.arange(32, dtype=np.int32))
    mg = _match_case(oracle, jobs, offers, t["users"])
    k = list(mg["considerable"]).index(3)
    assert mg["assign"][k] in (-1, 31)


def test_fresh_handle_many_port_ranges(oracle):
    """16 offers with 40k two-port ranges each (5 MB of ranges); a third of the jobs ask for ports."""
    t = traces.gen_pool(99, 600, 16, 10, 50)
    rng = np.random.default_rng(99)
    n = 40_000
    begin = np.tile(31000 + 3 * np.arange(n, dtype=np.int32), 16)
    off = (n * np.arange(17)).astype(np.int32)
    jobs = _with(t["jobs"], ports=np.where(rng.random(600) < 0.33, rng.integers(1, 3, 600), 0).astype(np.int32))
    offers = _with(t["offers"], port_off=off, port_begin=begin, port_end=begin + 1)
    mg = _match_case(oracle, jobs, offers, t["users"], max_ports=2)
    assert (mg["ports"][mg["assign"] >= 0] > 0).any()


def test_fresh_handle_large_groups_match(oracle):
    """60 jobs alternating between an attribute-equals and a unique group of 30k running cotasks each."""
    O, J, n = 12, 60, 30_000
    attr = np.array([[1 + v % 3 for v in range(O)]], np.int32)
    offers = abi.OffersSoA(n=O, hostname_id=np.arange(O, dtype=np.int32), name_rank=np.arange(O, dtype=np.int32),
                           cpus=np.full(O, 64.0), mem=np.full(O, 65536.0), run_cpus=np.zeros(O), run_mem=np.zeros(O),
                           run_count=np.zeros(O, np.int32), n_attr_cols=1, attr=attr.reshape(-1))
    off, idx = abi.csr([[j % 2] for j in range(J)])
    jobs = abi.JobsSoA(n=J, user=np.zeros(J, np.int32), cpus=np.ones(J), mem=np.full(J, 16.0), gpus=np.zeros(J),
                       group_off=off, group_idx=idx)
    # attribute-equals: values 1 and (past position 29 995) 2, so the VMs of value 3 fail; unique: cotasks on VMs
    # 0 and 1, then on hosts that are not offered
    groups = _groups([abi.GROUP_ATTR_EQUALS, abi.GROUP_UNIQUE], [0, -1], [0, 0],
                     [list(range(100, 100 + n)), [0, 1] + list(range(100 + n, 98 + 2 * n))],
                     [[1] * (n - 4) + [2] * 4, [0] * n])
    users = abi.make_users(1, div_mem=np.full(1, 1e6), div_cpus=np.full(1, 1e3), div_gpus=np.ones(1))
    mg = _match_case(oracle, jobs, offers, users, groups=groups)
    cons, a = mg["considerable"], mg["assign"]
    assert not np.isin(a[(cons % 2 == 0) & (a >= 0)], [2, 5, 8, 11]).any()
    assert not np.isin(a[(cons % 2 == 1) & (a >= 0)], [0, 1]).any()


def test_fresh_handle_large_group_rebalance(oracle):
    """An attribute-equals group of 40k cotasks whose values are 2 and 3: straw (4) fails, sticks (3) wins."""
    vals = [2] * 20_000 + [3] * 20_000
    groups = _groups([abi.GROUP_ATTR_EQUALS], [0], [0], [list(range(100, 100 + len(vals)))], [vals])
    args, groups = rebalance_case([[0]], groups)
    dg = _fresh(lambda e: e.rebalance(*args, groups=groups))
    assert dg == oracle.rebalance(*args, groups=groups)
    assert [d["host"] for d in dg] == [2]


def test_fresh_handle_forced_trace(oracle):
    """cook_rebalance_trace with 600 forced decisions, of which every tenth takes three victims of its host
    that no other decision took."""
    r = traces.gen_rebalance(100, 3000, 2000, 40, 30, constraints=False)
    host = r["running"].col("host")
    forced = []
    for i in range(600):
        h, k = i % 40, 3 * (i // 40)
        vs = [int(v) for v in np.flatnonzero(host == h)[k:k + 3]] if i % 10 == 0 else []
        forced.append((i, h, vs, 0.0, 0.0, 0.0))
    args = (r["running"], r["pending"], r["pending_job_id"], r["pending_priority"], r["hosts"], r["users"],
            r["params"])
    tg = _fresh(lambda e: e.rebalance_trace(*args, forced=forced))
    to = oracle.rebalance_trace(*args, forced=forced)
    assert tg["decisions"] == to["decisions"]
    assert tg["order"] == to["order"] and len(to["order"]) > 300
    assert np.array_equal(np.array(tg["order_dru"]).view(np.int64), np.array(to["order_dru"]).view(np.int64))
    assert tg["below_quota"] == to["below_quota"]
    assert np.array_equal(tg["pending_dru"], to["pending_dru"], equal_nan=True)
