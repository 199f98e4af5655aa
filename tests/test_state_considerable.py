"""cook_state_considerable (M0 over the resident queue without a match) and cook_state_rank_offensive (the jobs the
rank drops as offensive).

CPU: the exports, the struct layout and the prototypes against the ctypes signatures (checked by the C compiler),
the phase and usage-source codes, and considerable_ref (a plain restatement of filter-pending-jobs-for-quota /
pending-jobs->considerable-jobs) against the oracle on K14, K9 and random cases.
GPU (-m gpu): after every batch of a churn, the considerable call against cook_match on host tables built from a
model with an empty offer table, and against considerable_ref; the autoscaling selection after a match and its
launches; consumption; the match plan left as it was; the offensive list; K14 through the resident state; errors
and transfers.
"""
import ctypes as C
import itertools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import considerable_ref as CR
from cook_b200 import abi, cycle, engine, traces
from cook_b200.engine import CookError, GpuEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "cook_gpu.h")
KEYS = ("count", "cpus", "mem", "gpus")
QUOTA_FIELDS = ("quota_count", "quota_cpus", "quota_mem", "quota_gpus")
USAGE_FIELDS = ("usage_count", "usage_cpus", "usage_mem", "usage_gpus")
NEW = ("cook_state_considerable", "cook_state_rank_offensive")


# ---- CPU -------------------------------------------------------------------------------------------------
def _prototype(hdr, name):
    m = re.search(r"int32_t\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_entries_exported():
    hdr = open(HDR).read()
    for name in NEW:
        _prototype(hdr, name)
    if not os.path.exists(engine.LIB_PATH):
        pytest.skip("libcookgpu.so not built")
    lib = engine.load_library()
    for name in NEW:
        assert hasattr(lib, name), name
        assert getattr(lib, name).restype is C.c_int32
        assert getattr(lib, name).argtypes == abi.ARGTYPES[name]


# ctypes -> the C spelling the header uses
_C_OF = {C.c_void_p: "cook_pool*", C.c_int32: "int32_t", abi.P_I64: "int64_t*", abi.P_I32: "int32_t*",
         abi.P_F64: "const double*", C.POINTER(abi.UserTable): "const cook_user_table*",
         C.POINTER(abi.PoolQuota): "const cook_pool_quota*", C.POINTER(abi.RankParams): "const cook_rank_params*",
         C.POINTER(abi.ConsiderableParams): "const cook_considerable_params*"}
_C_FIELD = {C.c_int32: "int32_t"}


def test_layout_and_prototypes_compile(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    P = abi.ConsiderableParams
    lines = ['#include <stddef.h>', '#include "cook_gpu.h"',
             f'_Static_assert(sizeof(cook_considerable_params) == {C.sizeof(P)}, "size");']
    for name, ct in P._fields_:
        assert ct in _C_FIELD
        lines.append(f'_Static_assert(offsetof(cook_considerable_params, {name}) == {getattr(P, name).offset}, "{name}");')
        lines.append(f'_Static_assert(__builtin_types_compatible_p(__typeof__(((cook_considerable_params*)0)->{name}), '
                     f'{_C_FIELD[ct]}), "{name} type");')
    for fn in NEW:
        args = ", ".join(_C_OF[t] for t in abi.ARGTYPES[fn])
        lines.append(f'_Static_assert(__builtin_types_compatible_p(__typeof__({fn}), int32_t ({args})), "{fn}");')
    lines.append('_Static_assert(COOK_PHASE_CONSIDERABLE == %d, "phase");' % abi.PHASE_CONSIDERABLE)
    lines.append('_Static_assert(COOK_USAGE_GIVEN == %d && COOK_USAGE_DERIVED == %d && COOK_USAGE_LAST_MATCH == %d, '
                 '"usage sources");' % (abi.USAGE_GIVEN, abi.USAGE_DERIVED, abi.USAGE_LAST_MATCH))
    lines.append('int main(void) { return 0; }')
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    subprocess.check_call([cc, "-std=gnu11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "l")])


def test_phase_code():
    assert abi.PHASE_CONSIDERABLE == 7
    hdr = open(HDR).read()
    assert re.search(r"COOK_PHASE_CONSIDERABLE\s*=\s*7", hdr)
    # one more than the last phase before it
    assert abi.PHASE_CONSIDERABLE == abi.PHASE_COTASKS + 1


class RefEngine:
    """considerable_ref behind the `match` call shape the K14 / K9 cases use (considerable set only)."""

    @staticmethod
    def match(ranked_idx, jobs, offers, users, params, groups=None, pool_quota=None, max_ports=0):
        quota = {k: users.col(f) for k, f in zip(KEYS, QUOTA_FIELDS)}
        usage = {k: users.col(f) for k, f in zip(KEYS, USAGE_FIELDS)}
        pq = None
        if pool_quota is not None and pool_quota.enabled:
            pq = {k: getattr(pool_quota, k) for k in KEYS}
        gpus = jobs.col("gpus") if jobs.col("gpus") is not None else np.zeros(jobs.n)
        out = CR.considerable(list(ranked_idx), jobs.col("user"), jobs.col("cpus"), jobs.col("mem"), gpus, quota,
                              usage, params.num_considerable, tokens=users.col("tokens"),
                              enforce_rate_limit=params.enforce_rate_limit, pool_quota=pq,
                              allowed=jobs.col("allowed"), plugin_accept=jobs.col("plugin_accept"))
        return {"considerable": np.array(out, np.int32)}


def test_ref_known_answers():
    from considerable_golden_cases import check_all
    check_all(RefEngine())   # K14's hand-transcribed answers and K9


def _empty_offers():
    return abi.OffersSoA(n=0, hostname_id=np.zeros(1, np.int32), name_rank=np.zeros(1, np.int32), cpus=np.zeros(1),
                         mem=np.zeros(1), run_cpus=np.zeros(1), run_mem=np.zeros(1), run_count=np.zeros(1, np.int32),
                         n_attr_cols=0)


def _random_case(rng, J=300, U=7, grid=True):
    cpus = rng.choice([0.5, 1.0, 2.0, 4.0] if grid else [0.1, 0.3, 1.0, 2.7], J)
    mem = rng.choice([256.0, 1024.0, 4096.0] if grid else [100.1, 1000.3, 333.3], J)
    gpus = rng.choice([0.0, 0.0, 1.0], J)
    user = rng.integers(0, U, J).astype(np.int32)
    jobs = abi.JobsSoA(n=J, user=user, cpus=cpus, mem=mem, gpus=gpus,
                       allowed=(rng.random(J) < 0.9).astype(np.uint8), plugin_accept=(rng.random(J) < 0.95).astype(np.uint8))
    quota = {"count": rng.integers(5, 60, U).astype(float), "cpus": rng.choice([20.0, 60.0, 1e9], U),
             "mem": rng.choice([20000.0, 1e12], U), "gpus": rng.choice([3.0, 1e9], U)}
    usage = {"count": rng.integers(0, 5, U).astype(float), "cpus": rng.choice([0.0, 1.5, 3.1], U),
             "mem": rng.choice([0.0, 512.0, 777.7], U), "gpus": rng.choice([0.0, 1.0], U)}
    tokens = rng.integers(1, 40, U).astype(np.int32)
    users = abi.make_users(U, quota=quota, usage=usage, tokens=tokens)
    return jobs, users


@pytest.mark.parametrize("seed", range(6))
def test_ref_random_against_oracle(oracle, seed):
    rng = np.random.default_rng(seed)
    jobs, users = _random_case(rng, grid=seed % 2 == 0)
    queue = rng.permutation(jobs.n).astype(np.int32)[: jobs.n - 20]
    for enforce, pq, nc in itertools.product((0, 1), (None, {"count": 120, "cpus": 150.0, "mem": 1e6, "gpus": 30}),
                                             (1, 50, 1000)):
        prm = traces.match_params(nc, enforce_rate_limit=enforce)
        pool_q = abi.make_pool_quota(pq) if pq else None
        want = oracle.match(queue, jobs, _empty_offers(), users, prm, pool_quota=pool_q)["considerable"]
        got = RefEngine.match(queue, jobs, None, users, prm, pool_quota=pool_q)["considerable"]
        assert got.tolist() == list(want), (enforce, pq, nc)


# ---- GPU helpers -------------------------------------------------------------------------------------------
def _params(nc, enforce=0, quota_only=0, source=abi.USAGE_GIVEN, consume=0):
    return abi.ConsiderableParams(int(nc), int(enforce), int(quota_only), int(source), int(consume))


def _with(users, **over):
    kw = {n: users.col(n) if users.col(n) is not None else None for n, t in users._fields_ if t is not C.c_int32}
    kw.update(over)
    return abi.UserTable(n_users=users.n_users, **kw)


def _usage_users(users, usage):
    """users with usage_* = usage ({key: array})."""
    return _with(users, **{f: np.asarray(usage[k], np.float64) for f, k in zip(USAGE_FIELDS, KEYS)})


def _quota_users(base, rng):
    """The trace's users with quotas and tokens that cut: some users' queues are filtered, some not at all."""
    U = base.n_users
    big = np.finfo(np.float64).max
    q = {"count": np.where(rng.random(U) < 0.3, big, rng.integers(20, 200, U).astype(float)),
         "cpus": np.where(rng.random(U) < 0.3, big, rng.choice([40.0, 150.0, 600.0], U)),
         "mem": np.where(rng.random(U) < 0.5, big, rng.choice([1e5, 6e5], U)),
         "gpus": np.where(rng.random(U) < 0.5, big, rng.choice([0.0, 4.0], U))}
    return _with(base, **{f: q[k] for f, k in zip(QUOTA_FIELDS, KEYS)},
                 tokens=rng.integers(3, 80, U).astype(np.int32))


POOL_Q = {"count": 900.0, "cpus": 3000.0, "mem": 1e7, "gpus": 1e9}


class Pool:
    """A resident handle (`gpu`), a host-table handle (`ref`) and the model of the rows."""

    def __init__(self, t, users):
        from test_state_resident import Model
        self.t, self.users, self.offers = t, users, t["offers"]
        self.gpu, self.ref, self.m = GpuEngine(pool_name="considerable"), GpuEngine(pool_name="host"), Model()
        self.queue, self.gone = [], set()

    def close(self):
        self.gpu.close()
        self.ref.close()

    def apply(self, up=(), rm=(), run_up=(), run_rm=(), reset=False):
        from test_state_resident import delta
        self.gpu.state_apply(delta(reset, up, rm, run_up, run_rm))
        self.m.apply(up, rm, run_up, run_rm, reset)
        self.gone |= set(rm) | {j for j, _ in up}

    def rank(self, **kw):
        q = self.gpu.state_rank(self.users, **kw)
        self.queue, self.gone = q.tolist(), set()
        return q

    def usage(self):
        return self.gpu.state_usage(self.users.n_users)["user"]

    def host_considerable(self, prm, usage, pool_q=None):
        """cook_match on the model's tables, the live queue, an empty offer table; and considerable_ref."""
        _, _, jobs, jid = self.m.tables()
        pos = {j: i for i, j in enumerate(jid.tolist())}
        ranked = np.array([pos[j] for j in self.queue if j not in self.gone], np.int32)
        J = jobs.n
        ones = np.ones(J, np.uint8)
        al = ones if prm.quota_only else np.array([self.m.pend[j]["allowed"] for j in jid.tolist()], np.uint8)
        pa = ones if prm.quota_only else np.array([self.m.pend[j]["plugin_accept"] for j in jid.tolist()], np.uint8)
        plain = abi.JobsSoA(n=J, user=jobs.col("user"), cpus=jobs.col("cpus"), mem=jobs.col("mem"),
                            gpus=jobs.col("gpus"), allowed=al, plugin_accept=pa)
        users = _usage_users(self.users, usage)
        if len(ranked) == 0:
            return [], []
        mp = traces.match_params(prm.num_considerable, enforce_rate_limit=prm.enforce_rate_limit)
        pq = abi.make_pool_quota(pool_q) if pool_q else None
        want = self.ref.match(ranked, plain, _empty_offers(), users, mp, pool_quota=pq)["considerable"]
        quota = {k: self.users.col(f) for k, f in zip(KEYS, QUOTA_FIELDS)}
        gpus = jobs.col("gpus") if jobs.col("gpus") is not None else np.zeros(J)   # an all-zero column is absent
        ref = CR.considerable(ranked.tolist(), jobs.col("user"), jobs.col("cpus"), jobs.col("mem"), gpus,
                              quota, usage, prm.num_considerable, tokens=self.users.col("tokens"),
                              enforce_rate_limit=prm.enforce_rate_limit, pool_quota=pool_q, allowed=al,
                              plugin_accept=pa)
        return jid[want].tolist(), jid[np.array(ref, np.int64)].tolist() if ref else []


def _combos():
    return list(itertools.product((0, 1), (abi.USAGE_GIVEN, abi.USAGE_DERIVED, abi.USAGE_LAST_MATCH), (0, 1),
                                  (None, POOL_Q), (1, 1000, -1)))


def _match_derived(p, nc=400):
    """A derived match on the resident handle; returns it and the usage it read (cook_state_usage before it)."""
    usage = p.usage()
    users = _with(p.users, **{f: None for f in USAGE_FIELDS})
    offers = _with_offers(p.offers)
    got = p.gpu.state_match(offers, users, traces.match_params(nc), derived=True)
    return got, usage


def _with_offers(o):
    kw = {n: o.col(n) for n, t in o._fields_ if t is not C.c_int32 and o.col(n) is not None}
    for f in ("run_cpus", "run_mem", "run_count"):
        kw.pop(f, None)
    return abi.OffersSoA(n=o.n, n_attr_cols=o.n_attr_cols, **kw)


def _given_usage(p, rng):
    """An arbitrary usage table (the GIVEN source reads whatever the caller passes)."""
    U = p.users.n_users
    return {"count": rng.integers(0, 30, U).astype(float), "cpus": rng.choice([0.0, 4.5, 12.0], U),
            "mem": rng.choice([0.0, 4096.0, 9000.5], U), "gpus": np.zeros(U)}


def _check(p, prm, usage, pool_q, given=None):
    users = _usage_users(p.users, given) if given is not None else p.users
    if prm.usage_source != abi.USAGE_GIVEN:
        users = _with(p.users, **{f: None for f in USAGE_FIELDS})
    pq = abi.make_pool_quota(pool_q) if pool_q else None
    got = p.gpu.state_considerable(users, prm, pool_quota=pq).tolist()
    want, ref = p.host_considerable(prm, given if given is not None else usage, pool_q)
    assert got == want, "resident considerable != cook_match on host tables"
    assert got == ref, "resident considerable != considerable_ref"
    return got


# ---- GPU ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["c2", "c2_offgrid", "c3"])
def test_churn_equivalence(kind):
    from test_state_resident import _c2, _c3, _churn, pool_rows
    t = {"c2": lambda: _c2(11), "c2_offgrid": lambda: _c2(12, cpus=(0.1, 0.5, 1.0, 2.7)), "c3": lambda: _c3(13)}[kind]()
    rng = np.random.default_rng(7)
    p = Pool(t, _quota_users(t["users"], rng))
    combos = _combos()
    try:
        pend, run = pool_rows(t)
        items = sorted(pend.items())
        cut = int(len(items) * 0.85)
        reserve = items[cut:]
        p.apply(up=items[:cut], run_up=list(run.values()), reset=True)
        t_next = [10 ** 9]
        k = 0
        for batch in range(9):
            p.rank()
            got, last = _match_derived(p)
            now = p.usage()
            given = _given_usage(p, rng)
            for _ in range(8):
                qo, src, enf, pq, nc = combos[k % len(combos)]
                k += 1
                n_live = len([j for j in p.queue if j not in p.gone])
                prm = _params(n_live + 37 if nc < 0 else nc, enf, qo, src)
                usage = {abi.USAGE_GIVEN: given, abi.USAGE_DERIVED: now, abi.USAGE_LAST_MATCH: last}[src]
                _check(p, prm, usage, pq, given=given if src == abi.USAGE_GIVEN else None)
            launched = [int(j) for j, a in zip(got["considerable"], got["assign"]) if a >= 0][:40]
            up, rm, run_up, run_rm = _churn(p, rng, reserve, t_next, launched)
            p.apply(up, rm, run_up, run_rm)
            # between rank and the next calls the queue loses what the churn removed or replaced
            prm = _params(1000, 1, 0, abi.USAGE_DERIVED)
            _check(p, prm, p.usage(), POOL_Q)
        assert k >= len(combos)
    finally:
        p.close()


@pytest.mark.gpu
def test_layout_independence():
    from test_state_resident import _c2, pool_rows
    t = _c2(21, cpus=(0.1, 0.5, 1.0, 2.0))
    rng = np.random.default_rng(4)
    users = _quota_users(t["users"], rng)
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    a, b = Pool(t, users), Pool(t, users)
    try:
        a.apply(up=items, run_up=list(run.values()))
        junk = [(10 ** 11 + i, items[i][1]) for i in range(500)]
        b.apply(up=junk)
        b.apply(rm=[j for j, _ in junk])
        perm = rng.permutation(len(items))
        rr = list(run.values())
        b.apply(up=[items[i] for i in perm], run_up=[rr[i] for i in rng.permutation(len(rr))])
        assert np.array_equal(a.rank(), b.rank())
        for qo, src, enf, pq in itertools.product((0, 1), (abi.USAGE_GIVEN, abi.USAGE_DERIVED), (0, 1), (None, POOL_Q)):
            prm = _params(1000, enf, qo, src)
            u = users if src == abi.USAGE_GIVEN else _with(users, **{f: None for f in USAGE_FIELDS})
            q = abi.make_pool_quota(pq) if pq else None
            assert np.array_equal(a.gpu.state_considerable(u, prm, q), b.gpu.state_considerable(u, prm, q))
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_autoscaling_after_match():
    from test_state_resident import _c2, pool_rows
    t = _c2(31)
    rng = np.random.default_rng(9)
    p = Pool(t, _quota_users(t["users"], rng))
    try:
        pend, run = pool_rows(t)
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.rank()
        got, usage = _match_derived(p, nc=300)
        placed = [(int(j), int(a)) for j, a in zip(got["considerable"], got["assign"]) if a >= 0]
        assert placed
        _, _, jobs, jid = p.m.tables()
        pos = {j: i for i, j in enumerate(jid.tolist())}
        hid = p.offers.col("hostname_id")
        p.gpu.state_launch([j for j, _ in placed], [5 * 10 ** 9 + i for i in range(len(placed))],
                           np.full(len(placed), 1_700_000_000_000, np.int64), [int(hid[a]) for _, a in placed])
        gone = {j for j, _ in placed}
        queue_after = np.array([pos[j] for j in p.queue if j not in gone], np.int32)
        n_cons = len(got["considerable"])
        unmatched = n_cons - len(placed)
        users = _usage_users(p.users, usage)
        for max_jobs in (1, 250, 5000):
            want = cycle.autoscalable_jobs(p.ref, queue_after, jobs, users, number_considerable=n_cons,
                                           number_unmatched=unmatched, max_jobs_for_autoscaling=max_jobs,
                                           pool_quota=abi.make_pool_quota(POOL_Q))
            n = cycle.max_jobs_for_autoscaling_scaled(n_cons, unmatched, max_jobs, 1.0)
            res = p.gpu.state_considerable(_with(p.users, **{f: None for f in USAGE_FIELDS}),
                                           _params(n, quota_only=1, source=abi.USAGE_LAST_MATCH),
                                           abi.make_pool_quota(POOL_Q))
            assert res.tolist() == [int(jid[i]) for i in want]
            twin = cycle.autoscalable_jobs_resident(p.gpu, p.users, number_considerable=n_cons,
                                                    number_unmatched=unmatched, max_jobs_for_autoscaling=max_jobs,
                                                    pool_quota=abi.make_pool_quota(POOL_Q))
            assert twin == res.tolist()
    finally:
        p.close()


def _hosted(run, hid):
    """The running rows, each on a host of the offer table."""
    return [dict(r, host=int(hid[i % len(hid)])) for i, r in enumerate(run.values())]


def _apply_hosted(p, items, run_rows):
    from test_state_resident import jobs_soa, tasks_soa
    pj, pp, jid = jobs_soa(items)
    p.gpu.state_apply(abi.make_delta(reset=True, pending=pj, pending_priority=pp, pending_job_id=jid,
                                     running=tasks_soa(run_rows),
                                     running_hostname_id=np.array([r["host"] for r in run_rows], np.int32)))
    p.m.apply(items, (), run_rows, (), True)


@pytest.mark.gpu
def test_consume():
    from test_state_derived import host_inputs
    from test_state_resident import _c2, pool_rows
    t = _c2(41)
    rng = np.random.default_rng(2)
    users = _quota_users(t["users"], rng)
    p, twin = Pool(t, users), Pool(t, users)
    try:
        pend, run = pool_rows(t)
        items = sorted(pend.items())
        rows = _hosted(run, p.offers.col("hostname_id"))
        for x in (p, twin):
            _apply_hosted(x, items, rows)
            x.rank()
        nu = users.n_users
        hn = p.offers.col("hostname_id")
        usage0 = p.gpu.state_usage(nu, hn)
        cot0 = p.gpu.state_cotasks(4)
        du = _with(users, **{f: None for f in USAGE_FIELDS})
        first = p.gpu.state_considerable(du, _params(200, source=abi.USAGE_DERIVED, consume=1)).tolist()
        assert len(first) == 200
        p.gone |= set(first)
        # the rows stay live and unchanged
        usage1 = p.gpu.state_usage(nu, hn)
        for k in ("pool", "run_cpus", "run_mem", "run_count"):
            assert np.array_equal(usage0[k], usage1[k]), k
        for k in KEYS:
            assert np.array_equal(usage0["user"][k], usage1["user"][k])
        for x, y in zip(cot0, p.gpu.state_cotasks(4)):
            assert np.array_equal(x, y)
        # a second call takes the next jobs: the host tables' queue leaves out the consumed ones
        second = _check(p, _params(150, source=abi.USAGE_DERIVED, consume=1), p.usage(), None)
        assert len(second) == 150 and not set(second) & set(first)
        p.gone |= set(second)
        taken = set(first) | set(second)
        # a patch does not bring an entry back
        p.gpu.state_patch(first[:50], allowed=np.ones(50, np.uint8))
        third = _check(p, _params(1000, source=abi.USAGE_DERIVED), p.usage(), POOL_Q)
        assert not set(third) & taken
        # the twin removes the taken jobs after the same rank: its queue is the original one minus them
        twin.apply(rm=sorted(taken))
        # match and rebalance leave them out, as the twin and the host tables do
        prm = traces.match_params(500)
        m = p.gpu.state_match(_with_offers(p.offers), du, prm, derived=True)
        mt = twin.gpu.state_match(_with_offers(p.offers), du, prm, derived=True)
        for k in ("considerable", "assign", "ports", "fail"):
            assert np.array_equal(m[k], mt[k]), k
        _, _, jobs, jid = p.m.tables()
        pos = {j: i for i, j in enumerate(jid.tolist())}
        ranked = np.array([pos[j] for j in p.queue if j not in p.gone], np.int32)
        ho, hu, _ = host_inputs(list(p.m.run.values()), p.offers, users, None)
        want = p.ref.match(ranked, jobs, ho, hu, prm)
        assert np.array_equal(m["considerable"], jid[want["considerable"]])
        assert np.array_equal(m["assign"], want["assign"])
        hosts = _hosts_of(p)
        rp = abi.RebalanceParams(20, 0.0, 1e9, 0)
        for derived in (False, True):
            rb = p.gpu.state_rebalance(hosts, users, rp, derived=derived)
            assert rb == twin.gpu.state_rebalance(hosts, users, rp, derived=derived)
            assert not {d["job_id"] for d in rb} & taken
        # a later considerable call equals the twin's
        for src in (abi.USAGE_DERIVED, abi.USAGE_LAST_MATCH):
            prm = _params(800, 1, 0, src)
            assert np.array_equal(p.gpu.state_considerable(du, prm), twin.gpu.state_considerable(du, prm))
        # launching a consumed job works
        tids = [7 * 10 ** 9 + i for i in range(3)]
        p.gpu.state_launch(first[:3], tids, np.full(3, 1, np.int64), [int(hn[0])] * 3)
        new_rows = [dict(user=p.m.pend[j]["user"], priority=p.m.pend[j]["priority"], start_time=1, task_id=tid, job_id=j,
                         cpus=p.m.pend[j]["cpus"], mem=p.m.pend[j]["mem"], gpus=p.m.pend[j]["gpus"], host=int(hn[0]))
                    for j, tid in zip(first[:3], tids)]
        p.m.apply((), first[:3], new_rows, ())
        u2 = p.gpu.state_usage(nu)["user"]
        assert sum(u2["count"]) == sum(usage0["user"]["count"]) + 3
        # the next rank brings back every consumed job still pending
        q = p.rank()
        assert (taken - set(first[:3])) <= set(q.tolist())
        assert not set(first[:3]) & set(q.tolist())
        _check(p, _params(len(q) + 10, source=abi.USAGE_DERIVED), p.usage(), None)
    finally:
        p.close()
        twin.close()


def _hosts_of(p):
    """A host table over the offers (every running row's host must be listed)."""
    o = p.offers
    hid = list(o.col("hostname_id"))
    extra = sorted({int(r["host"]) for r in p.m.run.values() if "host" in r} - set(int(h) for h in hid))
    codes = np.array(hid + extra, np.int32)
    H = len(codes)
    return abi.HostTable(n=H, hostname_id=codes, name_rank=np.argsort(np.argsort(codes)).astype(np.int32),
                         has_spare=np.ones(H, np.uint8), spare_cpus=np.full(H, 4.0), spare_mem=np.full(H, 8192.0),
                         spare_gpus=np.zeros(H), n_attr_cols=0)


@pytest.mark.gpu
def test_plan_untouched():
    from test_state_resident import _c2, pool_rows
    t = _c2(51)
    p = Pool(t, _quota_users(t["users"], np.random.default_rng(1)))
    try:
        pend, run = pool_rows(t)
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.rank()
        got, _ = _match_derived(p)
        n = len(got["considerable"])
        k = np.arange(min(n, 32), dtype=np.int32)
        fw = p.gpu.match_failures(k)
        xw = p.gpu.exchange_usage(p.users.n_users)
        du = _with(p.users, **{f: None for f in USAGE_FIELDS})
        for src in (abi.USAGE_GIVEN, abi.USAGE_DERIVED, abi.USAGE_LAST_MATCH):
            p.gpu.state_considerable(p.users if src == abi.USAGE_GIVEN else du, _params(2000, 1, 0, src),
                                     abi.make_pool_quota(POOL_Q))
            assert p.gpu.match_failures(k) == fw
            assert np.array_equal(p.gpu.exchange_usage(p.users.n_users), xw)
    finally:
        p.close()


@pytest.mark.gpu
def test_offensive():
    from test_state_resident import _c2, pool_rows
    t = _c2(61)
    base = t["users"]
    pend, run = pool_rows(t)
    items = sorted(pend.items())
    a, b = Pool(t, base), Pool(t, base)
    try:
        for p in (a, b):
            p.apply(up=items, run_up=list(run.values()))
        _, pending, jobs, jid = a.m.tables()
        running = a.m.tables()[0]
        cpus, mem = jobs.col("cpus"), jobs.col("mem")
        caps = (float(np.quantile(mem, 0.8)), float(np.quantile(cpus, 0.9)))
        # quotas above the running usage, that cut the queue part way (the pool quota counts the running tasks)
        ru = a.gpu.state_usage(a.users.n_users)["pool"]
        quotas = [(None, None, None),
                  ({"count": ru[0] + 400, "cpus": ru[1] + 900.0, "mem": 1e12, "gpus": 1e9}, None, None),
                  (None, {"count": 800.0, "cpus": 1e9, "mem": 1e12, "gpus": 1e9}, np.array([100.0, 200.0, 4e5, 0.0]))]
        for pq, gq, gu in quotas:
            for filt in (1, 0):
                prm = abi.RankParams(100, filt, caps[0], caps[1])
                kw = dict(pool_quota=abi.make_pool_quota(pq) if pq else None,
                          group_quota=abi.make_pool_quota(gq) if gq else None, group_usage=gu, params=prm)
                q, off = a.gpu.state_rank(a.users, offensive=True, **kw)
                qb = b.gpu.state_rank(b.users, **kw)
                st_a, st_b = a.gpu.last_stats(abi.PHASE_RANK), b.gpu.last_stats(abi.PHASE_RANK)
                assert np.array_equal(q, qb)
                assert st_a["h2d_bytes"] == st_b["h2d_bytes"]
                assert st_a["d2h_bytes"] == st_b["d2h_bytes"] + 4 + 8 * len(off)
                # the order without the offensive filter, its offensive jobs
                host = a.ref.rank(running if running.n else None, pending, a.users,
                                  params=abi.RankParams(100, 0, 0.0, 0.0),
                                  **{k: v for k, v in kw.items() if k != "params"})
                order = host["ranked"].tolist()
                want = CR.offensive(order, cpus, mem, caps[0], caps[1]) if filt else []
                assert off.tolist() == [int(jid[i]) for i in want]
                if filt:
                    assert 0 < len(off) and len(q) > 0
                    keep = jid[np.array([i for i in order if i not in set(want)], np.int64)]
                    assert np.array_equal(q, keep)
        # the matches of the two handles agree after the offensive rank
        prm = traces.match_params(500)
        ma = a.gpu.state_match(a.offers, a.users, prm)
        mb = b.gpu.state_match(b.offers, b.users, prm)
        for k in ("considerable", "assign"):
            assert np.array_equal(ma[k], mb[k])
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_offensive_quota_cuts_first():
    """A job cut by the pool quota first is not listed, as filter-offensive-jobs only sees what the quota left."""
    e = GpuEngine(pool_name="offensive-quota")
    try:
        rows = [(i + 1, dict(user=0, priority=50, cpus=c, mem=m)) for i, (c, m) in
                enumerate([(1.0, 100.0), (1.0, 5000.0), (1.0, 100.0), (1.0, 9000.0), (1.0, 100.0)])]
        e.state_apply(_resident_delta(rows))
        users = abi.make_users(1)
        prm = abi.RankParams(100, 1, 1000.0, 10.0)
        q, off = e.state_rank(users, params=prm, offensive=True)
        assert q.tolist() == [1, 3, 5] and off.tolist() == [2, 4]
        q, off = e.state_rank(users, pool_quota=abi.make_pool_quota({"count": 3, "cpus": 1e9, "mem": 1e9, "gpus": 1e9}),
                              params=prm, offensive=True)
        assert q.tolist() == [1, 3] and off.tolist() == [2]   # job 4 fell to the pool quota before the offensive test
    finally:
        e.close()


def _resident_delta(rows):
    """A delta of pending rows [(job id, {user, priority, cpus, mem[, gpus]})]."""
    n = len(rows)
    jobs = abi.JobsSoA(n=n, user=np.array([r["user"] for _, r in rows], np.int32),
                       cpus=np.array([r["cpus"] for _, r in rows], float), mem=np.array([r["mem"] for _, r in rows], float),
                       gpus=np.array([r.get("gpus", 0.0) for _, r in rows], float))
    return abi.make_delta(reset=True, pending=jobs, pending_priority=np.array([r["priority"] for _, r in rows], np.int32),
                          pending_job_id=np.array([j for j, _ in rows], np.int64))


@pytest.mark.gpu
def test_filter_offensive_jobs_reference():
    """test-filter-offensive-jobs (reference scheduler test :857-888) through resident deltas: with caps of 10 GB
    and 20 cpus, the jobs of 12 GB or 30 cpus go to the channel and the rest stay, in order."""
    e = GpuEngine(pool_name="offensive-ref")
    try:
        shapes = [(10.0, 10 * 1024.0), (30.0, 10 * 1024.0), (10.0, 12 * 1024.0), (5.0, 1024.0)]
        rows = [(100 + i, dict(user=0, priority=50 - i, cpus=c, mem=m)) for i, (c, m) in enumerate(shapes)]
        e.state_apply(_resident_delta(rows))
        q, off = e.state_rank(abi.make_users(1), params=abi.RankParams(100, 1, 10 * 1024.0, 20.0), offensive=True)
        assert q.tolist() == [100, 103]
        assert off.tolist() == [101, 102]
    finally:
        e.close()


@pytest.mark.gpu
def test_k14_resident(monkeypatch):
    """K14's 17 answers through the resident state: one user, job ids ascending in queue order, GIVEN usage."""
    import considerable_golden_cases as K14
    monkeypatch.setattr(K14, "check_k9", lambda eng: None)   # K9 has several users: its queue is not job order

    class Resident:
        def __init__(self):
            self.e = GpuEngine(pool_name="k14")

        def match(self, ranked_idx, jobs, offers, users, params, groups=None, pool_quota=None, max_ports=0):
            J = jobs.n
            nu = users.n_users
            rows = [(int(j) + 1, dict(user=int(jobs.col("user")[j]), priority=50 + J - int(j),
                                      cpus=float(jobs.col("cpus")[j]), mem=float(jobs.col("mem")[j]),
                                      gpus=float(jobs.col("gpus")[j]))) for j in range(J)]
            self.e.state_apply(_resident_delta(rows))
            self.e.state_patch(np.arange(1, J + 1), plugin_accept=jobs.col("plugin_accept"))
            q = self.e.state_rank(abi.make_users(nu))
            assert q.tolist() == list(range(1, J + 1))   # priorities put the queue in job order
            got = self.e.state_considerable(users, _params(params.num_considerable, params.enforce_rate_limit),
                                            pool_quota)
            return {"considerable": np.array([int(j) - 1 for j in got], np.int32)}

    r = Resident()
    try:
        K14.check_all(r)
    finally:
        r.e.close()


@pytest.mark.gpu
def test_errors_and_transfers():
    from test_state_resident import _c2, pool_rows
    t = _c2(71)
    users = _quota_users(t["users"], np.random.default_rng(3))
    p = Pool(t, users)
    try:
        du = _with(users, **{f: None for f in USAGE_FIELDS})
        with pytest.raises(CookError):   # no rank yet
            p.gpu.state_considerable(users, _params(10))
        pend, run = pool_rows(t)
        p.apply(up=sorted(pend.items()), run_up=list(run.values()))
        p.rank()
        U = users.n_users

        def unconsumed():
            got = p.gpu.state_considerable(users, _params(100000))
            return got.tolist()

        before = unconsumed()
        bad = [
            (users, _params(10, source=7)),                                    # unknown source
            (du, _params(10, source=abi.USAGE_GIVEN, consume=1)),               # GIVEN without usage
            (_with(users, quota_mem=None), _params(10, consume=1)),            # no quota column
            (users, _params(10, source=abi.USAGE_LAST_MATCH, consume=1)),      # no match yet
            (abi.make_users(1), _params(10, consume=1)),                        # a user code >= n_users
        ]
        out = np.full(16, -7, np.int64)
        n = C.c_int32(-5)
        for u, prm in bad:
            rc = p.gpu.lib.cook_state_considerable(p.gpu.pool, C.byref(u), None, C.byref(prm), abi.ptr(out, abi.P_I64),
                                                   C.byref(n))
            assert rc == abi.COOK_E_BADARG
            assert (out == -7).all() and n.value == -5
        rc = p.gpu.lib.cook_state_considerable(p.gpu.pool, C.byref(users), None, C.byref(_params(10)), None, C.byref(n))
        assert rc == abi.COOK_E_BADARG
        # LAST_MATCH with another n_users
        _match_derived(p)
        wide = abi.make_users(U + 3)
        rc = p.gpu.lib.cook_state_considerable(p.gpu.pool, C.byref(wide), None,
                                               C.byref(_params(10, source=abi.USAGE_LAST_MATCH, consume=1)),
                                               abi.ptr(out, abi.P_I64), C.byref(n))
        assert rc == abi.COOK_E_BADARG and n.value == -5
        assert unconsumed() == before
        # nothing to do: no device work, zero statistics
        assert p.gpu.state_considerable(users, _params(0)).tolist() == []
        assert all(v == 0 for v in p.gpu.last_stats(abi.PHASE_CONSIDERABLE).values())
        # transfers
        tok = users.col("tokens")
        for src, enf in itertools.product((abi.USAGE_GIVEN, abi.USAGE_DERIVED, abi.USAGE_LAST_MATCH), (0, 1)):
            u = users if src == abi.USAGE_GIVEN else du
            got = p.gpu.state_considerable(u, _params(700, enf, 0, src), abi.make_pool_quota(POOL_Q))
            st = p.gpu.last_stats(abi.PHASE_CONSIDERABLE)
            want_up = 32 * U + (4 * U if enf and tok is not None else 0) + (32 * U if src == abi.USAGE_GIVEN else 0)
            assert st["h2d_bytes"] == want_up, (src, enf)
            assert st["d2h_bytes"] == 4 + 4 + 8 * len(got), (src, enf)
            assert st["n_launches"] > 0
        # the offensive rank's capacity
        off = np.zeros(4, np.int64)
        rq, rn, no = np.zeros(len(pend) + 1, np.int64), C.c_int32(0), C.c_int32(-3)
        gu = np.zeros(4)
        pq = abi.make_pool_quota(None)
        rc = p.gpu.lib.cook_state_rank_offensive(p.gpu.pool, C.byref(users), C.byref(pq), C.byref(pq),
                                                 abi.ptr(gu, abi.P_F64), C.byref(abi.RankParams(100, 1, 1.0, 1.0)),
                                                 abi.ptr(rq, abi.P_I64), C.byref(rn), abi.ptr(off, abi.P_I64), 4,
                                                 C.byref(no))
        assert rc == abi.COOK_E_BADARG
    finally:
        p.close()
