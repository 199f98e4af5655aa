"""-m gpu: Cook's hard constraints on the paths the generated traces do not reach, built by hand and
compared with the CPU oracle.

  explainer, large groups   cook_match_failures with attribute-equals and balanced groups whose
                            running cotasks (about 70) put the deciding values after position 64,
                            plus members placed earlier in the same cycle;
  explainer, check order    a VM table where VM i fails checks i and i + 1 of Cook's order: every
                            VM must be counted under its first failing check;
  rebalancer, scalar path   a pending job in more groups than the prepared group table holds, and a
                            group whose cotasks carry more distinct values than it holds.
"""
import numpy as np
import pytest

from cook_b200 import abi, traces

pytestmark = pytest.mark.gpu

FIRST = 2   # counts[FIRST + i]: VMs whose first failing hard constraint was i (COOK_FAILC_FIRST_CONSTRAINT)


def _users(n):
    return abi.make_users(n, div_mem=np.full(n, 1e6), div_cpus=np.full(n, 1e3), div_gpus=np.ones(n))


def _offers(O, attr, **kw):
    """O big, empty VMs with hostname = index = name rank; attr: [n_cols][O] value ids."""
    attr = np.asarray(attr, np.int32)
    return abi.OffersSoA(n=O, hostname_id=np.arange(O, dtype=np.int32), name_rank=np.arange(O, dtype=np.int32),
                         cpus=np.full(O, 64.0), mem=np.full(O, 65536.0), run_cpus=np.zeros(O), run_mem=np.zeros(O),
                         run_count=np.zeros(O, np.int32), n_attr_cols=len(attr), attr=attr.reshape(-1), **kw)


def _jobs(J, group_lists, **kw):
    off, idx = abi.csr(group_lists)
    return abi.JobsSoA(n=J, user=np.zeros(J, np.int32), cpus=np.ones(J), mem=np.full(J, 16.0), gpus=np.zeros(J),
                       ports=np.zeros(J, np.int32), allowed=np.ones(J, np.uint8), plugin_accept=np.ones(J, np.uint8),
                       group_off=off, group_idx=idx, **kw)


def _groups(kinds, cols, minimum, cot_hosts, cot_vals):
    coff, chost = abi.csr(cot_hosts)
    _, cval = abi.csr(cot_vals)
    return abi.Groups(n_groups=len(kinds), kind=np.array(kinds, np.int32), attr_col=np.array(cols, np.int32),
                      minimum=np.array(minimum, np.int32), cot_off=coff, cot_hostname_id=chost, cot_attr_val=cval)


def _failures(gpu, oracle, jobs, offers, groups, ks, host_lifetime_mins=0):
    ranked = np.arange(jobs.n, dtype=np.int32)
    prm = traces.match_params(jobs.n, host_lifetime_mins=host_lifetime_mins)
    users = _users(1)
    mg = gpu.match(ranked, jobs, offers, users, prm, groups=groups)
    mo = oracle.match(ranked, jobs, offers, users, prm, groups=groups)
    assert np.array_equal(mg["assign"], mo["assign"])
    fg = gpu.match_failures(ks)
    fo = oracle.match_failures(ranked, jobs, offers, users, prm, ks, groups=groups)
    return fg, fo, mo["assign"]


def large_group_case():
    """12 VMs whose attribute is 1, 2, 3, 1, 2, 3, ...; 60 one-cpu jobs alternate between
    group 0, attribute-equals, with 66 cotasks on value 1 and then 4 on value 2, and
    group 1, balanced (minimum 0), with 33 cotasks on value 1, 33 on value 2 and then 4 on value 3."""
    O, J = 12, 60
    offers = _offers(O, [[1 + v % 3 for v in range(O)]])
    jobs = _jobs(J, [[j % 2] for j in range(J)])
    groups = _groups([abi.GROUP_ATTR_EQUALS, abi.GROUP_BALANCED], [0, 0], [0, 0],
                     [list(range(100, 170)), list(range(200, 270))],
                     [[1] * 66 + [2] * 4, [1] * 33 + [2] * 33 + [3] * 4])
    return jobs, offers, groups


def test_explainer_groups_beyond_64_known_values(gpu, oracle):
    jobs, offers, groups = large_group_case()
    ks = np.array([0, 1, 2, 3] + list(range(40, 60)), np.int32)
    fg, fo, assign = _failures(gpu, oracle, jobs, offers, groups, ks)
    assert (assign >= 0).all()
    assert fg == fo
    for k, f in zip(ks, fo):
        if k % 2 == 0:   # attribute-equals: value 2, known only past position 64, passes; value 3 fails
            assert f["counts"][FIRST + 10] == 4 and f["n_passed"] == 8, (k, f)
    # balanced: at job 1's turn values 1 and 2 are the most frequent (33), only the 4 VMs of value 3 pass;
    # by job 59's turn the 29 earlier members, all on value 3, have evened the group out
    assert fo[1]["counts"][FIRST + 9] == 8 and fo[1]["n_passed"] == 4, fo[1]
    assert fo[-1]["counts"][FIRST + 9] == 0 and fo[-1]["n_passed"] == 12, fo[-1]


def check_order_case():
    """One job against 12 VMs: VM i (i < 10) fails hard constraints i and i + 1 of Cook's order, VM 10
    fails attribute-equals (10) only, VM 11 passes everything.  The job is in three groups, in the
    order unique (8), balanced (9), attribute-equals (10)."""
    O = 12
    lifetime, t_end = 1, 10**12                        # a host started at 1 s dies long before t_end
    location = np.zeros(O, np.int32); location[0] = 1                              # 0 checkpoint locality
    host_start = np.full(O, -1, np.int64); host_start[[0, 1]] = 1                  # 1 estimated completion
    col1 = np.ones(O, np.int32); col1[[1, 2]] = 2                                  # 2 user-defined attribute
    disk = [[100.0] for _ in range(O)]; disk[2] = disk[3] = [10.0]                 # 3 disk (every VM is k8s)
    gpu_m = [[0] if v in (3, 4) else [] for v in range(O)]                          # 4 gpu host: a gpu-less job
    novel = [4, 5]                                                                  # 5 novel host
    max_tasks = np.full(O, -1, np.int32); max_tasks[[5, 6]] = 1                     # 6 max tasks per host
    reserved = np.zeros(O, np.uint8); reserved[[6, 7]] = 1                          # 7 reservation
    unique_cot = [7, 8]                                                             # 8 unique: cotask hosts
    col2 = np.full(O, 2, np.int32); col2[[8, 9]] = 1                                # 9 balanced: {1, 1, 2}
    col3 = np.ones(O, np.int32); col3[[9, 10]] = 2                                  # 10 attribute-equals: {1}
    g_off, g_model = abi.csr(gpu_m)
    _, g_count = abi.csr([[1.0] * len(m) for m in gpu_m], np.float64)
    d_off, d_type = abi.csr([[0] for _ in range(O)])
    _, d_space = abi.csr(disk, np.float64)
    offers = _offers(O, [np.zeros(O, np.int32), col1, col2, col3], is_k8s=np.ones(O, np.uint8), location=location,
                     gpu_off=g_off, gpu_model=g_model, gpu_count=g_count, disk_off=d_off, disk_type=d_type,
                     disk_space=d_space, max_tasks=max_tasks, num_tasks=np.ones(O, np.int32),
                     host_start_time=host_start, reserved=reserved)
    a_off, a_col = abi.csr([[1]])
    _, a_val = abi.csr([[1]])
    n_off, n_host = abi.csr([novel])
    jobs = _jobs(1, [[0, 1, 2]], ckpt_location=np.zeros(1, np.int32), est_end_ms=np.array([t_end], np.int64),
                 attr_off=a_off, attr_col=a_col, attr_val=a_val, disk_request=np.array([50.0]),
                 disk_type=np.zeros(1, np.int32), gpu_model=np.full(1, -1, np.int32), novel_off=n_off,
                 novel_host=n_host, reserved_host=np.full(1, -1, np.int32))
    groups = _groups([abi.GROUP_UNIQUE, abi.GROUP_BALANCED, abi.GROUP_ATTR_EQUALS], [-1, 2, 3], [0, 0, 0],
                     [unique_cot, [300, 301, 302], [400]], [[0, 0], [1, 1, 2], [1]])
    return jobs, offers, groups, lifetime


def test_explainer_counts_the_first_failing_check(gpu, oracle):
    jobs, offers, groups, lifetime = check_order_case()
    fg, fo, assign = _failures(gpu, oracle, jobs, offers, groups, np.array([0], np.int32), lifetime)
    assert list(assign) == [11]
    assert fg == fo
    f = fo[0]
    assert f["counts"][FIRST:FIRST + 11] == [1] * 11 and f["n_passed"] == 1, f
    assert f["counts"][:FIRST] == [0, 0] and f["n_ports"] == 0, f


# ---- rebalancer: four hosts, each filled by one preemptable 100-cpu task of a different user; the
# pending job of user 0 asks 1 cpu.  Unconstrained, equal DRUs pick the greatest hostname (straw).
HOSTS = ["bricks", "rebar", "sticks", "straw"]   # hostname id = name rank = index
AZ = [1, 2, 3, 4]                                # attribute 0 of each host


def rebalance_case(group_lists, groups, own_hosts=()):
    """own_hosts: hosts that also run a 1-cpu task of the pending job's user (group members)."""
    run = [(u + 1, 100.0, h) for u, h in enumerate(range(4))] + [(0, 1.0, h) for h in own_hosts]
    R = len(run)
    t = abi.make_tasks(user=np.array([r[0] for r in run], np.int32), priority=np.full(R, 50, np.int32),
                       start_time=np.full(R, 1_600_000_000_000, np.int64), task_id=np.arange(1000, 1000 + R, dtype=np.int64),
                       job_id=np.arange(1, R + 1, dtype=np.int64), cpus=np.array([r[1] for r in run]),
                       mem=np.full(R, 10.0))
    running = abi.RunningSoA(t=t, host=np.array([r[2] for r in run], np.int32))
    off, gi = abi.csr(group_lists)
    jobs = abi.JobsSoA(n=1, user=np.zeros(1, np.int32), cpus=np.ones(1), mem=np.full(1, 10.0), gpus=np.zeros(1),
                       group_off=off, group_idx=gi)
    hosts = abi.HostTable(n=4, hostname_id=np.arange(4, dtype=np.int32), name_rank=np.arange(4, dtype=np.int32),
                          has_spare=np.zeros(4, np.uint8), spare_cpus=np.zeros(4), spare_mem=np.zeros(4),
                          spare_gpus=np.zeros(4), n_attr_cols=1, attr=np.array(AZ, np.int32))
    users = abi.make_users(5, div_mem=np.full(5, 10.0), div_cpus=np.full(5, 10.0), div_gpus=np.ones(5))
    args = (running, jobs, np.array([R + 1], np.int64), np.array([50], np.int32), hosts, users,
            abi.RebalanceParams(1, 0.05, 1.0, 0))
    return args, groups


def five_groups_case():
    """Five groups, more than the prepared table holds: unique with cotasks on straw and sticks,
    attribute-equals with cotask values {2, 3, 4} (bricks fails), two empty groups and a balanced one
    whose values are all equally frequent.  Only rebar passes them all."""
    groups = _groups([abi.GROUP_UNIQUE, abi.GROUP_ATTR_EQUALS, abi.GROUP_UNIQUE, abi.GROUP_ATTR_EQUALS,
                      abi.GROUP_BALANCED], [-1, 0, -1, 0, 0], [0, 0, 0, 0, 4],
                     [[3, 2], [50, 51, 52], [], [], [60, 61, 62, 63]],
                     [[0, 0], [2, 3, 4], [], [], [1, 2, 3, 4]])
    return rebalance_case([[0, 1, 2, 3, 4]], groups, own_hosts=(3, 2)), "rebar"


def many_values_case():
    """A balanced group whose 72 cotasks carry 70 distinct values, more than the prepared table holds:
    values 1..70 once each and 4 twice more, so straw (4) is the most frequent value and fails."""
    vals = list(range(1, 71)) + [4, 4]
    groups = _groups([abi.GROUP_BALANCED], [0], [0], [list(range(100, 100 + len(vals)))], [vals])
    return rebalance_case([[0]], groups), "sticks"


@pytest.mark.parametrize("case", [five_groups_case, many_values_case], ids=["five_groups", "many_values"])
def test_rebalancer_scalar_group_path(gpu, oracle, case):
    (args, groups), want = case()
    dg = gpu.rebalance(*args, groups=groups)
    do = oracle.rebalance(*args, groups=groups)
    assert dg == do
    assert [HOSTS[d["host"]] for d in do] == [want]
    free = oracle.rebalance(*args, groups=None)
    assert gpu.rebalance(*args, groups=None) == free
    assert [HOSTS[d["host"]] for d in free] == ["straw"]   # the groups decide the outcome
