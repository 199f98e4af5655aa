"""The probe cases of offer_probe_cases.py on the oracle (CPU): on the table offer_ref.LeaseBook restates, the probe
queue places exactly the exact jobs, each on its own VM, with the VM's ports in arrival order; with any probed VM's
cpus or mem folded in another order, or moved by one ulp, that VM's outcome changes.  The same for the rebalancer's
spare resources: the decisions follow the arrival-order fold, and a fold in reverse order flips every probed host."""
import numpy as np
import pytest

from cook_b200 import abi, traces
from offer_probe_cases import MatchProbes, SpareProbes, left, other_folds, ranked_order, up
from offer_ref import LeaseBook
from resident_model import jobs_soa, with_fields


def probe_book(seed, n_vms=24, filler=30):
    """Probes on n_vms VMs, their older leases in one batch and newest in another, among filler leases of other
    hosts; every VM named so that name order is neither code order nor its reverse."""
    rng = np.random.default_rng(seed)
    codes = (rng.permutation(n_vms + filler) * 3 + 5).tolist()
    names = {c: f"vm-{(c * 7919) % 10007:05d}" for c in codes}
    pr = MatchProbes(rng, codes[:n_vms], names)
    old, new, lid = pr.leases(100)
    fill = [dict(id=lid + i, code=c, hostname=names[c], cpus=0.5, mem=64.0, attr=[0])
            for i, c in enumerate(codes[n_vms:])]
    b = LeaseBook()
    b.add(old + fill[:filler // 2], 1_000, 1)
    b.add(fill[filler // 2:] + new, 2_000, 1)
    return pr, b


def oracle_match(oracle, pr, table, codes):
    jids = sorted(pr.rows)
    jobs, _, _ = jobs_soa([(j, pr.rows[j]) for j in jids])
    pos = {j: i for i, j in enumerate(jids)}
    ranked = np.array([pos[j] for j in ranked_order(pr.rows)], np.int32)
    mp = max(r["ports"] for r in pr.rows.values())
    m = oracle.match(ranked, jobs, table, abi.make_users(1), traces.match_params(len(jids)), max_ports=mp)
    cons = np.array(jids)[m["considerable"]]
    assign = np.array([int(codes[a]) if a >= 0 else -1 for a in m["assign"]])
    return cons, assign, m["ports"]


@pytest.mark.parametrize("seed", range(3))
def test_probes_place_exactly_the_exact_jobs(oracle, seed):
    pr, b = probe_book(seed)
    codes, table = b.merged([0])
    cons, assign, ports = oracle_match(oracle, pr, table, codes)
    assert pr.check(cons, assign, ports) == len(pr.rows)
    placed = assign[assign >= 0].tolist()
    assert sorted(placed) == sorted(v["code"] for v in pr.vms)   # each exact job on its own VM, nothing else
    kinds = {v["kind"] for v in pr.vms}
    assert kinds == {"plain", "gpu", "disk"} and any(v["ports"][0] for v in pr.vms)


def _altered(table, codes, pr, key, value_of):
    col = table.col(key).copy()
    idx = {int(c): v for v, c in enumerate(codes)}
    for vm in pr.vms:
        col[idx[vm["code"]]] = value_of(vm)
    return with_fields(table, **{key: col})


@pytest.mark.parametrize("seed", range(3))
def test_every_probed_vm_tells_another_fold_apart(oracle, seed):
    """The fold of a probed VM in another order (reverse, ascending, a shuffle, the pairwise sum) or one ulp off:
    the outcome of that VM's probes changes, for every probed VM at once."""
    pr, b = probe_book(seed)
    codes, table = b.merged([0])
    base = pr.vm_outcomes(*oracle_match(oracle, pr, table, codes)[:2])
    assert all(o == {"exact"} for o in base.values())
    alts = {"reverse": lambda xs: left(xs[::-1]), "ascending": lambda xs: left(sorted(xs)),
            "pairwise": lambda xs: other_folds(xs)["pairwise"], "up": lambda xs: up(left(xs)),
            "down": lambda xs: float(np.nextafter(left(xs), -np.inf))}
    for key in ("cpus", "mem"):
        for name, f in alts.items():
            t = _altered(table, codes, pr, key, lambda vm: f(vm[key]))
            got = pr.vm_outcomes(*oracle_match(oracle, pr, t, codes)[:2])
            same = [c for c in base if got[c] == base[c]]
            if name in ("up", "down", "pairwise") or all(len(vm[key]) > 2 for vm in pr.vms):
                assert not same, f"{key} folded {name}: VMs {same} keep their outcome"


def test_builder_folds_differ_from_every_other_order():
    rng = np.random.default_rng(3)
    names = {c: f"h{c}" for c in range(8)}
    pr = MatchProbes(rng, list(range(8)), names, many=300)
    assert pr.vms[0]["k"] == 300
    for v in pr.vms:
        for key in ("cpus", "mem"):
            a = left(v[key])
            assert all(x != a for x in other_folds(v[key]).values())
    old, new, _ = pr.leases(0)
    assert {l["code"] for l in old} == {l["code"] for l in new} == set(range(8))


# ---- the spare resources ----------------------------------------------------------------------------------------
def spare_case(seed, P=40, others=60):
    rng = np.random.default_rng(seed)
    H = P + others
    codes = (rng.permutation(H) * 5 + 2).astype(np.int32)   # host index -> code, shuffled against name order
    names = {int(c): f"node-{int(c):06d}" for c in codes}
    sp = SpareProbes(rng, codes, names, P)
    batches, lid = sp.leases(0)
    b = LeaseBook()
    for q, bt in enumerate(batches):
        b.add(bt, 1_000 + q, 0)
    b.add([dict(id=lid + i, code=int(c), hostname=names[int(c)], cpus=0.0625, mem=8.0) for i, c in
           enumerate(codes[P:])], 900, 0)   # received earlier, arrived later
    rank = np.argsort(np.argsort(codes)).astype(np.int32)   # names in code order
    hosts = abi.HostTable(n=H, hostname_id=codes, name_rank=rank, n_attr_cols=0)
    return sp, b, codes, hosts


def oracle_rebalance(oracle, sp, hosts, codes, spare):
    from cook_b200.engine import _empty_tasks
    jids = sorted(sp.rows)
    jobs, prio, jid = jobs_soa([(j, sp.rows[j]) for j in jids])
    running = abi.RunningSoA(t=_empty_tasks(), host=np.zeros(1, np.int32))
    prm = abi.RebalanceParams(len(jids), 0.5, 1.0, 0)
    out = oracle.rebalance(running, jobs, jid, prio, with_fields(hosts, **spare), abi.make_users(1), prm)
    for d in out:
        d["job_id"] = int(jid[d["pending_idx"]])
        d["host"] = int(codes[d["host"]])
    return sp.decided(out)


@pytest.mark.parametrize("seed", range(2))
def test_spare_probes_follow_the_arrival_fold(oracle, seed):
    sp, b, codes, hosts = spare_case(seed)
    spare = b.spare(codes)
    got = oracle_rebalance(oracle, sp, hosts, codes, spare)
    assert got == sp.want
    n = sum(1 for w in sp.want.values() if w >= 0)
    assert 0 < n < len(sp.want)
    # the reverse fold of every probed host flips every probe's decision
    idx = {int(c): h for h, c in enumerate(codes)}
    rev = dict(spare, spare_cpus=spare["spare_cpus"].copy())
    for h in sp.hosts:
        rev["spare_cpus"][idx[h["code"]]] = left(h["cpus"][::-1])
    flipped = oracle_rebalance(oracle, sp, hosts, codes, rev)
    assert all((flipped[j] >= 0) != (sp.want[j] >= 0) for j in sp.want)
