"""Lease streams whose merged columns are observable VM by VM: the probe cases of test_offer_probe_cases.py (CPU,
against the oracle) and test_state_offers_edges.py (GPU, against cook_state_match_offers and
cook_state_rebalance_offers).  Test infrastructure only: no GPU code is imported here.

Match probes.  Every probed VM's newest lease carries a tag of its own (from 1) in attribute column 0, and its
older leases another value, so a pending constraint (0, tag) pins a job to that VM and to the newest lease's
columns (match.cu reads a pending attr entry as "the host's column equals the value"; 0 or less never matches).
Each VM has three leases from two batches (one VM of a stream may have many), with cpus and mem off the binary grid,
chosen so that the left fold in arrival order differs in its last bit from the fold in every other order that is a
different sum (an order that only swaps the first two leases is the same sum): reverse, sorted, the order of the
offers' slots after reuse, whatever it is, and the pairwise sum.  A VM of many leases is only checked against the
reverse, ascending, descending and pairwise folds and eight shuffles; four to six leases are not used, as off-grid
draws whose fold differs from every other order are too rare there.  Its jobs:
  exact    cpus and mem equal to the folds (plus the VM's ports, gpu or disk need): placed on its VM;
  up-cpus  nextafter(cpus, inf): fails;           up-mem  nextafter(mem, inf): fails;
  port+1   one port more than the VM's leases carry: fails;
  old-gpu / old-disk  a model or disk type only an older lease's map has: fails.
The failing jobs have priority 90 and the exact job 50, so they are ranked first and fail on their own bits.

Spare probes (the rebalancer's view-incubating-offers).  Probed host i of P has spare cpus near 10 (i + 1) and
spare mem near 10 (P - i), so only host i can hold job i (a lower host lacks cpus, a higher one mem).  Job i asks
for cpus exactly at the arrival-order fold when the reverse fold is smaller, and one ulp above it when the reverse
fold is larger: the spare alone is enough iff spare >= request (rebalance.cu `consider`), so the host gets its
decision in the first case only, and a fold in reverse order flips the decision either way.
"""
import itertools

import numpy as np

PRIO_UP, PRIO_EXACT = 90, 50
OLD_ATTR = 1_000_000   # attribute column 0 of a probed VM's older leases: no job asks for it


# ---- folds ------------------------------------------------------------------------------------------------------
def left(xs):
    s = 0.0
    for x in xs:
        s = s + x
    return s


def pairwise(xs):
    if len(xs) <= 2:
        return left(xs)
    h = len(xs) // 2
    return pairwise(xs[:h]) + pairwise(xs[h:])


def other_folds(xs):
    """{name: the fold of xs in another order}: reverse, ascending, descending and pairwise; for three values also
    every other order that is a different sum; for more than six values also eight fixed shuffles."""
    k = len(xs)
    out = {"pairwise": pairwise(xs), "reverse": left(xs[::-1]), "ascending": left(sorted(xs)),
           "descending": left(sorted(xs, reverse=True))}
    if k == 3:
        for p in itertools.permutations(range(k)):
            if list(p[2:]) == list(range(2, k)) and set(p[:2]) == {0, 1}:
                continue
            out["perm" + "".join(map(str, p))] = left([xs[i] for i in p])
        return out
    if k <= 6:
        return out
    rng = np.random.default_rng(k)
    for s in range(8):
        out[f"shuffle{s}"] = left([xs[i] for i in rng.permutation(k)])
    return out


def distinct(xs):
    a = left(xs)
    return all(v != a for v in other_folds(xs).values())


def up(x):
    return float(np.nextafter(x, np.inf))


def off_grid(rng, k, bulk=0.0, unit=1.0, mixed=True):
    """k values off the binary grid whose arrival-order left fold is distinct: tenths, thirds and sevenths of `unit`
    plus a k-th of `bulk` each (values of one magnitude: a small value added to a large sum commutes with the next);
    mixed: some of them 1e3 + 0.1 units larger."""
    for _ in range(2000):
        xs = [float(rng.integers(1, 90)) / float(rng.choice([3.0, 7.0, 10.0])) * unit for _ in range(k)]
        for i in range(k):
            if mixed and rng.random() < 0.25:
                xs[i] = (1e3 + 0.1) * unit + xs[i]
        xs = [bulk / k + x for x in xs]
        if distinct(xs):
            return xs
    raise AssertionError("no distinct fold found")


# ---- match probes -----------------------------------------------------------------------------------------------
class MatchProbes:
    """Probed VMs with their leases split into older and newest batches, and the probe jobs.

    vms: [{code, hostname, tag, cpus: [per lease], mem, ports: [[(b, e)] per lease], gpu, disk (per lease maps),
    k8s}]; leases are dicts as offer_ref takes them.  Job ids start at jid0 and step by 2."""

    def __init__(self, rng, codes, names, ports_share=0.4, gpu_share=0.25, disk_share=0.25,
                 jid0=10, tag0=1, many=None):
        self.vms, self.rows, self.expect = [], {}, {}
        jid = jid0
        for n, code in enumerate(codes):
            k = many if many and n == 0 else 3
            f = rng.random()
            kind = "gpu" if f < gpu_share else "disk" if f < gpu_share + disk_share else "plain"
            v = dict(code=int(code), hostname=names[int(code)], tag=tag0 + n, k=k,
                     cpus=off_grid(rng, k, unit=0.25), mem=off_grid(rng, k, unit=100.0), kind=kind,
                     k8s=int(kind != "plain"))
            v["ports"] = self._ports(rng, k) if rng.random() < ports_share else [[] for _ in range(k)]
            mo, mn = int(rng.integers(1, 4)), int(rng.integers(4, 8))   # an older-only model, the newest's model
            v["gpu"] = [[(mo, 2.0)]] * (k - 1) + [[(mn, 1.0), (mn + 10, 4.0)]] if kind == "gpu" else [[]] * k
            v["disk"] = [[(mo, 9000.0)]] * (k - 1) + [[(mn, 5000.0)]] if kind == "disk" else [[]] * k
            v["fold"] = (left(v["cpus"]), left(v["mem"]))
            assert distinct(v["cpus"]) and distinct(v["mem"])
            self.vms.append(v)
            jid = self._jobs(v, jid)
        self.jid_end = jid

    @staticmethod
    def _ports(rng, k):
        """One or two ranges per lease, disjoint, the leases' ranges out of numeric order."""
        starts = rng.permutation(2 * k + 40)[:2 * k] * 50 + 31000
        out = [[(int(s), int(s) + int(rng.integers(0, 5)))] for s in starts[:k]]
        for q in range(k):
            if rng.random() < 0.3:
                s = int(starts[k + q])
                out[q].append((s, s + 2))
        return out

    def _jobs(self, v, jid):
        c, m = v["fold"]
        n_ports = sum(e - b + 1 for rs in v["ports"] for b, e in rs)
        base = dict(user=0, cpus=c, mem=m, gpus=0.0, ports=n_ports, allowed=1, plugin_accept=1, gpu_model=-1,
                    disk_request=-1.0, disk_type=-1, est_end_ms=-1, ckpt_location=-1, reserved_host=-1, novel=[],
                    attr=[(0, v["tag"])], groups=[])
        if v["kind"] == "gpu":
            model, count = v["gpu"][-1][0]
            base.update(gpus=count, gpu_model=model)
        if v["kind"] == "disk":
            dtype, space = v["disk"][-1][0]
            base.update(disk_request=space, disk_type=dtype)
        jobs = [("exact", dict(base, priority=PRIO_EXACT), v["code"]),
                ("up-cpus", dict(base, priority=PRIO_UP, cpus=up(c)), -1),
                ("up-mem", dict(base, priority=PRIO_UP, mem=up(m)), -1)]
        if n_ports:
            jobs.append(("port+1", dict(base, priority=PRIO_UP, ports=n_ports + 1), -1))
        if v["kind"] == "gpu":
            jobs.append(("old-gpu", dict(base, priority=PRIO_UP, gpus=2.0, gpu_model=v["gpu"][0][0][0]), -1))
        if v["kind"] == "disk":
            jobs.append(("old-disk", dict(base, priority=PRIO_UP, disk_request=9000.0, disk_type=v["disk"][0][0][0]),
                         -1))
        want_ports = [p for rs in v["ports"] for b, e in rs for p in range(b, e + 1)]
        for name, row, where in jobs:
            self.rows[jid] = row
            self.expect[jid] = (v["code"], name, where, want_ports if name == "exact" else None)
            jid += 2
        return jid

    def leases(self, lid0, split=None):
        """(older, newest) lease lists: every VM's leases but its last go in `older` (split: how many of them go to
        older, the rest to newest; at least one each), in VM order.  Lease ids from lid0."""
        older, newest, lid = [], [], lid0
        for v in self.vms:
            k = v["k"]
            cut = k - 1 if split is None else max(1, min(k - 1, split))
            for q in range(k):
                l = dict(id=lid, code=v["code"], hostname=v["hostname"], cpus=v["cpus"][q], mem=v["mem"][q],
                         ports=v["ports"][q], gpu=v["gpu"][q], disk=v["disk"][q], is_k8s=v["k8s"],
                         attr=[v["tag"] if q == k - 1 else OLD_ATTR], gpus=0.0)
                lid += 1
                (older if q < cut else newest).append(l)
        return older, newest, lid

    def pending(self):
        return sorted(self.rows.items())

    def check(self, considerable, assign, ports):
        """Every probe job's outcome: considerable job ids, their hostname codes (-1: unplaced), their port rows.
        Returns the number of probes checked."""
        pos = {int(j): k for k, j in enumerate(np.asarray(considerable).tolist())}
        for jid, (code, name, where, want_ports) in self.expect.items():
            assert jid in pos, f"probe {name} of VM {code} is not considerable"
            k = pos[jid]
            assert int(assign[k]) == where, f"probe {name} of VM {code}: placed on {int(assign[k])}, want {where}"
            if want_ports:
                got = [int(p) for p in np.asarray(ports[k]).tolist()[:len(want_ports)]]
                assert got == want_ports, f"ports of VM {code}"
        return len(self.expect)

    def vm_outcomes(self, considerable, assign):
        """{VM code: (the jobs placed, by probe name)} of a match."""
        pos = {int(j): k for k, j in enumerate(np.asarray(considerable).tolist())}
        out = {}
        for jid, (code, name, _, _) in self.expect.items():
            if int(assign[pos[jid]]) >= 0:
                out.setdefault(code, set()).add(name)
        return {v["code"]: frozenset(out.get(v["code"], ())) for v in self.vms}


def ranked_order(rows):
    """The one user's queue: priority descending, then job id."""
    return sorted(rows, key=lambda j: (-rows[j]["priority"], j))


# ---- spare probes -----------------------------------------------------------------------------------------------
class SpareProbes:
    """P probed hosts (codes[:P]) with three leases each, and one pending job per host (module docstring)."""

    def __init__(self, rng, codes, names, P, jid0=10):
        self.P, self.hosts, self.rows, self.want = P, [], {}, {}
        for i in range(P):
            code = int(codes[i])
            k = 3
            cpus = off_grid(rng, k, bulk=10.0 * (i + 1) - 1.0, unit=0.02, mixed=False)   # at most 0.6 a lease
            mem = off_grid(rng, k, bulk=10.0 * (P - i) - 1.0, unit=0.02, mixed=False)
            a, r = left(cpus), left(cpus[::-1])
            assert a != r
            req = a if r < a else up(a)
            jid = jid0 + 2 * i
            self.rows[jid] = dict(user=0, priority=50, cpus=req, mem=10.0 * (P - i) - 1.0, gpus=0.0, novel=[], attr=[],
                                  groups=[])
            self.want[jid] = code if r < a else -1
            self.hosts.append(dict(code=code, hostname=names[code], cpus=cpus, mem=mem, k=k))

    def leases(self, lid0):
        """Every probed host's leases, one batch per lease position (the first lease of every host, then the
        second, ...)."""
        batches, lid = [], lid0
        for q in range(max(h["k"] for h in self.hosts)):
            b = []
            for h in self.hosts:
                if q < h["k"]:
                    b.append(dict(id=lid, code=h["code"], hostname=h["hostname"], cpus=h["cpus"][q], mem=h["mem"][q],
                                  gpus=float(q % 2)))
                    lid += 1
            batches.append(b)
        return batches, lid

    def decided(self, decisions):
        """{job id: host code or -1} of a rebalance's decisions (each with job_id and host as a hostname code)."""
        got = {j: -1 for j in self.rows}
        for d in decisions:
            got[d["job_id"]] = d["host"]
        return got
