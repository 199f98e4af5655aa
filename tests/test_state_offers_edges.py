"""cook_state_match_offers and cook_state_rebalance_offers on the probe cases of offer_probe_cases.py (GPU, -m gpu).

Every match cycle is checked twice: by test_state_offers.cycle (bit equality with cook_state_match_derived fed the
table offer_ref.LeaseBook restates, the gone list, the transfers), and by the probes: every exact job placed on its
VM with the VM's ports in arrival order, every other probe failed.  The probes see each VM's merged cpus and mem at
the last bit, so a merge that folds in another order fails them even where no other placement depends on it.
  a. a few hundred VMs over several cycles, slots reused between them;
  b. past one tile: the live leases through 2047, 2048, 2049 and past 4096, more than 2048 VMs, the offer table's
     slots past 1024 and 2048 with live rows, the port and attribute arenas past 4096 entries, the attribute arena then
     compacted into a fresh buffer, one VM with 300 leases whose sorted run spans index 2048;
  c. bookkeeping edges: an older lease outliving a single-shot newest one with other map lengths and flags,
     attribute widths 3, 0, 1 with a pending row on column 2, receive times out of order and equal, gone_cap equal to
     the offers that leave, a reservation on a code without live offers, a reset then a batch past the old hw;
  d. the rebalancer's spare on more than 2048 hosts and 4096 live leases, the host table shuffled against the
     codes: equal to cook_state_rebalance_derived fed LeaseBook.spare and to the oracle, with the probes' decisions.
"""
import numpy as np
import pytest

from cook_b200 import abi, traces
from offer_probe_cases import MatchProbes, SpareProbes
from offer_ref import LeaseBook, gone_list
from resident_model import DEFAULTS, START, Pool, with_fields
from test_state_offers import INCUBATE, add, cycle

pytestmark = pytest.mark.gpu


def probe_pool(name):
    return Pool(name, send_hosts=True, send_lists=True, users=abi.make_users(1))


class Counters:
    """What the stream drove the handle through, from the test's own model: the live leases and VMs at each merge,
    the offer table's hw (slots ever used since the reset: the peak of the live leases, as freed slots are taken
    first), and per list arena (ports, attributes) its entries, capacity and the compactions into a fresh buffer.

    The model restates state.cu's policy and must follow it: ListArena::grow (capacity max(n, 2 cap, 4096), the
    compaction buffer `alt` freed), compact_lists (when dead entries outnumber live ones; a kernel into `alt`, then
    allocated if null, only with live entries) after every cook_state_offers_add and at the end of every
    cook_state_match_offers, and Table::take_slot (free slots first)."""

    def __init__(self):
        self.live, self.vms, self.hw = [], [], 0
        self.ar = {k: dict(tail=0, live=0, cap=0, alt=False, fresh=0, peak=0) for k in ("ports", "attr")}

    @staticmethod
    def _n(l, k):
        return len(l.get("ports", [])) if k == "ports" else len(l.get("attr", []))

    def added(self, book, leases):
        self.hw = max(self.hw, len(book.leases))
        for k, a in self.ar.items():
            n = sum(self._n(l, k) for l in leases)
            if a["tail"] + n > a["cap"]:
                a["cap"], a["alt"] = max(a["tail"] + n, 2 * a["cap"], 4096), False
            a["tail"] += n
            a["live"] += n
            a["peak"] = max(a["peak"], a["tail"])
            self._compact(a)

    def left(self, gone_leases):
        for k, a in self.ar.items():
            a["live"] -= sum(self._n(l, k) for l in gone_leases)
            self._compact(a)

    def _compact(self, a):
        if a["tail"] - a["live"] > a["live"]:
            if a["live"] > 0:
                a["fresh"] += not a["alt"]
                a["alt"] = True
            a["tail"] = a["live"]


def probe_cycle(p, book, pr, now, cnt=None):
    """One match of the probe queue: cycle()'s comparison, then the probes.  Returns the match."""
    p.apply(up=pr.pending())
    p.rank()
    before = {l["id"]: l for l in book.leases}
    mp = max(r["ports"] for r in pr.rows.values())
    live_vms = None
    if cnt is not None:
        after = [l for l in book.leases if now - l["received_ms"] < INCUBATE]
        live_vms = len({l["hostname"] for l in after})
        cnt.live.append(len(after))
        cnt.vms.append(live_vms)
    got, _ = cycle(p, book, now, traces.match_params(len(pr.rows)), max_ports=mp)
    assert pr.check(got["considerable"], got["assign"], got["ports"]) == len(pr.rows)
    if cnt is not None:
        cnt.left([before[i] for i, _ in got["gone"]])
    p.apply(rm=list(pr.rows))
    return got


def filler(lid, code, name, ports=True, maps=True):
    l = dict(id=lid, code=code, hostname=name, cpus=0.5, mem=64.0, attr=[0], gpus=0.0)
    if ports:
        l["ports"] = [(40000 + code % 1000, 40001 + code % 1000), (50000, 50000)]
    if maps:
        l.update(is_k8s=1, gpu=[(9, 1.0)], disk=[(9, 100.0)])
    return l


# ---- a. probes at small scale ---------------------------------------------------------------------------------------
def test_probes_over_reused_slots():
    rng = np.random.default_rng(5)
    names = {c: f"vm-{(c * 7919) % 10007:05d}" for c in range(400)}
    p, book = probe_pool("probe-small"), LeaseBook()
    now, lid, jid, fid = START, 0, 10, 10 ** 6
    try:
        for c in range(5):
            pr = MatchProbes(rng, rng.choice(300, 60, replace=False).tolist(), names, jid0=jid)
            jid = pr.jid_end
            old, new, lid = pr.leases(lid, split=int(rng.integers(1, 3)))
            fill = [dict(filler(fid + i, int(cd), names[int(cd)], ports=i % 2 == 0), single_shot=i % 4 == 1)
                    for i, cd in enumerate(rng.choice(np.arange(300, 400), 30, replace=False))]
            fid += 30
            add(p.gpu, book, fill[:15] + old, now, 1)
            add(p.gpu, book, new + fill[15:], now + 500, 1)
            probe_cycle(p, book, pr, now + 1_000)
            now += 6_000   # the fillers expire three cycles on: their slots and the consumed ones are taken again
    finally:
        p.close()


# ---- b. past one tile ------------------------------------------------------------------------------------------------
def test_probes_past_one_tile(capsys):
    rng = np.random.default_rng(7)
    p, book, cnt = probe_pool("probe-tile"), LeaseBook(), Counters()
    fnames = {c: f"f-{c:06d}" for c in range(100_000, 110_000)}     # fillers sort first,
    pnames = {c: f"p-{(c * 7919) % 10007:05d}" for c in range(6000)}  # then "m-", then the probed VMs
    pnames[9999] = "m-many"
    state = dict(lid=0, jid=10, fcode=100_000, tag=1)
    now = START

    def add_fill(n, at):
        ls = [filler(10 ** 7 + state["fcode"] + i, state["fcode"] + i, fnames[state["fcode"] + i]) for i in range(n)]
        state["fcode"] += n
        add(p.gpu, book, ls, at, 1)
        cnt.added(book, ls)

    def probes(codes, at, many=None):
        pr = MatchProbes(rng, codes, pnames, jid0=state["jid"], tag0=state["tag"], many=many)
        state["jid"], state["tag"] = pr.jid_end, state["tag"] + len(codes)
        old, new, state["lid"] = pr.leases(state["lid"])
        add(p.gpu, book, old, at, 1)
        cnt.added(book, old)
        add(p.gpu, book, new, at + 1, 1)
        cnt.added(book, new)
        return pr

    try:
        pool = rng.permutation(6000)
        nxt = 0
        for target in (600, 2047, 2048, 2049):    # live leases at the merge
            pr_codes = pool[nxt:nxt + 40].tolist()
            nxt += 40
            # the probe leases first, then fillers up to the target
            pr = probes(pr_codes, now)
            add_fill(target - len(book.leases), now + 2)
            probe_cycle(p, book, pr, now + 3, cnt)
            assert cnt.live[-1] == target
            now += 100
        # past 4096: the 300-lease VM's sorted run starts at the live fillers (< 2048) and spans index 2048
        F = len(book.leases)
        assert 1748 < F < 2048
        late = now + 8_000   # these survive the expiry below
        codes = [9999] + pool[nxt:nxt + 640].tolist()
        nxt += 641
        pr = probes(codes, late, many=300)
        vms = book.vms()
        runs, pos = {}, 0
        for h, ls in vms.items():
            runs[h] = (pos, pos + len(ls))
            pos += len(ls)
        s, e = runs["m-many"]
        assert s < 2048 < e and pos > 4096 and len(vms) > 2048
        probe_cycle(p, book, pr, late + 3, cnt)
        # every lease received before `late` expires: most of both arenas is dead, compacted into a fresh buffer
        now = START + INCUBATE + 1_000
        pr = probes(pool[nxt:nxt + 40].tolist(), now)
        nxt += 40
        probe_cycle(p, book, pr, max(now, late) + 4, cnt)
        t = max(now, late) + 10   # after the compaction, the arenas read from their new buffers
        pr = probes(pool[nxt:nxt + 40].tolist(), t)
        probe_cycle(p, book, pr, t + 2, cnt)
        ap, aa = cnt.ar["ports"], cnt.ar["attr"]
        with capsys.disabled():
            print(f"\n[offers past one tile] live leases at the merges {cnt.live}, VMs {cnt.vms}, offer hw {cnt.hw}, "
                  f"port arena peak {ap['peak']} (cap {ap['cap']}, fresh compactions {ap['fresh']}), attribute arena "
                  f"peak {aa['peak']} (cap {aa['cap']}, fresh compactions {aa['fresh']})")
        assert {2047, 2048, 2049} <= set(cnt.live) and max(cnt.live) > 4096 and max(cnt.vms) > 2048
        assert cnt.hw > 4096
        assert ap["peak"] > 4096 and aa["peak"] > 4096 and aa["cap"] > 4096 and aa["fresh"] >= 1
    finally:
        p.close()


# ---- c. bookkeeping edges ------------------------------------------------------------------------------------------
def plain_jobs(jid0, n=6, attr=()):
    return [(jid0 + 2 * i, dict(DEFAULTS, user=0, priority=50, cpus=1.0, mem=100.0, novel=[],
                                attr=list(attr) if i == 0 else [], groups=[])) for i in range(n)]


def test_bookkeeping_edges():
    p, book = probe_pool("offer-edges"), LeaseBook()
    prm = traces.match_params(50)
    names = {c: f"e-{c:04d}" for c in range(200)}
    now = START
    try:
        # an older lease that is not single-shot outlives its single-shot newest one, which has other gpu and disk map
        # lengths and other k8s and max-tasks flags: host 1 (k8s with maps and a max-tasks limit under a newest lease
        # without either) and host 2 (a max-tasks limit under a k8s newest lease without one).  No job fits them in
        # the first cycle, so the newest leases are dropped; the second cycle places on them only what the older
        # leases' columns allow, which needs the VM counts of the plan (is_k8s and max_tasks present, the gpu and disk
        # maps sized for the older leases) to have moved from the dropped leases to the older ones.
        old = [dict(id=1, code=1, hostname=names[1], cpus=0.5, mem=50.0, is_k8s=1, max_tasks=7, num_tasks=1,
                    gpu=[(2, 1.0), (3, 2.0)], disk=[(1, 10.0)], ports=[(31000, 31002)], attr=[4, 5, 6]),
               dict(id=6, code=2, hostname=names[2], cpus=0.5, mem=50.0, max_tasks=3, num_tasks=1, attr=[5, 0, 0])]
        newest = [dict(id=2, code=1, hostname=names[1], cpus=0.25, mem=25.0, single_shot=True, is_k8s=0,
                       gpu=[(4, 1.0)], disk=[(2, 5.0), (3, 6.0), (4, 7.0)], attr=[7, 8, 9]),
                  dict(id=7, code=2, hostname=names[2], cpus=0.25, mem=25.0, single_shot=True, is_k8s=1,
                       attr=[8, 0, 0])]
        other = [dict(id=3 + i, code=10 + i, hostname=names[10 + i], cpus=2.0, mem=500.0, attr=[1, 2, 3]) for i in
                 range(3)]
        add(p.gpu, book, old + other, now, 3)
        add(p.gpu, book, newest, now + 10, 3)
        p.apply(up=plain_jobs(10, attr=[(2, 3)]))
        p.rank()
        got, _ = cycle(p, book, now + 20, prm)
        ids = {i for i, _ in got["gone"]}
        assert {(2, abi.OFFER_SINGLE_SHOT), (7, abi.OFFER_SINGLE_SHOT)} <= set(got["gone"]) and not ids & {1, 6}
        assert [l["id"] for l in book.leases] == [1, 6]
        p.apply(rm=list(p.pend))
        on1 = dict(DEFAULTS, user=0, cpus=0.25, mem=10.0, gpus=2.0, gpu_model=3, disk_request=10.0, disk_type=1,
                   novel=[], attr=[(0, 4)], groups=[])
        jobs = {30: dict(on1, priority=50),                                     # the older lease's gpu and disk maps
                32: dict(on1, priority=90, gpus=1.0, gpu_model=4),              # a model only the dropped map has
                34: dict(on1, priority=90, disk_request=5.0, disk_type=2)}      # a disk type only the dropped map has
        for i in range(4):                                                      # two fit under max_tasks 3, num_tasks 1
            jobs[40 + 2 * i] = dict(DEFAULTS, user=0, priority=50, cpus=0.1, mem=1.0, novel=[], attr=[(0, 5)],
                                    groups=[])
        p.apply(up=sorted(jobs.items()))
        p.rank()
        got, _ = cycle(p, book, now + 30, prm)   # hosts 1 and 2 from the older leases' columns alone
        where = dict(zip(got["considerable"].tolist(), got["assign"].tolist()))
        assert where[30] == 1 and where[32] == where[34] == -1
        assert sorted(where[j] for j in (40, 42, 44, 46)) == [-1, -1, 2, 2]
        p.apply(rm=list(p.pend))
        # attribute widths 3, 0, 1 while a pending row names column 2: the merged value there is 0 where the newest
        # lease is narrower
        add(p.gpu, book, [dict(id=20, code=20, hostname=names[20], cpus=1.5, mem=300.0, attr=[1, 1, 3])], now + 40, 3)
        add(p.gpu, book, [dict(id=21, code=21, hostname=names[21], cpus=1.5, mem=300.0)], now + 41, 0)
        add(p.gpu, book, [dict(id=22, code=20, hostname=names[20], cpus=1.5, mem=300.0, attr=[1]),
                          dict(id=23, code=22, hostname=names[22], cpus=1.5, mem=300.0, attr=[2])], now + 42, 1)
        pinned = dict(DEFAULTS, user=0, priority=60, cpus=1.0, mem=100.0, novel=[], attr=[(0, 1)], groups=[])
        p.apply(up=plain_jobs(50, n=3, attr=[(2, 3)]) + [(60, pinned)])
        p.rank()
        cycle(p, book, now + 50, prm)
        # receive times out of order and equal: the expiry is no prefix of the arrival order
        t0 = now + 1_000
        add(p.gpu, book, [dict(id=30 + i, code=30 + i, hostname=names[30 + i], cpus=0.25, mem=10.0) for i in range(3)],
            t0, 0)
        add(p.gpu, book, [dict(id=40 + i, code=40 + i, hostname=names[40 + i], cpus=0.25, mem=10.0) for i in range(3)],
            t0 - 700, 0)
        add(p.gpu, book, [dict(id=50 + i, code=50 + i, hostname=names[50 + i], cpus=0.25, mem=10.0) for i in range(3)],
            t0, 0)
        add(p.gpu, book, [dict(id=60 + i, code=30 + i, hostname=names[30 + i], cpus=0.25, mem=10.0) for i in range(2)],
            t0 - 700, 0)
        p.apply(rm=list(p.pend))
        p.rank()
        got, _ = cycle(p, book, t0 - 700 + INCUBATE, prm)
        ids = {i for i, _ in got["gone"]}   # 60 and 61 arrived after 50-52, which stay
        assert {40, 41, 42, 60, 61} <= ids and not ids & {30, 31, 32, 50, 51, 52}
        # a reservation on a named code without a live offer
        p.apply(up=plain_jobs(70, n=4))
        p.patch([70, 72], reserved_host=np.array([40, 1], np.int32))
        p.rank()
        cycle(p, book, t0 - 600 + INCUBATE, prm)
        # gone_cap equal to the offers that leave: every live offer expires
        p.apply(rm=list(p.pend))
        p.rank()
        n = len(book.leases)
        assert n > 0
        late = max(l["received_ms"] for l in book.leases) + INCUBATE
        old = book.expire(late, INCUBATE)
        g = p.gpu.state_match_offers(late, INCUBATE, with_fields(p.users, usage_count=None, usage_cpus=None,
                                                                 usage_mem=None, usage_gpus=None), prm, gone_cap=n)
        assert g["gone"] == gone_list(old, [], []) and len(g["gone"]) == n and not book.leases
        # a reset, then a batch larger than the handle's hw before it
        add(p.gpu, book, [dict(id=100 + i, code=100 + i % 50, hostname=names[100 + i % 50], cpus=0.5, mem=30.0)
                          for i in range(80)], late + 1, 0)
        p.apply(up=plain_jobs(90), reset=True)
        book.drop_all()
        big = [dict(id=300 + i, code=100 + i % 90, hostname=names[100 + i % 90], cpus=0.5 + (i % 3) / 10,
                    mem=30.0 + i / 7, ports=[(31000 + i, 31000 + i)], gpu=[(1, 1.0)] * (i % 2), is_k8s=i % 2,
                    attr=[i % 5, 1]) for i in range(300)]
        add(p.gpu, book, big, late + 2, 2)
        p.rank()
        cycle(p, book, late + 3, prm, max_ports=0)
    finally:
        p.close()


# ---- d. the rebalancer's spare resources past one tile ------------------------------------------------------------
def test_rebalance_spare_past_one_tile(oracle):
    from cook_b200.engine import _empty_tasks
    from resident_model import jobs_soa
    rng = np.random.default_rng(11)
    P, H = 300, 2600
    codes = (rng.permutation(H) * 5 + 2).astype(np.int32)   # host index -> code, shuffled against name order
    names = {int(c): f"node-{int(c):06d}" for c in codes}
    sp = SpareProbes(rng, codes, names, P)
    rank = np.argsort(np.argsort(codes)).astype(np.int32)
    hosts = abi.HostTable(n=H, hostname_id=codes, name_rank=rank, n_attr_cols=0)
    p, book = probe_pool("spare-tile"), LeaseBook()
    try:
        batches, lid = sp.leases(0)
        for q, bt in enumerate(batches):
            add(p.gpu, book, bt, START + q, 0)
        rest = [dict(id=lid + i, code=int(codes[P + i % (H - P)]), hostname=names[int(codes[P + i % (H - P)])],
                     cpus=0.0625, mem=8.0, gpus=float(i % 2)) for i in range(2 * (H - P))]
        add(p.gpu, book, rest, START - 5, 0)
        assert len(book.leases) > 4096 and len(book.vms()) > 2048
        p.apply(up=sorted(sp.rows.items()))
        p.rank()
        prm = abi.RebalanceParams(P, 0.5, 1.0, 0)
        spare = book.spare(codes)
        want = p.gpu.state_rebalance(with_fields(hosts, **spare), p.users, prm, derived=True)
        got = p.gpu.state_rebalance(hosts, p.users, prm, offers=True)
        key = ("job_id", "pending_idx", "host", "victims", "dru", "mem", "cpus", "gpus")
        assert [tuple(d[k] for k in key) for d in got] == [tuple(d[k] for k in key) for d in want]
        jids = sorted(sp.rows)
        jobs, prio, jid = jobs_soa([(j, sp.rows[j]) for j in jids])
        o = oracle.rebalance(abi.RunningSoA(t=_empty_tasks(), host=np.zeros(1, np.int32)), jobs, jid, prio,
                             with_fields(hosts, **spare), abi.make_users(1), prm)
        assert [(int(jid[d["pending_idx"]]), d["host"], d["cpus"], d["mem"]) for d in o] == \
               [(d["job_id"], d["host"], d["cpus"], d["mem"]) for d in got]
        assert sp.decided([dict(d, host=int(codes[d["host"]])) for d in got]) == sp.want
    finally:
        p.close()
