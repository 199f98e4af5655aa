"""cook_state_offers_add / cook_state_match_offers: a pool's offers kept on the device as Fenzo's leases, and a
resident match that expires, merges and consumes them itself.

CPU: the restatement (offer_ref) against cook_b200.cycle's OfferCache and offers_from_cache: cpus, mem and ports of
the merged table on the lease golden case and on random streams, the byte order of hostnames, and the expiry,
consumption and single-shot fates.
GPU (-m gpu): churn on a C2-shaped and a config-#3-shaped pool, every cycle against cook_state_match_derived fed the
restated table (bit equality of considerable, hostnames, ports, fail, evals, offers used, failure counts and the usage
exchange; the gone list; the transfer formula); errors that leave the handle unchanged; reset;
cook_state_rebalance_offers against cook_state_rebalance_derived fed the restated spare on a config-#4 pool; K15's
handle-resource-offers! answers through cycle.PoolCycle.handle_resource_offers_resident.
"""
import numpy as np
import pytest

from cook_b200 import abi, traces
from cook_b200.cycle import OfferCache, offers_from_cache
from cook_b200.engine import CookError
from offer_ref import LeaseBook, gone_list, name_key, offers_soa
from resident_model import START, Pool, pool_rows, with_fields


def cache_of(stream):
    """OfferCache and LeaseBook fed the same (now_ms, leases) stream."""
    c, b = OfferCache(incubate_ms=15_000), LeaseBook()
    for now, leases in stream:
        c.add(leases, now)
        b.add(leases, now)
    return c, b


def merged_by_host(c):
    names, of = offers_from_cache(c, {l["hostname"]: l["code"] for l in c.leases})
    off = of.col("port_off")
    return {n: (of.col("cpus")[i], of.col("mem")[i], list(zip(of.col("port_begin")[off[i]:off[i + 1]].tolist(),
                                                               of.col("port_end")[off[i]:off[i + 1]].tolist())))
            for i, n in enumerate(names)}


def book_by_host(b):
    codes, t = b.merged()
    names = list(b.vms())
    off = t.col("port_off")
    return {n: (t.col("cpus")[i], t.col("mem")[i],
                list(zip(t.col("port_begin")[off[i]:off[i + 1]].tolist(), t.col("port_end")[off[i]:off[i + 1]].tolist()))
                if off is not None else [])
            for i, n in enumerate(names)}


def random_stream(rng, n_batches, n_hosts=12, cpus=(0.25, 0.5, 1.0, 3.0), mem=(100.0, 0.375, 1024.0)):
    names = ["a", "a-1", "b", "été", "z", "Z", "aÿ", "b0"][:n_hosts] + [f"h{i}" for i in range(n_hosts)]
    lid, out, now = 0, [], 0
    for _ in range(n_batches):
        now += int(rng.choice([0, 2500, 5000]))
        batch = []
        for _ in range(int(rng.integers(1, 6))):
            h = int(rng.integers(len(names)))
            batch.append({"id": lid, "hostname": names[h], "code": h, "cpus": float(rng.choice(cpus)),
                          "mem": float(rng.choice(mem)), "single_shot": bool(rng.random() < 0.2),
                          "ports": [(int(p), int(p) + 4) for p in rng.integers(31000, 32000, int(rng.integers(0, 3)))]})
            lid += 1
        out.append((now, batch))
    return out


# ---- CPU: the restatement against OfferCache / offers_from_cache --------------------------------------------
def test_restatement_on_the_lease_golden_case():
    stream = [(0, [{"id": 0, "hostname": "a", "code": 7, "cpus": 4.0, "mem": 100.0, "ports": [(31000, 31009)]},
                   {"id": 1, "hostname": "b", "code": 8, "cpus": 1.0, "mem": 10.0, "single_shot": True}]),
              (10_000, [{"id": 2, "hostname": "a", "code": 7, "cpus": 2.0, "mem": 50.0, "ports": [(31500, 31504)]}])]
    c, b = cache_of(stream)
    assert book_by_host(b) == merged_by_host(c) == {"a": (6.0, 150.0, [(31000, 31009), (31500, 31504)]),
                                                     "b": (1.0, 10.0, [])}
    consumed, dropped = b.after_match([])
    assert not consumed and [l["id"] for l in dropped] == [1]
    assert [l["id"] for l in b.expire(16_000, 15_000)] == [0] and [l["id"] for l in b.expire(26_000, 15_000)] == [2]


@pytest.mark.parametrize("seed", range(6))
def test_restatement_on_random_streams(seed):
    """On the binary grid: offers_from_cache's sum() is compensated on Python 3.12, so only exact sums compare bit
    for bit with the left fold (test_merge_is_a_left_fold covers the rest)."""
    rng = np.random.default_rng(seed)
    c, b = cache_of(random_stream(rng, 12))
    for step in range(6):
        now = 30_000 + 5_000 * step
        assert [l["id"] for l in b.expire(now, 15_000)] == [l["id"] for l in c.expire(now)]
        got, want = book_by_host(b), merged_by_host(c)
        assert got.keys() == want.keys()
        for h in got:   # the same left folds, bit for bit
            assert got[h][0].tobytes() == np.float64(want[h][0]).tobytes() and got[h][1] == want[h][1]
            assert got[h][2] == want[h][2]
        used = {l["code"] for l in b.leases if rng.random() < 0.3}
        bc, bd = b.after_match(used)
        cc, cd = c.after_match({l["hostname"] for l in c.leases if l["code"] in used})
        assert [l["id"] for l in bc] == [l["id"] for l in cc] and [l["id"] for l in bd] == [l["id"] for l in cd]
        for now2, leases in random_stream(rng, 1):
            c.add(leases, now + 1)
            b.add(leases, now + 1)


def test_merge_is_a_left_fold():
    b = LeaseBook()
    xs = [0.1, 0.2, 0.3, 1e16, 1.0, -1e16]
    b.add([{"id": i, "hostname": "h", "code": 0, "cpus": x, "mem": x} for i, x in enumerate(xs)], 0)
    _, t = b.merged()
    left = 0.0
    for x in xs:
        left = left + x
    assert t.col("cpus")[0] == left and t.col("mem")[0] == left


def test_name_order_is_byte_order():
    b = LeaseBook()
    names = ["b", "a-1", "a", "é", "e", "Z", "aĀ", "aÿ"]
    b.add([{"id": i, "hostname": n, "code": i, "cpus": 1.0, "mem": 1.0} for i, n in enumerate(names)], 0)
    assert list(b.vms()) == ["Z", "a", "a-1", "aÿ", "aĀ", "b", "e", "é"]
    assert sorted(n.encode() for n in names) == [name_key(n) for n in b.vms()]


def test_gone_list_is_in_arrival_order():
    b = LeaseBook()
    b.add([{"id": 10, "hostname": "x", "code": 1, "cpus": 1.0, "mem": 1.0}], 0)
    b.add([{"id": 11, "hostname": "y", "code": 2, "cpus": 1.0, "mem": 1.0, "single_shot": True},
           {"id": 12, "hostname": "x", "code": 1, "cpus": 1.0, "mem": 1.0}], 5)
    old = b.expire(10, 10)
    consumed, dropped = b.after_match([1])
    assert gone_list(old, consumed, dropped) == [(10, abi.OFFER_EXPIRED), (11, abi.OFFER_SINGLE_SHOT),
                                                 (12, abi.OFFER_USED)]


# ---- GPU helpers ------------------------------------------------------------------------------------------------
INCUBATE = 15_000


class Stream:
    """Leases cut from a trace's offer table: each listed host gets 1-3 leases that split its cpus, mem and port
    ranges; its other columns come from the table, num_tasks varies per lease."""

    def __init__(self, tmpl, rng, k8s_share=0.0):
        self.t, self.rng, self.lid = tmpl, rng, 0
        self.codes = tmpl.col("hostname_id")
        specials = ["a", "a-1", "b", "été", "Z"]
        self.names = {int(c): (specials[i] if i < len(specials) else f"host-{int(c) * 7919 % 100003:06d}")
                      for i, c in enumerate(self.codes)}
        self.named = set()
        k = tmpl.col("is_k8s")
        self.k8s = k.astype(bool) if k is not None else rng.random(tmpl.n) < k8s_share
        self.W = tmpl.n_attr_cols if tmpl.col("attr") is not None else 0

    def _list(self, off, *vals, h):
        o = self.t.col(off)
        if o is None:
            return []
        return list(zip(*[self.t.col(v)[o[h]:o[h + 1]].tolist() for v in vals]))

    def batch(self, n_hosts, crumbs=0):
        """Leases of n_hosts of the table's hosts, and `crumbs` leases on hosts of their own too small for any job,
        which only leave by expiry (every third one is single-shot and leaves after the next match)."""
        rng, t = self.rng, self.t
        out = [{"id": 1000 + self.lid + i, "code": 10 ** 6 + i % 7, "hostname": f"crumb-{i % 7}", "cpus": 0.0625,
                "mem": 1.0, "single_shot": i % 3 == 2} for i in range(crumbs)]
        self.lid += crumbs
        for h in rng.choice(t.n, n_hosts, replace=False).tolist():
            code = int(self.codes[h])
            k = int(rng.choice([1, 1, 1, 2, 3]))
            ports = self._list("port_off", "port_begin", "port_end", h=h)
            attr = t.col("attr").reshape(t.n_attr_cols, t.n)[:, h].tolist() if self.W else []
            for q in range(k):
                l = {"id": 1000 + self.lid, "code": code, "hostname": self.names[code],
                     "cpus": float(t.col("cpus")[h]) / k, "mem": float(t.col("mem")[h]) / k,
                     "gpus": float(rng.choice([0.0, 1.0, 2.0])), "ports": ports[q::k],
                     "num_tasks": int(rng.integers(0, 5)), "is_k8s": int(self.k8s[h]),
                     "single_shot": bool(self.k8s[h]), "attr": attr}
                for c, dt in (("location", int), ("max_tasks", int), ("host_start_time", int)):
                    if t.col(c) is not None:
                        l[c] = dt(t.col(c)[h])
                l["gpu"] = self._list("gpu_off", "gpu_model", "gpu_count", h=h)
                l["disk"] = self._list("disk_off", "disk_type", "disk_space", h=h)
                if q < k - 1:   # an older lease of the host differs from its newest: the merge must take the newest
                    l["attr"] = [(a + 1) % 4 for a in attr]
                    l["gpu"], l["disk"] = l["gpu"][:-1], l["disk"][1:]
                    l["location"] = l.get("location", -1) + 1
                    l["max_tasks"] = -1
                    l["host_start_time"] = l.get("host_start_time", -1) + 7
                # a known code may come without its name
                l["name"] = "" if code in self.named and rng.random() < 0.5 else self.names[code]
                self.named.add(code)
                out.append(l)
                self.lid += 1
        return out


def add(e, book, leases, now, W):
    soa, ids, single, gpus, names = offers_soa(leases, W)
    e.state_offers_add(soa, ids, now, single_shot=single, offer_gpus=gpus, hostnames=names)
    book.add(leases, now, W)


def table_bytes(t):
    """The bytes of offer table t that cook_match's build uploads (run_* derived: not uploaded)."""
    O = t.n
    if O == 0:
        return 0
    b = (4 + 8 + 8 + 4) * O   # permutation, cpus, mem, hostname codes
    for c, sz in (("is_k8s", 1), ("reserved", 1), ("location", 4), ("max_tasks", 4), ("num_tasks", 4),
                  ("host_start_time", 8)):
        if t.col(c) is not None:
            b += sz * O
    for off, a, bb, sa, sb in (("port_off", "port_begin", "port_end", 4, 4), ("gpu_off", "gpu_model", "gpu_count", 4, 8),
                               ("disk_off", "disk_type", "disk_space", 4, 8)):
        if t.col(off) is not None:
            n = max(1, int(t.col(off)[-1]))
            b += 4 * (O + 1) + (sa + sb) * n
    if t.col("attr") is not None:
        b += 4 * t.n_attr_cols * O
    return b


def derived_tables(table, users, groups):
    table = with_fields(table, run_cpus=None, run_mem=None, run_count=None)
    users = with_fields(users, usage_count=None, usage_cpus=None, usage_mem=None, usage_gpus=None)
    if groups is not None:
        groups = with_fields(groups, cot_off=None, cot_hostname_id=None, cot_attr_val=None)
    return table, users, groups


def cycle(p, book, now, prm, groups=None, max_ports=0):
    """One cook_state_match_offers against cook_state_match_derived fed the restated table on the same handle.
    Returns the match and the restated VM codes."""
    e = p.gpu
    old = book.expire(now, INCUBATE)
    pend_cols = {c for r in p.pend.values() for c, _ in r["attr"]}
    gcols = [int(c) for c in groups.col("attr_col") if c >= 0] if groups is not None else []
    rs = [r["reserved_host"] for r in p.pend.values() if r["reserved_host"] != -1]
    codes, table = book.merged(pend_cols, gcols, rs if rs else None)
    dt, du, dg = derived_tables(table, p.users, groups)
    want = e.state_match(dt, du, prm, groups=dg, max_ports=max_ports, derived=True)
    n = len(want["considerable"])
    kk = np.arange(n, dtype=np.int32)
    fw = e.match_failures(kk) if n else []
    xw = e.exchange_usage(p.users.n_users)
    got = e.state_match_offers(now, INCUBATE, du, prm, groups=dg, max_ports=max_ports)
    assert np.array_equal(got["considerable"], want["considerable"])
    assert got["assign"].tolist() == [int(codes[a]) if a >= 0 else -1 for a in want["assign"].tolist()]
    for k in ("ports", "fail"):
        assert np.array_equal(got[k], want[k]), k
    sg, sw = got["stats"], want["stats"]
    for k in ("n_considerable", "n_matched", "evals", "n_offers_used", "head_matched"):
        assert sg[k] == sw[k], k
    if n:
        assert e.match_failures(kk) == fw
    assert np.array_equal(e.exchange_usage(p.users.n_users), xw)
    consumed, dropped = book.after_match(got["assign"][got["assign"] >= 0].tolist())
    gone = gone_list(old, consumed, dropped)
    assert got["gone"] == gone
    nres = len(rs) if table.col("reserved") is not None and table.n else 0
    if n:
        assert sg["h2d_bytes"] == sw["h2d_bytes"] - table_bytes(table) + 4 * table.n + 4 * nres + 4 * len(gone)
        assert sg["d2h_bytes"] == sw["d2h_bytes"]
    else:
        assert sg["h2d_bytes"] == 4 * len(gone)
    return got, codes


def launch_some(p, got, tid, limit):
    placed = got["assign"] >= 0
    jl = got["considerable"][placed].tolist()[:limit]
    hs = got["assign"][placed][:len(jl)].astype(np.int32)
    p.launch(jl, [tid + 3 * i for i in range(len(jl))], np.full(len(jl), START, np.int64), hs)
    return tid + 3 * len(jl) + 3, len(jl)


def run_churn(t, seed, n_cycles, groups=None, reserve_hosts=False, k8s_share=0.0):
    rng = np.random.default_rng(seed)
    users, tmpl = t["users"], t["offers"]
    pend, run = pool_rows(t)
    codes = tmpl.col("hostname_id")
    for r in run.values():
        r["host"] = int(rng.choice(codes))
        r["groups"] = []
    items = sorted(pend.items())
    cut = int(len(items) * 0.6)
    reserve = items[cut:]
    ports = t["jobs"].col("ports")
    max_ports = int(ports.max()) if ports is not None else 0
    prm = traces.match_params(1000, host_lifetime_mins=t.get("host_lifetime_mins", 0))
    p = Pool("offers", send_hosts=True, send_lists=True, users=users)
    s = Stream(tmpl, rng, k8s_share)
    book = LeaseBook()
    now, tid, placed, fates = START, 10 ** 9, 0, set()
    try:
        p.apply(up=items[:cut], run_up=list(run.values()), reset=True)
        for c in range(n_cycles):
            now += 5_000          # every lease meets the incubation boundary exactly, three cycles on
            add(p.gpu, book, s.batch(int(tmpl.n * 0.4), crumbs=3), now, s.W)
            if reserve_hosts and c % 3 == 1:   # reservations on some VMs
                js = sorted(p.pend)[:6]
                p.patch(js, reserved_host=np.array([int(x) for x in rng.choice(codes, len(js))], np.int32))
            p.rank()
            got, _ = cycle(p, book, now, prm, groups=groups, max_ports=max_ports)
            fates |= {f for _, f in got["gone"]}
            tid, k = launch_some(p, got, tid, 80)
            placed += k
            fin = [x for x in p.run if rng.random() < 0.03]
            new = [reserve.pop() for _ in range(min(len(reserve), len(fin) + 30))]
            p.apply(up=new, run_rm=fin)
        assert placed > 0 and fates == {abi.OFFER_USED, abi.OFFER_EXPIRED, abi.OFFER_SINGLE_SHOT}
    finally:
        p.close()


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_c2_churn():
    run_churn(traces.gen_pool(41, 3000, 200, 30, 600), 3, 12, k8s_share=0.2)


@pytest.mark.gpu
def test_c3_churn_with_groups_and_reservations():
    t = traces.gen_c3_pool(17, n_jobs=2500, n_offers=160, n_users=24, n_running=500)
    run_churn(t, 5, 12, groups=t["groups"], reserve_hosts=True)


def small_pool(rng):
    t = traces.gen_pool(11, 300, 20, 6, 60)
    pend, run = pool_rows(t)
    codes = t["offers"].col("hostname_id")
    for r in run.values():
        r["host"] = int(rng.choice(codes))
        r["groups"] = []
    p = Pool("offers-small", send_hosts=True, send_lists=True, users=t["users"])
    p.apply(up=sorted(pend.items()), run_up=list(run.values()), reset=True)
    return p, Stream(t["offers"], rng)


@pytest.mark.gpu
def test_errors_leave_the_handle_unchanged():
    rng = np.random.default_rng(23)
    p, s = small_pool(rng)
    book = LeaseBook()
    prm = traces.match_params(100)
    now = START
    try:
        add(p.gpu, book, s.batch(10), now, 0)
        live = book.leases[0]
        named = set(s.named)
        fresh = s.batch(3)
        s.named = named   # none of these reach the handle
        bad = [
            [dict(fresh[0], id=live["id"])],                                   # an id already live
            [fresh[0], dict(fresh[1], id=fresh[0]["id"])],                     # an id twice in the batch
            [dict(fresh[0], code=-1)],                                         # a negative code
            [dict(fresh[0], code=99_999, hostname="new-host", name="")],       # a new code without a name
            [dict(fresh[0], name=live["hostname"] + "-other", code=live["code"])],   # a known code, another name
            [dict(fresh[0], code=99_998, hostname=live["hostname"], name=live["hostname"])],   # one name, two codes
            [dict(fresh[0], code=99_997, hostname="n1", name="n1"), dict(fresh[1], code=99_996, hostname="n1",
                                                                         name="n1")],
        ]
        for leases in bad:
            soa, ids, single, gpus, names = offers_soa(leases, 0)
            with pytest.raises(CookError) as ei:
                p.gpu.state_offers_add(soa, ids, now, single_shot=single, offer_gpus=gpus, hostnames=names)
            assert ei.value.code == abi.COOK_E_BADARG
        # a malformed port CSR
        soa, ids, single, gpus, names = offers_soa(fresh[:2], 0)
        soa = with_fields(soa, port_off=np.array([0, 3, 1], np.int32), port_begin=np.zeros(3, np.int32),
                          port_end=np.zeros(3, np.int32))
        with pytest.raises(CookError):
            p.gpu.state_offers_add(soa, ids, now, hostnames=names)
        p.rank()
        for kw in (dict(incubate_ms=0), dict(gone_cap=len(book.leases) - 1)):
            with pytest.raises(CookError) as ei:
                p.gpu.state_match_offers(now, kw.get("incubate_ms", INCUBATE), p.users, prm,
                                         gone_cap=kw.get("gone_cap"))
            assert ei.value.code == abi.COOK_E_BADARG
        reuse = traces.match_params(100)
        reuse.reuse_resident = 1
        with pytest.raises(CookError):
            p.gpu.state_match_offers(now, INCUBATE, p.users, reuse)
        # nothing changed: the next cycle equals the restatement
        cycle(p, book, now + 1_000, prm)
        # reset drops the offers
        add(p.gpu, book, s.batch(5), now + 2_000, 0)
        p.apply(up=sorted(p.pend.items()), run_up=list(p.run.values()), reset=True)
        book.drop_all()
        p.rank()
        got, codes = cycle(p, book, now + 3_000, prm)
        assert len(codes) == 0 and got["gone"] == [] and (got["assign"] == -1).all()
    finally:
        p.close()


@pytest.mark.gpu
def test_no_queue_still_expires_and_drops_single_shot():
    rng = np.random.default_rng(29)
    p, s = small_pool(rng)
    book = LeaseBook()
    try:
        leases = s.batch(8)
        for l in leases[:3]:
            l["single_shot"] = True
        add(p.gpu, book, leases, START, 0)
        p.apply(rm=sorted(p.pend))
        p.rank()
        got, _ = cycle(p, book, START + INCUBATE - 1, traces.match_params(100))
        assert {f for _, f in got["gone"]} == {abi.OFFER_SINGLE_SHOT}
        got, _ = cycle(p, book, START + INCUBATE, traces.match_params(100))
        assert got["gone"] and {f for _, f in got["gone"]} == {abi.OFFER_EXPIRED} and not book.leases
    finally:
        p.close()


# ---- GPU: the rebalancer's spare resources from the live offers (config-#4 shape) -------------------------------
@pytest.mark.gpu
def test_c4_rebalance_offers():
    from resident_model import COT_FIELDS, decisions_eq, jobs_soa, rebalance_trace, rows_of, tasks_soa
    r, codes = rebalance_trace(23, True)
    rng = np.random.default_rng(31)
    g0, hosts = r["groups"], r["hosts"]
    G, H = g0.n_groups, hosts.n
    pend, run = rows_of(r, codes)
    for row in run.values():
        row["groups"] = [int(rng.integers(G))] if rng.random() < 0.2 else []
    p = Pool.of_rebalance(r, codes)
    book = LeaseBook()
    lid = [0]

    def leases(n_hosts, now):
        out = []
        for h in rng.choice(H, n_hosts, replace=False).tolist():
            for _ in range(int(rng.choice([1, 1, 2, 3]))):   # several leases per host, off the grid too
                out.append({"id": lid[0], "code": int(codes[h]), "hostname": f"node-{int(codes[h])}",
                            "cpus": float(rng.choice([0.5, 1.0, 2.1, 7.0])), "mem": float(rng.choice([512.0, 1000.3])),
                            "gpus": float(rng.choice([0.0, 1.0, 2.0]))})
                lid[0] += 1
        add(p.gpu, book, out, now, 0)

    dg = with_fields(g0, **{f: None for f in COT_FIELDS})
    bare = with_fields(hosts, has_spare=None, spare_cpus=None, spare_mem=None, spare_gpus=None)
    try:
        run_up = list(run.values())
        pj, pp, jid = jobs_soa(sorted(pend.items()))
        off, idx = abi.csr([x["groups"] for x in run_up])
        p.gpu.state_apply(abi.make_delta(reset=True, pending=pj, pending_priority=pp, pending_job_id=jid,
                                         running=tasks_soa(run_up),
                                         running_hostname_id=np.array([x["host"] for x in run_up], np.int32),
                                         running_group_off=off, running_group_idx=idx))
        p.pend, p.run = dict(pend), dict(run)
        differs = 0
        for step in range(4):
            leases(H // 3, START + step)
            p.rank()
            sp = book.spare(codes)
            assert sp["has_spare"].sum() > 0 and (sp["spare_gpus"] > 0).any()
            want = p.gpu.state_rebalance(with_fields(hosts, **sp), p.users, p.rparams, groups=dg, derived=True)
            sw = p.gpu.last_stats(abi.PHASE_REBALANCE)
            got = p.gpu.state_rebalance(bare, p.users, p.rparams, groups=dg, offers=True)
            sd = p.gpu.last_stats(abi.PHASE_REBALANCE)
            decisions_eq(got, want)
            assert got
            assert sd["h2d_bytes"] == sw["h2d_bytes"] - 25 * H and sd["d2h_bytes"] == sw["d2h_bytes"]
            none = p.gpu.state_rebalance(with_fields(hosts, has_spare=np.zeros(H, np.uint8)), p.users, p.rparams,
                                         groups=dg, derived=True)
            differs += [(d["job_id"], d["host"]) for d in none] != [(d["job_id"], d["host"]) for d in got]
            p.apply(run_rm=[t for t in p.run if rng.random() < 0.1])
        assert differs   # the spare resources decide some placements
        # a host with a live lease that the table does not list
        add(p.gpu, book, [{"id": 10 ** 6, "code": 10 ** 6, "hostname": "not-listed", "cpus": 1.0, "mem": 1.0}],
            START + 9, 0)
        with pytest.raises(CookError) as ei:
            p.gpu.state_rebalance(bare, p.users, p.rparams, groups=dg, offers=True)
        assert ei.value.code == abi.COOK_E_BADARG
    finally:
        p.close()


# ---- GPU: K15 (handle-resource-offers!, scheduler.clj:1947-2133) through the resident path ----------------------
def k15_cycle(offer_ids, nc, queue_prio=None, reserved=None, extra=None, **kw):
    """The K15 fixture as a resident pool: the eight jobs (job id = index), the user's usage as one running task, the
    Mesos offers host-i (code i) added once; one PoolCycle.handle_resource_offers_resident."""
    from cycle_golden_cases import _users
    from handle_offers_golden_cases import JOBS, MESOS, P100
    from cook_b200.cycle import PoolCycle
    from resident_model import DEFAULTS
    users = with_fields(_users(), usage_count=None, usage_cpus=None, usage_mem=None, usage_gpus=None)
    p = Pool("k15", send_hosts=True, users=users)
    try:
        rows = []
        for j, (c, m, g, _, _) in enumerate(JOBS):
            if queue_prio is not None and j not in queue_prio:
                continue
            rows.append((j, dict(DEFAULTS, user=0, priority=queue_prio[j] if queue_prio else 50, cpus=float(c),
                                 mem=float(m), gpus=float(g), gpu_model=P100,
                                 reserved_host=(reserved or {}).get(j, -1), novel=[], attr=[], groups=[])))
        for j, r in (extra or {}).items():
            rows.append((j, dict(DEFAULTS, user=0, priority=50, novel=[], attr=[], groups=[], **r)))
        task = dict(user=0, priority=50, start_time=START, task_id=1, job_id=10 ** 6, cpus=2.0, mem=1024.0, gpus=0.0,
                    host=-1, groups=[])
        p.apply(up=rows, run_up=[task])
        pc = PoolCycle(p.gpu, max_considerable=nc)
        if reserved:
            pc.job_reserved_host = dict(reserved)
        if extra:
            pc.job_reserved_host.update({j: r["reserved_host"] for j, r in extra.items()})
        leases = [{"id": 100 + i, "code": i, "hostname": f"host-{i}", "cpus": float(MESOS[i][0]),
                   "mem": float(MESOS[i][1])} for i in offer_ids]
        soa, ids, _, _, names = offers_soa(leases)
        pc.add_offers(soa, ids, START, hostnames=names)
        p.rank()
        r = pc.handle_resource_offers_resident(START, users, **kw)
        for mt in r["matches"]:
            assert mt["leases"] == [100 + mt["hostname_id"]]
        assert not r["decline"] and not r["dropped"]
        return r, pc
    finally:
        p.close()


@pytest.mark.gpu
def test_k15_through_the_resident_path():
    # :1957-1964 enough offers, nc 6: true, 4 jobs on 3 offers
    r, _ = k15_cycle([1, 2, 3], 6)
    assert r["matched_head_or_no_matches"] is True and r["launched_jobs"] == {0, 1, 2, 3}
    assert len(r["launched_offers"]) == 3 and r["next_considerable"] == 6
    # :1966-1982 limited by num-considerable 1 / 2
    for nc, want in ((1, {0}), (2, {0, 1})):
        r, _ = k15_cycle([1, 2, 3], nc)
        assert r["matched_head_or_no_matches"] and r["launched_jobs"] == want and len(r["launched_offers"]) == len(want)
    # :2015-2028 the cluster's launch-rate limiter is enforcing and in debt: nothing launches, true; the leases of the
    # dropped matches come back to be declined
    r, pc = k15_cycle([1, 2, 3], 10, cluster_of_host={1: "cc", 2: "cc", 3: "cc"}, cluster_tokens={"cc": -1},
                      cluster_enforce={"cc": True})
    assert r["matched_head_or_no_matches"] is True and not r["launched_jobs"] and not r["launched_offers"]
    assert sorted(r["unlaunched"]) == [101, 102, 103] and pc.num_considerable == 10
    # :2002-2013 limiter with tokens left: nothing is dropped
    r, _ = k15_cycle([1, 2, 3], 6, cluster_of_host={1: "cc", 2: "cc", 3: "cc"}, cluster_tokens={"cc": 1},
                     cluster_enforce={"cc": True})
    assert r["launched_jobs"] == {0, 1, 2, 3}
    # :2086-2092 an offer that fits no job: true, nothing launches
    r, _ = k15_cycle([5], 10)
    assert r["matched_head_or_no_matches"] is True and not r["launched_jobs"]
    # :2112-2119 a host reserved for somebody else's job (job 99, not allowed to start): nothing launches
    r, pc = k15_cycle([1], 10, extra={99: dict(cpus=1.0, mem=1.0, allowed=0, reserved_host=1)})
    assert not r["launched_jobs"] and pc.job_reserved_host == {99: 1}
    # :2121-2133 only the jobs the host is reserved for launch there; their reservations are released
    r, pc = k15_cycle([9], 10, reserved={0: 9, 1: 9})
    assert r["launched_jobs"] == {0, 1} and pc.job_reserved_host == {} and pc.launched_jobs == {0, 1}
    # the head (job 1, 13 cpus) does not fit offer-1 (10 cpus) but job 0 does: false, fewer jobs next cycle
    r, _ = k15_cycle([1], 1000, queue_prio={1: 90, 0: 80, 2: 70, 3: 60})
    assert r["matched_head_or_no_matches"] is False and r["launched_jobs"] == {0} and r["next_considerable"] == 950
