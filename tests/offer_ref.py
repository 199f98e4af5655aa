"""Plain-Python restatement of the live offers cook_state_offers_add and cook_state_match_offers keep: Fenzo's leases
(scheduler.clj:617-687, :2301-2324) with the rules include/cook_gpu.h states.

A lease is a dict: id, hostname (str), code (its hostname code), cpus, mem, and optionally gpus (the "gpus" scalar),
ports [(begin, end)], single_shot, is_k8s, location, max_tasks, num_tasks, host_start_time, gpu [(model, count)],
disk [(type, MiB)] and attr [value per column].  `LeaseBook` adds the arrival number and the receive time, expires,
merges into the cook_offers_soa the device builds, and consumes after a match.  It follows cook_b200.cycle.OfferCache
(expire, after_match) and offers_from_cache (cpus, mem, ports), which the CPU tests pin it on.
"""
import numpy as np

from cook_b200 import abi

ABSENT = dict(gpus=0.0, is_k8s=0, location=-1, max_tasks=-1, num_tasks=0, host_start_time=-1)


def name_key(name):
    """The VM order: memcmp order of the hostname bytes."""
    return name.encode() if isinstance(name, str) else bytes(name)


class LeaseBook:
    def __init__(self):
        self.leases = []   # live, in arrival order
        self.seq = 0

    def add(self, leases, now_ms, n_attr_cols=0):
        """One cook_state_offers_add batch: every row is n_attr_cols attribute columns wide."""
        for l in leases:
            a = list(l.get("attr", []))[:n_attr_cols]
            self.leases.append(dict(l, attr=a + [0] * (n_attr_cols - len(a)), seq=self.seq, received_ms=now_ms))
            self.seq += 1

    def drop_all(self):
        self.leases = []

    def expire(self, now_ms, incubate_ms):
        """OfferCache.expire's rule: leases with now - received >= incubate leave."""
        old = [l for l in self.leases if now_ms - l["received_ms"] >= incubate_ms]
        self.leases = [l for l in self.leases if now_ms - l["received_ms"] < incubate_ms]
        return old

    def vms(self):
        """{hostname: its live leases in arrival order}, hostnames in byte order."""
        by = {}
        for l in self.leases:
            by.setdefault(l["hostname"], []).append(l)
        return {h: by[h] for h in sorted(by, key=name_key)}

    def merged(self, pending_attr_cols=(), group_attr_cols=(), reserved_codes=None):
        """The table cook_state_match_offers matches against, after its expiry: (VM codes in name order, OffersSoA).
        pending_attr_cols: the attribute columns live pending rows name; reserved_codes: the reserved_host codes of the
        live pending rows (None: no row has one, so the table has no reserved column)."""
        vms = self.vms()
        groups = list(vms.values())
        O = len(groups)
        newest = [g[-1] for g in groups]
        codes = np.array([g[0]["code"] for g in groups], np.int32)
        cpus, mem = np.zeros(O), np.zeros(O)
        for v, g in enumerate(groups):
            c = m = 0.0
            for l in g:   # left folds in arrival order
                c = c + l["cpus"]
                m = m + l["mem"]
            cpus[v], mem[v] = c, m
        kw = dict(hostname_id=codes, name_rank=np.arange(O, dtype=np.int32), cpus=cpus, mem=mem,
                  run_cpus=np.zeros(O), run_mem=np.zeros(O), run_count=np.zeros(O, np.int32))
        if any(l.get("ports") for l in self.leases):
            kw["port_off"], kw["port_begin"] = abi.csr([[r[0] for l in g for r in l.get("ports", [])] for g in groups])
            kw["port_end"] = abi.csr([[r[1] for l in g for r in l.get("ports", [])] for g in groups])[1]

        def col(key, dt):
            return np.array([l.get(key, ABSENT[key]) for l in newest], dt)

        if any(l.get("is_k8s", 0) for l in newest):
            kw["is_k8s"] = col("is_k8s", np.uint8)
        kw["location"] = col("location", np.int32)
        kw["num_tasks"] = col("num_tasks", np.int32)
        kw["host_start_time"] = col("host_start_time", np.int64)
        if any(l.get("max_tasks", -1) != -1 for l in newest):
            kw["max_tasks"] = col("max_tasks", np.int32)
        for key, a, b in (("gpu", "gpu_model", "gpu_count"), ("disk", "disk_type", "disk_space")):
            if any(l.get(key) for l in newest):
                off, first = abi.csr([[e[0] for e in l.get(key, [])] for l in newest])
                kw[key + "_off"], kw[a] = off, first
                kw[b] = abi.csr([[e[1] for e in l.get(key, [])] for l in newest], np.float64)[1]
        W = max([len(l.get("attr", [])) for l in self.leases] + [c + 1 for c in pending_attr_cols] +
                [c + 1 for c in group_attr_cols] + [0])
        if W > 0:
            attr = np.zeros((W, O), np.int32)
            for v, l in enumerate(newest):
                a = l.get("attr", [])
                attr[:len(a), v] = a
            kw["attr"] = attr.reshape(-1)
        if reserved_codes is not None:
            rs = set(reserved_codes)
            kw["reserved"] = np.array([1 if int(c) in rs else 0 for c in codes], np.uint8)
        return codes, abi.OffersSoA(n=O, n_attr_cols=W, **kw)

    def spare(self, host_codes):
        """The spare resources cook_state_rebalance_offers derives (view-incubating-offers): has_spare, spare_cpus,
        spare_mem and spare_gpus at each index of a host table with these hostname codes, left folds in arrival
        order of the host's live leases' cpus, mem and gpus scalar."""
        idx = {int(c): i for i, c in enumerate(host_codes)}
        H = len(host_codes)
        has, out = np.zeros(H, np.uint8), {k: np.zeros(H) for k in ("cpus", "mem", "gpus")}
        for l in self.leases:
            h = idx[l["code"]]
            has[h] = 1
            for k in out:
                out[k][h] = out[k][h] + l.get(k, 0.0)
        return dict(has_spare=has, spare_cpus=out["cpus"], spare_mem=out["mem"], spare_gpus=out["gpus"])

    def after_match(self, used_codes):
        """OfferCache.after_match's rule: every lease of a host with an assignment is consumed, every remaining
        single-shot lease dropped.  Returns (consumed, dropped)."""
        used = set(int(c) for c in used_codes)
        consumed = [l for l in self.leases if l["code"] in used]
        dropped = [l for l in self.leases if l["code"] not in used and l.get("single_shot")]
        self.leases = [l for l in self.leases if l["code"] not in used and not l.get("single_shot")]
        return consumed, dropped


def gone_list(expired, consumed, dropped):
    """The gone list cook_state_match_offers writes: (offer id, fate) in arrival order."""
    gone = [(l, abi.OFFER_EXPIRED) for l in expired] + [(l, abi.OFFER_USED) for l in consumed] + \
           [(l, abi.OFFER_SINGLE_SHOT) for l in dropped]
    return [(l["id"], f) for l, f in sorted(gone, key=lambda x: x[0]["seq"])]


def offers_soa(leases, n_attr_cols=0):
    """The rows cook_state_offers_add takes for `leases` (one batch: every row n_attr_cols wide), with the offer ids,
    single-shot flags, gpus scalars and hostnames."""
    n = len(leases)

    def col(key, dt):
        return np.array([l.get(key, ABSENT[key]) for l in leases], dt)

    kw = dict(hostname_id=np.array([l["code"] for l in leases], np.int32), cpus=col_f(leases, "cpus"),
              mem=col_f(leases, "mem"), is_k8s=col("is_k8s", np.uint8), location=col("location", np.int32),
              max_tasks=col("max_tasks", np.int32), num_tasks=col("num_tasks", np.int32),
              host_start_time=col("host_start_time", np.int64))
    if any(l.get("ports") for l in leases):
        kw["port_off"], kw["port_begin"] = abi.csr([[r[0] for r in l.get("ports", [])] for l in leases])
        kw["port_end"] = abi.csr([[r[1] for r in l.get("ports", [])] for l in leases])[1]
    for key, a, b in (("gpu", "gpu_model", "gpu_count"), ("disk", "disk_type", "disk_space")):
        if any(l.get(key) for l in leases):
            kw[key + "_off"], kw[a] = abi.csr([[e[0] for e in l.get(key, [])] for l in leases])
            kw[b] = abi.csr([[e[1] for e in l.get(key, [])] for l in leases], np.float64)[1]
    if n_attr_cols:
        attr = np.zeros((n_attr_cols, n), np.int32)
        for i, l in enumerate(leases):
            a = l.get("attr", [])
            attr[:len(a), i] = a
        kw["attr"] = attr.reshape(-1)
    soa = abi.OffersSoA(n=n, n_attr_cols=n_attr_cols, **kw)
    ids = np.array([l["id"] for l in leases], np.int64)
    single = np.array([1 if l.get("single_shot") else 0 for l in leases], np.uint8)
    return soa, ids, single, col("gpus", np.float64), [l.get("name", l["hostname"]) for l in leases]


def col_f(leases, key):
    return np.array([float(l[key]) for l in leases], np.float64)
