"""Host side of the match cycle above the C ABI: SURVEY rows M5 and M6.

This is the state machine `cook.scheduler.gpu` (clj/cook/scheduler/gpu.clj, the JVM shim) runs
around `cook_match`; the Python form exists because the reference toolchain is absent here and
because the reference's own `handle-resource-offers!` known answers (K15) then run through the CUDA
path end to end.  It computes nothing numeric: every placement decision is `engine.match`.

  OfferCache            what Fenzo kept between cycles (scheduler.clj:617-687, :2301-2324): live Mesos
                        leases merged per hostname, offer expiry after `offer-incubate-time-ms`,
                        single-shot (Kubernetes) offers dropped after every match attempt
  PoolCycle             handle-resource-offers! (:1339-1535): considerable jobs -> match ->
                        per-cluster launch-rate filter (:887-924) -> matched jobs leave the queue
                        (:790-795) -> reservations released (:1050-1057) -> head-matched feedback
                        + num-considerable scale-back / reset (handle-fenzo-pool :1613-1651); its resident
                        form takes the offers the library keeps (cook_state_match_offers) and turns the
                        offers that left into the matches' leases, the declines and the dropped ones
  summarize_failures    fenzo_utils.clj:45-89 shape from cook_match_failures' counters (8f-3)
  resync                the audit of a resident pool fed by deltas: bucket fingerprints compared with the host's,
                        the differing buckets exported, the repairing delta built
  monitor_stats         the counters set-stats-counters! (monitor.clj:177-207) sets, from cook_state_user_stats
  queue_lengths         jobs->queue-lengths (queue_limit.clj:64-90), from single-pool cook_state_user_stats calls
  unscheduled_reasons   reasons (unscheduled.clj:172-200) of a resident pool's job from cook_state_unscheduled and the
                        host's limit maps and facts; Investigations, the host half of record-placement-failures!
  usage_response        the body of GET /usage (get-user-usage, api.clj:2946-2969) from cook_state_user_usage answers
  instance_stats_response  the body of GET /stats/instances (task-stats/get-stats) from a cook_state_instance_stats
                        answer
  match_cycle_metrics_response  the match-cycle logs (handle-match-cycle-metrics) and the unmatched-too-long warning
                        from a cook_state_match_metrics answer
  list_jobs_response    the jobs GET /list and GET /jobs list (get-jobs-by-user-and-states, list-job-ents) from a
                        cook_state_list_jobs answer and the states the Datomic path answers
"""
import numpy as np

from . import abi, traces
from .engine import STATS_KEYS

CONSTRAINT_NAMES = [  # Cook's evaluation order (constraints.clj:459-495; defrecord class names)
    "checkpoint_locality_constraint", "estimated_completion_constraint", "user_defined_constraint",
    "disk_host_constraint", "gpu_host_constraint", "novel_host_constraint", "max_tasks_per_host",
    "rebalancer_reservation_constraint", "unique_host_placement_group_constraint",
    "balanced_host_placement_group_constraint", "attribute_equals_host_placement_group_constraint"]
RESOURCE_NAMES = ["cpus", "mem"]   # the scalar requests whose AssignmentFailure carries a message (fenzo_utils.clj:21-44)


def summarize_failures(counts):
    """cook_match_failures counters of one job -> {:resources {"cpus" n "mem" n} :constraints {name n}}
    (summarize-placement-failure, fenzo_utils.clj:45-57), zero entries omitted like `(fnil inc 0)`."""
    c = [int(x) for x in counts]
    res = {n: c[i] for i, n in enumerate(RESOURCE_NAMES) if c[i]}
    con = {n: c[2 + i] for i, n in enumerate(CONSTRAINT_NAMES) if c[2 + i]}
    out = {}
    if res:
        out["resources"] = res
    if con:
        out["constraints"] = con
    return out


class OfferCache:
    """Fenzo's lease bookkeeping that the stateless cook_match leaves to the host (M5): unused Mesos
    offers stay live - merged per hostname with later ones - until `incubate_ms` pass (then they are
    declined, scheduler.clj:2315-2323); offers with reject_after_match_attempt (Kubernetes: offers are
    regenerated from node state every cycle) never survive a match attempt (:674-678)."""

    def __init__(self, incubate_ms=15_000):
        self.incubate_ms = incubate_ms
        self.leases = []   # dicts: hostname, cpus, mem, ports [(b, e)], received_ms, single_shot, cluster, id

    def add(self, offers, now_ms):
        for o in offers:
            self.leases.append(dict(o, received_ms=o.get("received_ms", now_ms)))

    def expire(self, now_ms):
        """Leases older than the incubation time are declined; returns them."""
        old = [l for l in self.leases if now_ms - l["received_ms"] >= self.incubate_ms]
        self.leases = [l for l in self.leases if now_ms - l["received_ms"] < self.incubate_ms]
        return old

    def merged(self):
        """One assignable VM per hostname = the sum of its live leases (FENZO rule 1), in first-seen
        order; returns (hostnames, per-host lease lists)."""
        by = {}
        for l in self.leases:
            by.setdefault(l["hostname"], []).append(l)
        return list(by), list(by.values())

    def after_match(self, used_hostnames):
        """Leases of hosts that got an assignment are consumed (FENZO rule 7); single-shot leases
        are expired whether used or not.  Returns (consumed, expired_unused)."""
        used = set(used_hostnames)
        consumed = [l for l in self.leases if l["hostname"] in used]
        dropped = [l for l in self.leases if l["hostname"] not in used and l.get("single_shot")]
        self.leases = [l for l in self.leases if l["hostname"] not in used and not l.get("single_shot")]
        return consumed, dropped


def next_considerable(num_considerable, matched_head_or_no_matches, max_considerable, scaleback,
                      iterations_at_floor, floor_iterations_before_reset):
    """handle-fenzo-pool (scheduler.clj:1613-1651): the head of the queue not matched => fewer jobs
    next cycle, max(1, floor(scaleback * n)); after `floor_iterations_before_reset` cycles at 1 the
    pool gives up and shows Fenzo max-considerable jobs again.
    Returns (num_considerable for the next cycle, iterations_at_floor)."""
    nxt = max_considerable if matched_head_or_no_matches else max(1, int(scaleback * num_considerable))
    iterations_at_floor = iterations_at_floor + 1 if nxt == 1 else 0
    if iterations_at_floor >= floor_iterations_before_reset:
        return max_considerable, iterations_at_floor
    return nxt, iterations_at_floor


class PoolCycle:
    """handle-resource-offers! for one pool, around an engine with GpuEngine's `match` signature."""

    def __init__(self, engine, max_considerable=1000, scaleback=0.95, floor_iterations_before_warn=10,
                 floor_iterations_before_reset=1000, incubate_ms=15_000):
        self.eng = engine
        self.max_considerable = max_considerable
        self.num_considerable = max_considerable
        self.scaleback = scaleback
        self.floor_iterations_before_warn = floor_iterations_before_warn
        self.floor_iterations_before_reset = floor_iterations_before_reset
        self.iterations_at_floor = 0
        self.offers = OfferCache(incubate_ms)
        # rebalancer-reservation-atom (rebalancer.clj:419-432, scheduler.clj:1050-1057)
        self.job_reserved_host = {}     # job index -> hostname id
        self.launched_jobs = set()
        self.unmatched_cycles = {}      # job -> consecutive cycles considered but unmatched (:1400-1470)
        self.offer_host = {}            # resident pools: live offer id -> hostname code

    # ---- M6 ------------------------------------------------------------------------------------
    def handle_resource_offers(self, queue, jobs, offers, users, *, num_considerable=None, groups=None,
                               pool_quota=None, max_ports=0, host_lifetime_mins=0, enforce_rate_limit=0,
                               cluster_of_offer=None, cluster_tokens=None, cluster_enforce=None):
        """One cycle.  `queue`: ranked job indices (cook_rank output); `offers`: an OffersSoA of ALL
        live offers merged per host (build it from OfferCache.merged()).  Returns a dict with
        :matches [{hostname_id, offer, jobs}], launched job / offer sets, the queue without the
        matched jobs, and `matched_head_or_no_matches` (the function's return value in the
        reference)."""
        nc = self.num_considerable if num_considerable is None else num_considerable
        queue = np.ascontiguousarray(queue, np.int32)
        single_shot = offers.col("reserved") is not None and False   # single-shot is a property of the cache entries
        J = jobs.n
        # jobs reserved a host by the rebalancer may use it; everybody else must keep off reserved hosts
        reserved_hosts = set(self.job_reserved_host.values())
        rh = np.full(J, -1, np.int32)
        for j, h in self.job_reserved_host.items():
            if 0 <= j < J:
                rh[j] = h
        hid = offers.col("hostname_id")
        res_col = np.array([1 if int(h) in reserved_hosts else 0 for h in hid], np.uint8) if reserved_hosts else None
        jobs_c, offers_c = jobs, offers
        if reserved_hosts:
            jk = {n: jobs.col(n) for n, _ in jobs._fields_ if jobs.col(n) is not None}
            jk["reserved_host"] = rh
            jobs_c = abi.JobsSoA(n=J, **jk)
            ok = {n: offers.col(n) for n, _ in offers._fields_ if offers.col(n) is not None}
            ok["reserved"] = res_col
            offers_c = abi.OffersSoA(n=offers.n, n_attr_cols=offers.n_attr_cols, **ok)
        if len(queue) == 0 or offers.n == 0 or nc <= 0:
            # :627-635 nothing to consider (and nothing a match attempt could change)
            return self._finish(queue, [], set(), set(), True, 0, nc)
        prm = traces.match_params(min(nc, len(queue)), enforce_rate_limit=enforce_rate_limit,
                                  host_lifetime_mins=host_lifetime_mins)
        m = self.eng.match(queue, jobs_c, offers_c, users, prm, groups=groups, pool_quota=pool_quota,
                           max_ports=max_ports)
        cons, assign = m["considerable"], m["assign"]
        by_offer = {}
        for k in range(len(cons)):
            if assign[k] >= 0:
                by_offer.setdefault(int(assign[k]), []).append(int(cons[k]))
        matches = [{"offer": o, "hostname_id": int(hid[o]), "jobs": js,
                    "ports": {int(cons[k]): [int(p) for p in m["ports"][k] if p >= 0]
                              for k in range(len(cons)) if assign[k] == o}}
                   for o, js in by_offer.items()]
        # filter-matches-for-ratelimit (:887-924): a compute cluster whose launch-rate limiter is
        # enforcing and in debt loses ALL its matches of this cycle
        if cluster_of_offer is not None and cluster_tokens is not None:
            def skipped(o):
                c = cluster_of_offer[o]
                enf = True if cluster_enforce is None else bool(cluster_enforce.get(c, False))
                return enf and cluster_tokens.get(c, 0) < 0
            matches = [mt for mt in matches if not skipped(mt["offer"])]
        matched_jobs = {j for mt in matches for j in mt["jobs"]}
        head = int(cons[0]) if len(cons) else None
        matched_head = head is not None and head in matched_jobs
        no_matches = len(matches) == 0
        return self._finish(queue, matches, matched_jobs, {mt["offer"] for mt in matches},
                            no_matches or matched_head, len(cons), nc, considerable=[int(c) for c in cons],
                            fail=m["fail"])

    # ---- M5 + M6 for a resident pool: the offers live in the library (cook_state_offers_add / _match_offers) ----
    def add_offers(self, offers, offer_id, now_ms, **kw):
        """cook_state_offers_add (engine.state_offers_add's keywords), remembering each offer's hostname code: the
        match reports the offers that left by id."""
        self.eng.state_offers_add(offers, offer_id, now_ms, **kw)
        self.offer_host.update(zip(np.asarray(offer_id).tolist(), offers.col("hostname_id").tolist()))

    def handle_resource_offers_resident(self, now_ms, users, *, num_considerable=None, groups=None, pool_quota=None,
                                        max_ports=0, host_lifetime_mins=0, enforce_rate_limit=0, cluster_of_host=None,
                                        cluster_tokens=None, cluster_enforce=None):
        """One cycle of a resident pool (after its deltas and cook_state_rank): cook_state_match_offers with the
        pool's incubation time, then the reference's shape of the result.  Returns handle_resource_offers' dict, with
        job ids for jobs and hostname codes for hosts, where each match is {hostname_id, leases (the USED offer ids of
        the host, for launch-tasks), jobs, ports}, plus 'decline' (the EXPIRED offer ids: the lease reject action),
        'dropped' (the SINGLE_SHOT ones) and 'unlaunched' (the leases of the matches the launch-rate filter dropped;
        they are consumed, so the caller declines them too).  cluster_of_host: hostname code -> compute cluster."""
        nc = self.num_considerable if num_considerable is None else num_considerable
        prm = traces.match_params(max(nc, 0), enforce_rate_limit=enforce_rate_limit,
                                  host_lifetime_mins=host_lifetime_mins)
        m = self.eng.state_match_offers(now_ms, self.offers.incubate_ms, users, prm, groups=groups,
                                        pool_quota=pool_quota, max_ports=max_ports)
        leases, decline, dropped = {}, [], []
        for oid, fate in m["gone"]:
            code = self.offer_host.pop(oid)
            if fate == abi.OFFER_USED:
                leases.setdefault(code, []).append(oid)
            elif fate == abi.OFFER_EXPIRED:
                decline.append(oid)
            else:
                dropped.append(oid)
        cons, assign = m["considerable"], m["assign"]
        by_host = {}
        for k in range(len(cons)):
            if assign[k] >= 0:
                by_host.setdefault(int(assign[k]), []).append(k)
        matches = [{"hostname_id": h, "leases": leases[h], "jobs": [int(cons[k]) for k in ks],
                    "ports": {int(cons[k]): [int(p) for p in m["ports"][k] if p >= 0] for k in ks}}
                   for h, ks in by_host.items()]
        unlaunched = []
        if cluster_of_host is not None and cluster_tokens is not None:   # filter-matches-for-ratelimit (:887-924)
            def skipped(h):
                c = cluster_of_host[h]
                enf = True if cluster_enforce is None else bool(cluster_enforce.get(c, False))
                return enf and cluster_tokens.get(c, 0) < 0
            unlaunched = [l for mt in matches if skipped(mt["hostname_id"]) for l in mt["leases"]]
            matches = [mt for mt in matches if not skipped(mt["hostname_id"])]
        matched_jobs = {j for mt in matches for j in mt["jobs"]}
        head = int(cons[0]) if len(cons) else None
        ok = len(matches) == 0 or (head is not None and head in matched_jobs)
        r = self._finish(np.zeros(0, np.int32), matches, matched_jobs, {mt["hostname_id"] for mt in matches}, ok,
                         len(cons), nc, considerable=[int(c) for c in cons], fail=m["fail"])
        del r["queue"]   # the queue is the resident one: the launches take the matched jobs out of it
        r.update(decline=decline, dropped=dropped, unlaunched=unlaunched, stats=m["stats"])
        return r

    def _finish(self, queue, matches, matched_jobs, used_offers, ok, n_considerable, nc, considerable=(), fail=None):
        if matches:
            # remove-matched-jobs-from-pending-jobs (:790-795), update-host-reservations! (:1050-1057)
            queue = np.array([j for j in queue if int(j) not in matched_jobs], np.int32)
            for j in matched_jobs:
                self.job_reserved_host.pop(j, None)
            self.launched_jobs |= matched_jobs
        # :1400-1470 consecutive unmatched cycles per considerable job (jobs that left the
        # considerable set are forgotten: no leak of historic jobs)
        self.unmatched_cycles = {j: self.unmatched_cycles.get(j, 0) + 1 for j in considerable if j not in matched_jobs}
        self.num_considerable, self.iterations_at_floor = next_considerable(
            nc, ok, self.max_considerable, self.scaleback, self.iterations_at_floor, self.floor_iterations_before_reset)
        return {"matches": matches, "launched_jobs": matched_jobs, "launched_offers": used_offers,
                "queue": queue, "matched_head_or_no_matches": ok, "n_considerable": n_considerable,
                "next_considerable": self.num_considerable,
                "failures": [j for j, f in zip(considerable, fail if fail is not None else []) if j not in matched_jobs]}

    # ---- rebalancer hand-over (rebalancer.clj:419-432 reserve-hosts!) -----------------------------
    def reserve_hosts(self, decisions, pending_job_index, host_hostname_id):
        """Decisions with more than one victim reserve their host for the job they make room for;
        jobs launched meanwhile are not reserved."""
        for d in decisions:
            j = int(pending_job_index[d["pending_idx"]])
            if len(d["victims"]) > 1 and j not in self.launched_jobs:
                self.job_reserved_host[j] = int(host_hostname_id[d["host"]])
        self.launched_jobs = set()


def offers_from_cache(cache, hostname_ids, *, k8s=None):
    """cook_offers_soa of everything live in the cache, one entry per hostname: cpus / mem summed
    over the host's leases, port ranges concatenated in lease order (FENZO rules 1 and 6)."""
    names, groups = cache.merged()
    O = len(names)
    cpus = np.array([sum(l["cpus"] for l in g) for g in groups], float)
    mem = np.array([sum(l["mem"] for l in g) for g in groups], float)
    pb = [[r[0] for l in g for r in l.get("ports", [])] for g in groups]
    pe = [[r[1] for l in g for r in l.get("ports", [])] for g in groups]
    port_off, port_begin = abi.csr(pb)
    _, port_end = abi.csr(pe)
    order = sorted(range(O), key=lambda i: names[i])
    rank = np.zeros(O, np.int32)
    for r, i in enumerate(order):
        rank[i] = r
    kw = {}
    if k8s is not None:
        kw["is_k8s"] = np.array([1 if k8s(n) else 0 for n in names], np.uint8)
    return names, abi.OffersSoA(n=O, hostname_id=np.array([hostname_ids[n] for n in names], np.int32), name_rank=rank,
                                cpus=cpus, mem=mem, run_cpus=np.zeros(O), run_mem=np.zeros(O),
                                run_count=np.zeros(O, np.int32), port_off=port_off, port_begin=port_begin,
                                port_end=port_end, n_attr_cols=0, **kw)


# ---- SURVEY §8f-4: autoscaling job selection (scheduler.clj:1283-1335) --------------------------
def max_jobs_for_autoscaling_scaled(number_considerable, number_unmatched, max_jobs_for_autoscaling, scale_factor):
    """`(-> fraction-unmatched (* scale-factor) (min 1) (* max-jobs) int (max number-unmatched))` with
    `fraction-unmatched = (/ (float unmatched) considerable)` (single precision, as in the reference)."""
    frac = float(np.float32(number_unmatched) / np.float32(number_considerable)) if number_considerable > 0 else 0.0
    return max(int(min(frac * scale_factor, 1.0) * max_jobs_for_autoscaling), number_unmatched)


def autoscalable_jobs(engine, queue_after_match, jobs, users, *, number_considerable, number_unmatched,
                      max_jobs_for_autoscaling=1000, scale_factor=1.0, pool_quota=None, enforce_rate_limit=0,
                      recent_synthetic_pod_jobs=()):
    """The quota-filtered prefix of the still-pending queue that autoscaling creates synthetic pods for:
    `filter-pending-jobs-for-quota` (user quota -> launch-rate tokens -> pool quota, tools.clj:961-973)
    over the queue WITHOUT the jobs just launched, `take` the scaled maximum, minus the jobs that got a
    synthetic pod recently.  The filter is M0 without `job-allowed-to-start?` / the launch plugin, so it
    runs on the device as a match against an EMPTY offer table (considerable set only, no matcher)."""
    n = max_jobs_for_autoscaling_scaled(number_considerable, number_unmatched, max_jobs_for_autoscaling, scale_factor)
    queue = np.ascontiguousarray(queue_after_match, np.int32)
    if n <= 0 or len(queue) == 0:
        return []
    jk = {c: jobs.col(c) for c in ("user", "cpus", "mem", "gpus") if jobs.col(c) is not None}
    plain = abi.JobsSoA(n=jobs.n, allowed=np.ones(jobs.n, np.uint8), plugin_accept=np.ones(jobs.n, np.uint8), **jk)
    empty = abi.OffersSoA(n=0, hostname_id=np.zeros(1, np.int32), name_rank=np.zeros(1, np.int32), cpus=np.zeros(1),
                          mem=np.zeros(1), run_cpus=np.zeros(1), run_mem=np.zeros(1), run_count=np.zeros(1, np.int32),
                          n_attr_cols=0)
    m = engine.match(queue, plain, empty, users, traces.match_params(min(n, len(queue)), enforce_rate_limit=enforce_rate_limit),
                     pool_quota=pool_quota)
    skip = set(recent_synthetic_pod_jobs)
    return [int(j) for j in m["considerable"] if int(j) not in skip]


def autoscalable_jobs_resident(engine, users, *, number_considerable, number_unmatched, max_jobs_for_autoscaling=1000,
                               scale_factor=1.0, pool_quota=None, enforce_rate_limit=0, recent_synthetic_pod_jobs=()):
    """autoscalable_jobs for a resident pool, after its cook_state_match(_derived) and the launches of the matched
    jobs: the same selection by cook_state_considerable with quota_only over the resident queue (the launched jobs
    have left it) and the usage the match read (COOK_USAGE_LAST_MATCH), so no job row or usage table crosses the bus.
    The scaled maximum and the recent-synthetic-pod skip stay here.  Returns job ids."""
    n = max_jobs_for_autoscaling_scaled(number_considerable, number_unmatched, max_jobs_for_autoscaling, scale_factor)
    if n <= 0:
        return []
    prm = abi.ConsiderableParams(n, int(enforce_rate_limit), 1, abi.USAGE_LAST_MATCH, 0)
    skip = set(recent_synthetic_pod_jobs)
    return [int(j) for j in engine.state_considerable(users, prm, pool_quota=pool_quota) if int(j) not in skip]


def resync(engine, host_digest_buckets, rows_of_bucket):
    """Audit a resident pool against the host's source of truth and build the delta that repairs it.

    host_digest_buckets: {"pending": [(sum, xor, n)] * n_buckets, "running": likewise}, the host's own bucket
    fingerprints (n_buckets a power of two).  rows_of_bucket(buckets) -> the host's rows of those buckets as the
    keyword arguments of abi.make_delta (pending / pending_priority / pending_job_id / running / ...).
    Returns (buckets, delta): the sorted differing buckets, and the abi.StateDelta that removes the device rows of
    those buckets the host does not have and upserts the host's rows there; (,) and None when nothing differs.  The
    caller applies it with engine.state_apply."""
    nb = len(host_digest_buckets["pending"])
    if nb == 0 or nb & (nb - 1) or len(host_digest_buckets["running"]) != nb:
        raise ValueError("resync: the bucket lists need one power-of-two length")
    dev = engine.state_digest(nb)
    diff = set()
    for table in ("pending", "running"):
        d = dev[table + "_buckets"]
        for b, want in enumerate(host_digest_buckets[table]):
            if (int(d["sum"][b]), int(d["xr"][b]), int(d["n"][b])) != tuple(int(x) for x in want):
                diff.add(b)
    if not diff:
        return [], None
    buckets = sorted(diff)
    mask = np.zeros(nb, np.uint8)
    mask[buckets] = 1
    held = engine.state_export(mask)
    want = dict(rows_of_bucket(buckets))
    wp, wr = want.get("pending_job_id"), want.get("running")
    host_jobs = set(np.asarray(wp, np.int64).tolist()) if wp is not None else set()
    host_tasks = set(wr.col("task_id").tolist()) if wr is not None and wr.n else set()
    want["pending_rm"] = [j for j in held["pending_job_id"].tolist() if j not in host_jobs]
    want["running_rm"] = [t for t in held["running"].col("task_id").tolist() if t not in host_tasks]
    return buckets, abi.make_delta(**want)


# ---- the monitor's user stats and the queue lengths from resident pools (SURVEY §8f-1) --------------------------
LONG_MAX = 2 ** 63 - 1


def counter_value(x):
    """What set-counter! (monitor.clj:118-123) stores: (long (min value Long/MAX_VALUE)), saturating at
    Long/MAX_VALUE and truncating toward zero."""
    if isinstance(x, (int, np.integer)):
        return min(int(x), LONG_MAX)
    x = float(x)
    return LONG_MAX if x >= 2.0 ** 63 else int(x)


def monitor_stats(stats, user_names, quota_extra=None):
    """The counters set-stats-counters! sets for one pool or quota-group name, from engine.state_user_stats over its
    handles: {state: {user name: {"jobs", "cpus", "mem", ...}}} for each of engine.STATS_KEYS, each with its "all"
    entry (add-aggregated-stats: {"cpus" 0 "mem" 0 "jobs" 0} when nobody is in the state), and "users": the five user
    counts.  Every value is the one set-counter! stores.
    quota_extra: per user code, the keys of the user's quota map beyond count, cpus and mem (gpus, the launch rates)
    by counter name.  A waiting-under-quota user's map carries them unchanged (the merges pass them through), and the
    state's "all" entry sums them over its users in ascending user code."""
    out = {}
    for s, state in enumerate(STATS_KEYS):
        users = np.flatnonzero((stats["member"] >> s) & 1)
        m = {}
        for u in users:
            e = {"jobs": int(stats["jobs"][s, u]), "cpus": float(stats["cpus"][s, u]), "mem": float(stats["mem"][s, u])}
            if s == abi.STATS_WUQ and quota_extra is not None:
                e.update({k: v for k, v in quota_extra[u].items() if k not in e})
            m[user_names[u]] = e
        if m:
            total = dict(zip(("jobs", "cpus", "mem"), stats["all"][state]))
            for e in m.values():
                for k, v in e.items():
                    if k not in ("jobs", "cpus", "mem"):
                        total[k] = total[k] + v if k in total else v
            m["all"] = total
        else:
            m["all"] = {"cpus": 0, "mem": 0, "jobs": 0}
        out[state] = {name: {k: counter_value(v) for k, v in e.items()} for name, e in m.items()}
    out["users"] = dict(stats["users"])
    return out


def queue_lengths(pool_stats, user_names):
    """jobs->queue-lengths from {pool name: engine.state_user_stats of that pool alone}: {"pool->queue-length":
    {pool: pending jobs}, "pool->user->queue-length": {pool: {user name: pending jobs}}}.  As group-by, a pool or user
    without a pending job has no entry."""
    per = {}
    for pool, st in pool_stats.items():
        w = np.flatnonzero((st["member"] >> abi.STATS_WAITING) & 1)
        if len(w):
            per[pool] = {user_names[u]: int(st["jobs"][abi.STATS_WAITING, u]) for u in w}
    return {"pool->queue-length": {p: sum(m.values()) for p, m in per.items()}, "pool->user->queue-length": per}


# ---- the periodic killers over resident pools --------------------------------------------------------------------
KILL_REASONS = {"linger": "max-runtime-exceeded", "straggler": "straggler", "cancel": "reason-killed-by-user"}


def lingering_timeouts_ms(timeout_hours=48, max_timeout_hours=None, default_timeout_hours=None):
    """kill-lingering-tasks' (scheduler.clj:1912-1918) default and max timeouts in ms: each falls back to
    timeout-hours (48 in lingering-task-killer)."""
    dflt = default_timeout_hours if default_timeout_hours is not None else timeout_hours
    mx = max_timeout_hours if max_timeout_hours is not None else timeout_hours
    return int(dflt * 3_600_000), int(mx * 3_600_000)


def kill_lists(engines, now_ms, default_timeout_ms, max_timeout_ms, groups=None,
               lists=("linger", "cancel", "straggler")):
    """One trigger of the killers over resident pools (engine.state_sweep): [(reason, task id, engine index, group or
    None)] in the sweep's orders, lingering first, then stragglers, then cancelled.  The status updates of the killed
    tasks come back through the tap and go to engine.state_finish."""
    from .engine import state_sweep
    got = state_sweep(engines, now_ms, default_timeout_ms, max_timeout_ms, groups, lists)
    out = []
    for k in ("linger", "straggler", "cancel"):
        for x in got[k] or ():
            g, (t, p) = (x[0], x[1:]) if k == "straggler" else (None, x)
            out.append((KILL_REASONS[k], t, p, g))
    return out


# ---- why a resident pool's job is not scheduled (/unscheduled_jobs, unscheduled.clj:172-200) -----------------------
CONSTRAINT_MESSAGES = {   # constraint-name->message (unscheduled.clj:71-75), key spellings as the reference has them
    "novel_host_constraint": "Job already ran on this host.",
    "gpu_host_constraint": "Host has no GPU support.",
    "non_gpu_host_constraint": "Host is reserved for jobs that need GPU support.",
    "attribute-equals-host-placement-group-constraint": "Host had a different attribute than other jobs in the group."}
USAGE_KEYS = ("count", "cpus", "mem", "gpus")   # cook_state_unscheduled's usage columns


def fenzo_failures_for_user(summary):
    """fenzo-failures-for-user (:77-90): a placement-failure summary -> [{reason, host_count}], resources first; a
    constraint the message table lacks is shown by its name."""
    return ([{"reason": f"Not enough {k} available.", "host_count": v} for k, v in summary.get("resources", {}).items()] +
            [{"reason": CONSTRAINT_MESSAGES.get(k, k), "host_count": v}
             for k, v in summary.get("constraints", {}).items()])


def exceeded(limits, usage):
    """how-job-would-exceed-resource-limits (:37-52) on the device's usage including the job: {key: {limit, usage}}
    for the keys of `limits` (in their order) whose usage is strictly above the limit; a key the usage lacks reads 0."""
    got = dict(zip(USAGE_KEYS, (float(x) for x in usage)))
    return {k: {"limit": v, "usage": got.get(k)} for k, v in limits.items() if got.get(k, 0) > v}


class Investigations:
    """The host half of record-placement-failures! (fenzo_utils.clj:47-89) for a resident pool: the jobs under
    investigation and the last placement-failure summary of each job."""

    def __init__(self):
        self.marked, self.summary = set(), {}

    def investigate(self, job_id):
        """check-fenzo-placement's mark: the next match that leaves the job unplaced records why."""
        self.marked.add(int(job_id))

    def record(self, engine, match):
        """After a resident match (engine.state_match_offers' or state_match's result, on the same handle before its
        next match): the marked considerable jobs left unplaced get cook_match_failures' summary; a non-empty one is
        stored and ends the investigation, an empty one (ports only) leaves the job under investigation."""
        cons, assign = match["considerable"], match["assign"]
        ks = [k for k in range(len(cons)) if assign[k] < 0 and int(cons[k]) in self.marked]
        if not ks:
            return
        for k, f in zip(ks, engine.match_failures(ks)):
            s = summarize_failures(f["counts"])
            if s:
                j = int(cons[k])
                self.summary[j] = s
                self.marked.discard(j)


def unscheduled_reasons(answer, i, *, job_state="completed", quota=None, share=None, attempts_consumed=0,
                        max_retries=None, enforcing_rate_limit=False, num_rate_limited=0, plugin="", plugin_message=None,
                        investigations=None, job_of=None):
    """reasons (:172-200) for query i of engine.state_unscheduled's `answer`: [[message, data]] in the reference's
    order.  The host facts: job_state (a job the handle does not hold: "running" or "completed"), the user's quota and
    share maps in this pool, attempts consumed and max retries, whether the launch rate limit is enforced and the
    user's rate-limited count summed over pools, the launch plugin's name and message, the pool's Investigations (the
    job is marked) and job_of (job id -> what the answer shows, e.g. its uuid; default the id)."""
    status = int(answer["status"][i])
    if status == abi.UNSCHED_RUNNING or (status == abi.UNSCHED_ABSENT and job_state == "running"):
        return [["The job is running now.", {}]]
    if status == abi.UNSCHED_ABSENT:
        return [["The job already completed.", {}]]
    job_of = job_of or (lambda j: j)
    usage = answer["usage"][i]
    out = []
    if max_retries is not None and attempts_consumed >= max_retries:
        out.append(["Job has exhausted its maximum number of retries.",
                    {"max-retries": max_retries, "instance-count": attempts_consumed}])
    for limits, msg in ((quota, "The job would cause you to exceed resource quotas."),
                        (share, "The job would cause you to exceed resource shares.")):
        ways = exceeded(limits or {}, usage)
        if ways:
            out.append([msg, ways])
    if enforcing_rate_limit and num_rate_limited > 0:
        out.append(["You are currently rate limited on how many jobs you launch per minute.",
                    {"num-ratelimited": num_rate_limited}])
    if answer["plugin_deferred"][i]:
        out.append(["The launch filter plugin is blocking the job launch.", {"plugin": plugin, "message": plugin_message}])
    pos, ahead = int(answer["position"][i]), answer["ahead"][i]
    if ahead:
        out.append([f"You have {pos} other jobs ahead in the queue.", {"jobs": [job_of(j) for j in ahead]}])
    inv = investigations if investigations is not None else Investigations()
    j = int(answer["job_id"][i])
    inv.investigate(j)   # check-fenzo-placement (:92-108) marks the job whether or not a summary is stored
    if j in inv.summary:
        out.append(["The job couldn't be placed on any available hosts.",
                    {"reasons": fenzo_failures_for_user(inv.summary[j])}])
    else:
        out.append(["The job is now under investigation. Check back in a minute for more details!", {}])
    return out


# ---- users' running usage (GET /usage, get-user-usage api.clj:2946-2969) -----------------------------------------
def _usage_map(v):
    """{cpus mem gpus jobs} of (jobs, cpus, mem, gpus); None: the reference's zero-usage."""
    return {"cpus": 0.0, "mem": 0.0, "gpus": 0.0, "jobs": 0} if v is None else \
        {"cpus": v[1], "mem": v[2], "gpus": v[3], "jobs": v[0]}


def _add(a, b):
    return b if a is None else tuple(x + y for x, y in zip(a, b))


def usage_response(answers, *, user=None, pool=None, pools=(), group_breakdown=False, job_uuid=None, group_info=None,
                   user_name=None):
    """The body of GET /usage from engine.state_user_usage answers, in the reference's shape (usage, user-usage and
    no-usage-map, api.clj:2894-2944).  answers: [(answer, names)], one per device, each over handles whose pool names
    are `names` in handle order, asked with by_group = group_breakdown and per_pool = (pool is None and pools).  With
    a `pool` (the parameter or header), the answers cover that pool's handle alone and the response has no "pools".
    user: the queried user code, else {"users": {name: usage}} over the users that run a job.  pools: every pool name
    in the database (the zero maps; empty: no pools).  job_uuid(job id), group_info(group code) -> (uuid, name) and
    user_name(code) give what the response shows (default: the codes, a None name).  The device folds are exact; the
    totals of several devices are added here in device order."""
    job_of = job_uuid or (lambda j: j)
    info = group_info or (lambda g: (g, None))
    name_of = user_name or (lambda u: u)
    per_pool = pool is None and len(pools) > 0
    acc = {}   # user -> scope name (None: every pool) -> {"total": usage, "groups": {group: [usage, job ids]}}
    for ans, names in answers:
        for d in range(len(ans["user"])):
            sc, g = int(ans["scope"][d]), int(ans["group"][d])
            slot = acc.setdefault(int(ans["user"][d]), {}).setdefault(None if sc < 0 else names[sc],
                                                                       {"total": None, "groups": {}})
            v = (int(ans["jobs"][d]), float(ans["cpus"][d]), float(ans["mem"][d]), float(ans["gpus"][d]))
            if g == abi.UU_TOTAL:
                slot["total"] = _add(slot["total"], v)
            else:
                cur = slot["groups"].setdefault(g, [None, []])
                cur[0] = _add(cur[0], v)
                cur[1] += ans["lists"][d]

    def user_usage(slot):
        out = {"total_usage": _usage_map(slot and slot["total"])}
        if group_breakdown:
            groups = slot["groups"] if slot else {}
            out["grouped"] = [{"group": {"uuid": info(g)[0], "name": info(g)[1],
                                         "running_jobs": [job_of(j) for j in js]}, "usage": _usage_map(v)}
                              for g, (v, js) in sorted(groups.items()) if g >= 0]
            v, js = groups.get(abi.UU_UNGROUPED, (None, []))
            out["ungrouped"] = {"running_jobs": [job_of(j) for j in js], "usage": _usage_map(v)}
        return out

    def usage(u):
        per = acc.get(u, {})
        out = user_usage(per.get(None))
        if per_pool:
            out["pools"] = {p: user_usage(per.get(p)) for p in list(pools) + [p for p in per if p is not None and p not in pools]}
        return out

    if user is not None:
        return usage(int(user))
    return {"users": {name_of(u): usage(u) for u in sorted(acc)}}


# ---- instance stats (GET /stats/instances, task-stats/get-stats task_stats.clj) ----------------------------------
_IS_METRICS = ("run-time-seconds", "cpu-seconds", "mem-seconds")   # by abi.IS_RUN_TIME, IS_CPU, IS_MEM
_IS_PCTS = (50, 75, 95, 99, 100)


def instance_stats_response(answer, *, user_name=None, reason_string=None):
    """The body of GET /stats/instances from an engine.state_instance_stats answer, in the reference's shape
    (generate-all-stats): "overall" ({} when no instance is selected), "by-reason" {reason: stats},
    "by-user-and-reason" {user: {reason: stats}} and "leaders" {"cpu-seconds" / "mem-seconds": {user: total}}, the
    leaders in descending total.  stats = {"count", and per metric {"percentiles": {50 75 95 99 100}, "total"}}.
    user_name(code) and reason_string(code >= 0) give what the response shows (default: the codes).  The nil reason
    (code -1) is the key "", which is how the reference's JSON encoder writes a nil map key."""
    name_of = user_name or (lambda u: u)
    reason_of = reason_string or (lambda r: r)
    key = lambda r: "" if r == -1 else reason_of(r)

    def stats(d):
        out = {"count": int(answer["count"][d])}
        for m, k in enumerate(_IS_METRICS):
            out[k] = {"percentiles": {p: float(answer["pct"][d][m][j]) for j, p in enumerate(_IS_PCTS)},
                      "total": float(answer["total"][d][m])}
        return out

    out = {"by-reason": {}, "by-user-and-reason": {}, "leaders": {}, "overall": {}}
    for d in range(len(answer["kind"])):
        kind, u, r = int(answer["kind"][d]), int(answer["user"][d]), int(answer["reason"][d])
        if kind == abi.IS_OVERALL:
            out["overall"] = stats(d)
        elif kind == abi.IS_REASON:
            out["by-reason"][key(r)] = stats(d)
        else:
            out["by-user-and-reason"].setdefault(name_of(u), {})[key(r)] = stats(d)
    out["leaders"] = {"cpu-seconds": {name_of(u): t for u, t in answer["leaders_cpu"]},
                      "mem-seconds": {name_of(u): t for u, t in answer["leaders_mem"]}}
    return out


JOB_STATS_ERROR = "Error collecting job stats"   # what jobs->stats returns when it throws (scheduler.clj:594-602)


def _mm_key(kind, code, gpu_model_name, disk_type_name):
    """A keyed total's resource key as jobs->resource-maps (scheduler.clj:511-545) writes it."""
    if kind == abi.MM_GPUS:
        return "gpus/" + (gpu_model_name(code) if code >= 0 else "unspecified-gpu-model")
    t = disk_type_name(code) if code >= 0 else "unspecified-disk-type"
    return f"disk/{t}/" + ("request" if kind == abi.MM_DISK_REQUEST else "limit")


def _mm_resource_map(row, gpu_model_name, disk_type_name, uris):
    """job->resource-map of a cook_state_match_metrics row, formatted for structured logging (numbers stay numbers,
    the uris vector becomes its string)."""
    m = {"cpus": row["cpus"], "mem": row["mem"]}
    f = row["facts"]
    if f & abi.JF_GPUS:
        m[_mm_key(abi.MM_GPUS, row["gpu_model"], gpu_model_name, disk_type_name)] = row["gpus"]
    if f & abi.JF_DISK_REQUEST:
        m[_mm_key(abi.MM_DISK_REQUEST, row["disk_type"], gpu_model_name, disk_type_name)] = row["disk_request"]
    if f & abi.JF_DISK_LIMIT:
        m[_mm_key(abi.MM_DISK_LIMIT, row["disk_type"], gpu_model_name, disk_type_name)] = row["disk_limit"]
    if f & abi.JF_URIS:
        m["uris"] = str(uris(row["job_id"]))
    return m


def _mm_head_resources(row, gpu_model_name, disk_type_name, uris):
    """tools/job-ent->resources of the head (tools.clj:247-273): cpus, mem, ports, gpus when present, the disk map (the
    type only when the job names one) and the uris."""
    f = row["facts"]
    out = {"ports": row["ports"], "cpus": row["cpus"], "mem": row["mem"]}
    if f & abi.JF_GPUS:
        out["gpus"] = row["gpus"]
    if f & abi.JF_DISK:
        d = {"request": row["disk_request"] if f & abi.JF_DISK_REQUEST else None}
        if f & abi.JF_DISK_LIMIT:
            d["limit"] = row["disk_limit"]
        if row["disk_type"] >= 0:
            d["type"] = disk_type_name(row["disk_type"])
        out["disk"] = d
    if f & abi.JF_URIS:
        out["uris"] = uris(row["job_id"])
    return out


def match_cycle_metrics_response(answer, considerable_job_id, *, pool, max_considerable, n_offers, n_offers_scheduled,
                                 offers_stats=None,
                                 user_name=None, job_name=None, gpu_model_name=None, disk_type_name=None, uris=None,
                                 unmatched_cycles_warn_threshold=500, unmatched_fraction_warn_threshold=0.5):
    """What handle-match-cycle-metrics (scheduler.clj:1210-1280) and the unmatched tracking (:1399-1486) log, from an
    engine.state_match_metrics answer, the round's considerable job ids (the match's output) and the host's
    dictionaries (each maps a code to its name; default: the code).
    Returns {"users": ["user match cycle metric" maps, in ascending user code], "total": the "total match cycle metric"
    map, "warn": the "Jobs are unmatched for too long" map or None, "front": (cpus, mem) of the front-of-queue gauges}.
    match-percent is a fractions.Fraction, as Clojure's ratio.  :stats :offers (offers->stats) is the host's
    `offers_stats`; :jobs-considerable is the error string when two or more considerable jobs carry uris.  uris(job id)
    gives a job's uri vector (the one row jobs->resource-maps keeps, and the head's)."""
    from fractions import Fraction
    name_of = user_name or (lambda u: u)
    job_of = job_name or (lambda j: j)
    gname = gpu_model_name or (lambda c: str(c))
    dname = disk_type_name or (lambda c: str(c))
    uris = uris or (lambda j: [])
    n, nm = answer["considerable"], answer["matched"]
    out = {"users": [], "warn": None, "front": (0, 0)}
    if n == 0:   # the slim form of the zero-considerable case
        out["total"] = {"inputs": {"jobs-considerable": 0}, "pool": pool}
        return out
    for u, (c, m) in enumerate(zip(answer["user_considerable"], answer["user_matched"])):
        if c:
            out["users"].append({"user": name_of(u), "pool": pool, "user-considerable": int(c),
                                 "user-matched": int(m), "user-unmatched": int(c - m)})
    head, lc, lm = answer["rows"]
    if answer["uris"] >= 2:
        jobs_stats = JOB_STATS_ERROR
    else:
        totals = {"cpus": answer["total_cpus"], "mem": answer["total_mem"]}
        for kind, code, total in answer["keys"]:
            totals[_mm_key(kind, code, gname, dname)] = total
        if answer["uris"] == 1:
            totals["uris"] = str(uris(int(considerable_job_id[answer["uris_position"]])))
        jobs_stats = {"largest-by": {"cpus": _mm_resource_map(lc, gname, dname, uris),
                                     "mem": _mm_resource_map(lm, gname, dname, uris)},
                      "percentiles": {r: dict(zip((50, 95, 100), answer["pct_" + r])) for r in ("cpus", "mem")},
                      "totals": totals}
    out["total"] = {
        "inputs": {"jobs-considerable": n, "offers": n_offers, "max-considerable": max_considerable,
                   "queue-was-full": max_considerable == n},
        "matched": {"jobs-considerable": nm, "offers": n_offers_scheduled, "match-percent": Fraction(nm, n),
                    "head-was-matched": bool(answer["head_matched"])},
        "pool": pool,
        "unmatched": {"jobs-considerable": n - nm, "offers": n_offers - n_offers_scheduled},
        "stats": {"jobs-considerable": jobs_stats, "offers": offers_stats,
                  "head-resources": _mm_head_resources(head, gname, dname, uris)}}
    out["front"] = (head["cpus"], head["mem"])
    # the warning's fraction test: Clojure's (/ a n) ratio compared as a double with the threshold
    if float(Fraction(answer["too_long"], n)) > unmatched_fraction_warn_threshold:
        out["warn"] = {"pool": pool, "first-ten-unmatched-too-long": [(job_of(j), c) for j, c in answer["first"]],
                       "number-considerable": n, "number-unmatched-too-long": answer["too_long"],
                       "unmatched-cycles-warn-threshold": unmatched_cycles_warn_threshold,
                       "unmatched-fraction-warn-threshold": unmatched_fraction_warn_threshold}
    return out


def retry_facts(instances, reason_table):
    """A job's done-instance reasons for cook_state_retry_facts, from its instances as (status, reason name or None):
    the reason codes of the success and failed ones in order (-1: no reason; :job/attempts-consumed reads both), and
    whether one succeeded (then the job is completed: pass abi.RF_COMPLETED).  reason_table: name -> :reason/code."""
    done = [reason_table[r] if r is not None else -1 for st, r in instances if st in ("success", "failed")]
    return done, any(st == "success" for st, _ in instances)


LIST_STATE_NAMES = {abi.LJ_WAITING: "waiting", abi.LJ_RUNNING: "running"}


def list_jobs_response(answer, *, states, limit, completed=(), uncommitted=()):
    """The job ids GET /list or GET /jobs lists, newest first, from engine.state_list_jobs' answer (made with this
    limit) and the host's part:
      uncommitted  [(job id, submit ms)]: the uncommitted waiting jobs that pass the request's filters.  Only /list
                   (include-custom-executor false) keeps them (get-active-jobs-by-user-and-state removes them only
                   with include-custom-executor); they merge into the waiting list by job id, cut to limit again.
      completed    {state: [(job id, submit ms)]} for "completed", "success" and "failed", each the Datomic path's
                   answer, in entity-id order and cut to limit.
    The per-state lists are concatenated in the order of `states` (mapcat), stably sorted by submit time and cut to
    limit (get-jobs-by-user-and-states), then reversed (list-job-ents): entries of equal submit time come out in the
    reverse of their concatenation order."""
    per = {"waiting": [], "running": []}
    for s, j, t in zip(answer["state"], answer["job_id"], answer["submit_ms"]):
        per[LIST_STATE_NAMES[int(s)]].append((int(j), int(t)))
    if uncommitted:
        merged = per["waiting"] + [(int(j), int(t)) for j, t in uncommitted]
        per["waiting"] = sorted(merged, key=lambda e: e[0])[:limit]
    done = dict(completed)
    cat = [e for s in states for e in (per[s] if s in per else done.get(s, []))]
    oldest = sorted(cat, key=lambda e: e[1])[:limit]
    return [j for j, _ in reversed(oldest)][:limit]
