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
                        + num-considerable scale-back / reset (handle-fenzo-pool :1613-1651)
  summarize_failures    fenzo_utils.clj:45-89 shape from cook_match_failures' counters (8f-3)
"""
import numpy as np

from . import abi, traces

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
