;; cook.scheduler.gpu — the JVM side of the H100 hot path (include/cook_gpu.h through jni/cook_gpu_jni.c).
;;
;; Drop-in seams (SURVEY §8b; all line numbers in scheduler/src/cook/scheduler/scheduler.clj):
;;   :2073-2091 sort-jobs-by-dru-helper      -> (rank-pool! ...)                    [cook_rank]
;;   :1339-1535 handle-resource-offers!      -> (handle-resource-offers! ...)       [cook_match]
;;   rebalancer.clj:434-467 rebalance        -> (rebalance! ...)                    [cook_rebalance]
;;   :2125-2157 quota-group usage            -> (exchange-usage! ...)               [cook_exchange_usage]
;;   :2262-2284 rank-jobs, resident pool     -> (rank-resident! ...)                [cook_state_rank_offensive]
;;   :1749-1800 Kubernetes-scheduler pool    -> (kubernetes-considerable! ...)      [cook_state_considerable]
;;   :1283-1335 autoscaling helper           -> (autoscalable-jobs! ...)            [cook_state_considerable]
;;   monitor.clj:177-207 set-stats-counters! -> (monitor-resident! ...)             [cook_state_user_stats]
;;   :1888-2016 the three killers            -> (sweep! ...), fed by task-facts! / finish! / group-runtimes!
;;                                              [cook_state_sweep, cook_state_task_facts, cook_state_finish,
;;                                               cook_state_group_runtimes]
;;   unscheduled.clj:172-200 reasons      -> (unscheduled! ...) + cycle.py's unscheduled_reasons  [cook_state_unscheduled]
;;   api.clj:2946-2969 get-user-usage       -> (user-usage! ...) + cycle.py's usage_response  [cook_state_user_usage]
;;   api.clj:3150-3232 task-stats-handler   -> (instance-stats! ...) + cycle.py's instance_stats_response, fed by
;;                                              task-reason! [cook_state_instance_stats, cook_state_task_reason], and
;;                                              for success / failed by history-seed!, finish-history! and
;;                                              history-advance! [cook_state_history_*]
;;   api.clj:3038-3085 list-resource, :1684-1776 list-job-ents (waiting, running)
;;                                           -> (list-jobs ...) + cycle.py's list_jobs_response, fed by list-facts!
;;                                              [cook_state_list_jobs, cook_state_list_facts]
;;   tools.clj:393-434 get-completed-jobs-by-user (completed, success, failed)
;;                                           -> (list-completed ...), fed by completed-seed!, completed-record! and
;;                                              completed-advance! [cook_state_list_completed, cook_state_completed_*]
;;   :217-313 write-status-to-datomic       -> (status! ...), fed by retry-config! and retry-facts!
;;                                             [cook_state_status, cook_state_retry_config, cook_state_retry_facts]
;;   :1210-1280 handle-match-cycle-metrics and the unmatched tracking :1399-1486
;;                                           -> (match-metrics! ...) + cycle.py's match_cycle_metrics_response, fed by
;;                                              job-facts! [cook_state_match_metrics, cook_state_job_facts]
;; selected per pool with {:scheduler-config {:scheduler "gpu"}} next to "fenzo" / "kubernetes"
;; (config.clj:110-122, make-pool-handler :2425-2466).  Everything numeric happens in libcookgpu;
;; this namespace marshals columns and keeps the state Fenzo kept (cook_b200/cycle.py is the same
;; state machine in Python, with the K15 known answers running through it).
;;
;; NOT COMPILED in this repository's image (no JVM): reviewed against scheduler.clj and abi.py.
(ns cook.scheduler.gpu
  (:require [clojure.core.async :as async]
            [clojure.tools.logging :as log]
            [cook.config :as config]
            [cook.scheduler.constraints :as constraints]
            [cook.tools :as tools])
  (:import (cook.gpu Native)
           (java.nio ByteBuffer ByteOrder)))

;; ---------------------------------------------------------------------------------------------
;; marshalling: one direct ByteBuffer per column, native byte order (the JNI shim takes addresses)
(defn- direct ^ByteBuffer [n-bytes]
  (doto (ByteBuffer/allocateDirect (max 8 (long n-bytes))) (.order (ByteOrder/nativeOrder))))
(defn i32-col ^ByteBuffer [xs] (let [b (direct (* 4 (count xs)))] (doseq [x xs] (.putInt b (int x))) (.rewind b) b))
(defn i64-col ^ByteBuffer [xs] (let [b (direct (* 8 (count xs)))] (doseq [x xs] (.putLong b (long x))) (.rewind b) b))
(defn f64-col ^ByteBuffer [xs] (let [b (direct (* 8 (count xs)))] (doseq [x xs] (.putDouble b (double x))) (.rewind b) b))
(defn u8-col ^ByteBuffer [xs] (let [b (direct (count xs))] (doseq [x xs] (.put b (byte (if x 1 0)))) (.rewind b) b))
(defn csr "CSR of a seq of seqs: [offsets values]" [lists]
  [(i32-col (reductions + 0 (map count lists))) (i32-col (apply concat lists))])

(defn- check! [pool rc what]
  (when-not (zero? rc)
    (throw (ex-info (str what " failed: " (Native/lastError pool)) {:code rc :what what}))))

;; dictionary encoding (the host shim's job, cook_gpu.h "id / idx columns"): dense int32 codes
(defn dictionary [] (atom {}))
(defn code! [dict x] (if (nil? x) -1 (or (@dict x) (get (swap! dict #(if (% x) % (assoc % x (count %)))) x))))

;; ---------------------------------------------------------------------------------------------
;; constraint plugin API: every JobConstraint record gains `encode` -> columns of cook_jobs_soa.
;; A record without `encode` makes config validation fail for a "gpu" pool
;; (COOK_E_UNSUPPORTED_CONSTRAINT): there is no CPU fallback.
(defprotocol EncodableConstraint
  (encode [this ctx] "Returns a map of cook_jobs_soa column contributions for this job, e.g.
                     {:novel-hosts [host-id ...]} | {:attr [[col val] ...]} | {:est-end-ms t} | ..."))

(extend-protocol EncodableConstraint
  cook.scheduler.constraints.novel_host_constraint
  (encode [c {:keys [host-dict]}] {:novel-hosts (mapv #(code! host-dict %) (:previous-hosts c))})
  cook.scheduler.constraints.gpu_host_constraint
  (encode [c {:keys [gpu-model-dict]}] {:gpu-model (code! gpu-model-dict (:job-gpu-model-requested c))})
  cook.scheduler.constraints.disk_host_constraint
  (encode [c {:keys [disk-type-dict]}] {:disk-request (:job-disk-request c) :disk-type (code! disk-type-dict (:job-disk-type c))})
  cook.scheduler.constraints.user_defined_constraint
  (encode [c {:keys [attr-col attr-val-dict]}]
    ;; EQUALS only (constraints.clj:355-383); value ids are per attribute column, 0 = absent on the host,
    ;; -1 = pattern not in the host dictionary (never matches)
    {:attr (mapv (fn [{:keys [attribute pattern]}] [(attr-col attribute) (or (get-in @attr-val-dict [attribute pattern]) -1)])
                 (:constraints c))})
  cook.scheduler.constraints.estimated_completion_constraint
  (encode [c _] {:est-end-ms (:estimated-end-time c)})
  cook.scheduler.constraints.checkpoint_locality_constraint
  (encode [c {:keys [location-dict]}] {:ckpt-location (code! location-dict (:job-last-checkpoint-location c))})
  cook.scheduler.constraints.rebalancer_reservation_constraint
  (encode [_ _] {}))   ; expressed through offers.reserved + jobs.reserved_host

;; ---------------------------------------------------------------------------------------------
;; M5: what Fenzo kept between cycles (:617-687, :2301-2324).  Unused Mesos leases stay live, summed
;; per hostname with later offers, until offer-incubate-time-ms; :reject-after-match-attempt offers
;; (Kubernetes) never survive a match attempt.
(defn add-offers [cache offers now-ms] (into cache (map #(assoc % ::received now-ms) offers)))
(defn expire-offers [cache now-ms incubate-ms]
  [(filterv #(< (- now-ms (::received %)) incubate-ms) cache)
   (filterv #(>= (- now-ms (::received %)) incubate-ms) cache)])   ; [live declined]
(defn merged-offers "hostname -> [leases], first-seen order (one assignable VM per hostname, FENZO rule 1)" [cache]
  (reduce (fn [m o] (update m (:hostname o) (fnil conj []) o)) (array-map) cache))
(defn after-match [cache used-hostnames]
  (filterv #(and (not (used-hostnames (:hostname %))) (not (:reject-after-match-attempt %))) cache))

;; M6: handle-fenzo-pool's feedback loop (:1613-1651)
(defn next-considerable
  [{:keys [num-considerable iterations-at-floor]} matched-head-or-no-matches?
   {:keys [max-considerable scaleback floor-iterations-before-reset]}]
  (let [nxt (if matched-head-or-no-matches? max-considerable (max 1 (long (* scaleback num-considerable))))
        at-floor (if (= nxt 1) (inc iterations-at-floor) 0)]
    (if (>= at-floor floor-iterations-before-reset)
      {:num-considerable max-considerable :iterations-at-floor at-floor}
      {:num-considerable nxt :iterations-at-floor at-floor})))

(defn filter-matches-for-ratelimit
  "scheduler.clj:887-924: a compute cluster whose launch-rate limiter is enforcing and in debt loses
   all its matches of the cycle."
  [matches cluster->tokens cluster->enforce?]
  (remove (fn [{:keys [compute-cluster]}] (and (cluster->enforce? compute-cluster) (neg? (cluster->tokens compute-cluster)))) matches))

(defn handle-resource-offers!
  "One match cycle of a pool.  `marshal` turns (pending queue, offers, usage, quota, reservations) into
   the column arrays Native/match takes (see cook_b200/abi.py for the field order); the result is
   reshaped to the {:matches [{:leases :tasks :hostname}] :failures} map match-offer-to-schedule
   returned, so launch-matched-tasks! (:926-1048) is unchanged.  Returns matched-head-or-no-matches?."
  [{:keys [pool handle state-atom reservation-atom pending-jobs-atom marshal launch! limiter-state]} offers now-ms]
  (locking handle                                    ; exactly where (locking fenzo ...) is today (:665)
    (let [{:keys [cache num-considerable]} @state-atom
          cache (add-offers cache offers now-ms)
          queue (get @pending-jobs-atom pool)
          {:keys [args out unpack]} (marshal queue (merged-offers cache) @reservation-atom num-considerable)]
      (if (or (empty? queue) (empty? cache))
        (do (swap! state-atom merge (next-considerable @state-atom true config/fenzo-params)) true)
        (do
          (check! handle (apply #(Native/match handle %&) args) "cook_match")
          (let [{:keys [matches failures considerable]} (unpack out)
                matches (filter-matches-for-ratelimit matches (:tokens limiter-state) (:enforce? limiter-state))
                matched (set (mapcat :tasks matches))
                head? (contains? matched (first considerable))
                ok? (or (empty? matches) head?)]
            (when (seq matches)
              (swap! pending-jobs-atom update pool (fn [q] (remove matched q)))             ; :790-795
              (launch! matches)
              (swap! reservation-atom (fn [{:keys [job-uuid->reserved-host launched-job-uuids]}]  ; :1050-1057
                                        {:job-uuid->reserved-host (apply dissoc job-uuid->reserved-host matched)
                                         :launched-job-uuids (into launched-job-uuids matched)})))
            (swap! state-atom (fn [s] (-> s
                                         (assoc :cache (after-match cache (set (map :hostname matches))))
                                         (merge (next-considerable s ok? config/fenzo-params)))))
            (when (seq failures) (log/debug "placement failures" (count failures)))
            ok?))))))

;; ---------------------------------------------------------------------------------------------
(defn rank-pool!
  "Replaces sort-jobs-by-dru-helper + filter-based-on-quota + filter-offensive-jobs for one pool.
   NB (ADVICE): cook_rank returns the survivors only; the shim recomputes `is-offensive?` (:2198-2210)
   on the JVM for the jobs that were dropped so that they are still pushed to offensive-jobs-ch."
  [handle {:keys [running pending users pool-quota group-quota group-usage params out]}]
  (check! handle (Native/rank handle (:n running) (:cols running) (:n pending) (:cols pending) (:n users) (:cols users)
                              pool-quota group-quota group-usage (:max-over-quota-jobs params) (if (:filter-offensive params) 1 0)
                              (:offensive-max-mem-mb params) (:offensive-max-cpus params)
                              (:ranked out) (:n out) (:dru out) (:order out) (:order-n out))
          "cook_rank"))

(defn rebalance!
  "Replaces init-state + rebalance (rebalancer.clj:222-266, :434-467).  Decisions with more than one
   victim reserve their host for the job (reserve-hosts! :419-432)."
  [handle args reservation-atom decode]
  (check! handle (apply #(Native/rebalance handle %&) args) "cook_rebalance")
  (let [decisions (decode)]
    (swap! reservation-atom
           (fn [{:keys [job-uuid->reserved-host launched-job-uuids] :as m}]
             (assoc m :job-uuid->reserved-host
                      (into job-uuid->reserved-host
                            (for [{:keys [to-make-room-for hostname task]} decisions
                                  :when (and (> (count task) 1) (not (contains? launched-job-uuids (:job/uuid to-make-room-for))))]
                              [(:job/uuid to-make-room-for) hostname]))
                      :launched-job-uuids #{})))
    decisions))

(defn cotasks!
  "Each group's running cotasks from the resident running rows (cook_state_cotasks), for the groups columns of
   the next state match or rebalance: `args` are Native/stateCotasks' arguments after the handle, with
   out-cot-hostname-id nil to ask for the size first.  Replaces the host index running task -> job -> groups
   -> host that get-cotasks-from-tracker-state (constraints.clj:539-552) would otherwise need."
  [handle args]
  (check! handle (apply #(Native/stateCotasks handle %&) args) "cook_state_cotasks"))

(defn match-derived!
  "The resident match cycle in one call (cook_state_match_derived): the users' usage, the offers' run columns and
   the groups' cotask lists are read from the resident running rows on the device, so `args` (Native/stateMatch's
   arguments after the handle) may leave those columns nil.  Replaces cotasks! and the usage fold before a state
   match."
  [handle args]
  (check! handle (apply #(Native/stateMatchDerived handle %&) args) "cook_state_match_derived"))

(defn rank-resident!
  "Ranks the resident pool (cook_state_rank_offensive) and pushes the jobs the rank dropped as offensive to
   offensive-jobs-ch, as filter-offensive-jobs (scheduler.clj:2198-2229) does: the stifler marks them completed.
   `args` are Native/stateRankOffensive's arguments after the handle; `job-id->job` resolves a job id, `out-off` /
   `out-n-off` are its offensive-job-id buffer and count array.  Returns the queue's length."
  [handle args ^ByteBuffer out-off ^ints out-n-off job-id->job offensive-jobs-ch]
  (check! handle (apply #(Native/stateRankOffensive handle %&) args) "cook_state_rank_offensive")
  (let [n (aget out-n-off 0)
        lb (.asLongBuffer out-off)
        jobs (mapv #(job-id->job (.get lb (int %))) (range n))]
    (when (seq jobs) (async/>!! offensive-jobs-ch jobs))
    n))

(defn kubernetes-considerable!
  "handle-kubernetes-scheduler-pool (scheduler.clj:1749-1800) on a resident pool: pending-jobs->considerable-jobs in
   one call (cook_state_considerable with the allowed / plugin masks read, the usage derived from the resident running
   rows, consume on: the jobs leave the queue until the next rank, as remove-matched-jobs-from-pending-jobs does).
   `args` are Native/stateConsiderable's arguments after the handle and before iparams.  Returns the job ids; the
   caller launches them."
  [handle num-considerable enforce-rate-limit? args ^ByteBuffer out ^ints out-n]
  (check! handle (apply #(Native/stateConsiderable handle %&)
                        (concat args [(int-array [num-considerable (if enforce-rate-limit? 1 0) 0 1 1]) out out-n]))
          "cook_state_considerable")
  (let [lb (.asLongBuffer out)] (mapv #(.get lb (int %)) (range (aget out-n 0)))))

(defn autoscalable-jobs!
  "handle-resource-offers-autoscaling-helper (scheduler.clj:1283-1335) after a resident match and its launches:
   filter-pending-jobs-for-quota over what is left of the queue (quota_only), with the usage the match read
   (COOK_USAGE_LAST_MATCH).  `n` is the scaled maximum; the recent-synthetic-pod skip stays with the caller."
  [handle n enforce-rate-limit? args ^ByteBuffer out ^ints out-n]
  (check! handle (apply #(Native/stateConsiderable handle %&)
                        (concat args [(int-array [n (if enforce-rate-limit? 1 0) 1 2 0]) out out-n]))
          "cook_state_considerable")
  (let [lb (.asLongBuffer out)] (mapv #(.get lb (int %)) (range (aget out-n 0)))))

;; cook_state_user_stats' states (COOK_STATS_*) and user counts (COOK_USERS_*), by index
(def ^:private stat-states ["running" "waiting" "starved" "waiting-under-quota"])
(def ^:private user-counts ["total" "starved" "waiting-under-quota" "hungry" "satisfied"])

(defn monitor-resident!
  "set-stats-counters! (monitor.clj:177-207) for one pool or quota-group name from its resident handles (the pool's
   own, or every pool the quota grouping maps to the name, on one device or several): cook_state_user_stats, then the
   per-user and \"all\" counters through `set-user-counter!` (fn [state user type amount]) and the user counts through
   `set-total-counter!` (fn [state n]), the monitor's own setters, which clear stale users and feed Prometheus.
   `args` are Native/stateUserStats' n_users, users and quota_rest_ok; `names` maps user codes to names; `quota-extra`
   (fn [code]) gives a waiting-under-quota user's other quota keys ({\"gpus\" x \"launch-rate-saved\" y ...}), which
   the reference's merges pass through.  Out buffers are direct, n_users = (count names)."
  [handles args names quota-extra set-user-counter! set-total-counter!]
  (let [u (count names)
        jobs (direct (* 32 u)) cpus (direct (* 32 u)) mem (direct (* 32 u)) member (direct u)
        all-jobs (direct 32) all-cpus (direct 32) all-mem (direct 32) counts (direct 40)]
    (check! (first handles)
            (apply #(Native/stateUserStats (long-array handles) %&)
                   (concat args [jobs cpus mem member all-jobs all-cpus all-mem counts nil]))
            "cook_state_user_stats")
    (doseq [[s state] (map-indexed vector stat-states)]
      (let [in (filter #(bit-test (.get ^ByteBuffer member (int %)) s) (range u))
            at (fn [^ByteBuffer b i] (.getDouble b (* 8 (+ (* s u) i))))
            stats (into {} (for [i in]
                             [(names i) (merge (when (= s 3) (quota-extra i))
                                               {"jobs" (.getLong ^ByteBuffer jobs (* 8 (+ (* s u) i)))
                                                "cpus" (at cpus i) "mem" (at mem i)})]))
            all (if (seq in)
                  (merge (apply merge-with + (map #(dissoc (stats (names %)) "jobs" "cpus" "mem") in))
                         {"jobs" (.getLong ^ByteBuffer all-jobs (* 8 s)) "cpus" (.getDouble ^ByteBuffer all-cpus (* 8 s))
                          "mem" (.getDouble ^ByteBuffer all-mem (* 8 s))})
                  {"cpus" 0 "mem" 0 "jobs" 0})]
        (doseq [[user m] (assoc stats "all" all) [type amount] m]
          (set-user-counter! state user type amount))))
    (doseq [[i c] (map-indexed vector user-counts)]
      (set-total-counter! c (.getLong ^ByteBuffer counts (* 8 i))))))

;; cook_fp as 24 bytes of a little-endian direct buffer
(defn- fp-at [^ByteBuffer b i] [(.getLong b (* 24 i)) (.getLong b (+ 8 (* 24 i))) (.getLong b (+ 16 (* 24 i)))])

(defn audit-resident!
  "Proves a resident pool equal to the database, or says where it is not (cook_state_digest, then cook_state_export
   of the differing buckets).  `host-buckets` is {:pending [[sum xor n] ...] :running [...]}, the host's own bucket
   fingerprints of its rows (the hash is stated in cook_gpu.h); `out`, `out-p`, `out-r` are the direct buffers of
   Native/stateDigest.  Returns nil when every bucket agrees, else {:buckets [...] :consistent? bool}: the caller
   exports those buckets (Native/stateExport with a mask of them), removes the exported ids it does not have and
   upserts its own rows of those buckets in one apply!."
  [handle n-buckets host-buckets ^ByteBuffer out ^ByteBuffer out-p ^ByteBuffer out-r]
  (check! handle (Native/stateDigest handle n-buckets out out-p out-r) "cook_state_digest")
  (let [differs? (fn [^ByteBuffer b want] (fn [i] (not= (fp-at b i) (nth want i))))
        bad (into (sorted-set)
                  (concat (filter (differs? out-p (:pending host-buckets)) (range n-buckets))
                          (filter (differs? out-r (:running host-buckets)) (range n-buckets))))]
    (when (seq bad)
      {:buckets (vec bad) :consistent? (= 1 (.getInt out 104))})))

(defn queue-resident
  "The live queue of a resident pool as job ids (cook_state_queue): what the /queue endpoint reads between two ranks,
   after the launches, removals, replacements and consumed jobs since the rank.  `out` holds `cap` longs."
  [handle cap ^ByteBuffer out ^ints out-n]
  (check! handle (Native/stateQueue handle cap out out-n) "cook_state_queue")
  (let [lb (.asLongBuffer out)] (mapv #(.get lb (int %)) (range (aget out-n 0)))))

(defn rebalance-derived!
  "cook_state_rebalance_derived: the rebalancer over the resident rows with the groups' cotask lists derived on the
   device over the host table in `args` (Native/stateRebalance's arguments after the handle)."
  [handle args]
  (check! handle (apply #(Native/stateRebalanceDerived handle %&) args) "cook_state_rebalance_derived"))

(defn offers-add!
  "cook_state_offers_add: the offers that arrived since the last cycle (cc/pending-offers), each once, stamped with
   the cycle's time.  `args` are Native/stateOffersAdd's arguments after the handle."
  [handle args]
  (check! handle (apply #(Native/stateOffersAdd handle %&) args) "cook_state_offers_add"))

(defn match-offers!
  "handle-fenzo-pool's match for a \"gpu\" pool whose offers are resident (cook_state_match_offers): expiry after
   offer-incubate-time-ms, the merge per hostname, the derived match and the consumption, in one call.  `args` are
   Native/stateMatchOffers' arguments after the handle; `offer-id->offer` resolves an offer id, `out-gone-id`,
   `out-gone-fate` and `out-n-gone` are its gone buffers.  Returns {:used {hostname-code [offers]} :expired [offers]
   :single-shot [offers]}: the caller launches each placement on the :used offers of its host (the match's
   :leases), declines :expired (the lease reject action, scheduler.clj:2315-2323) and forgets :single-shot."
  [handle args offer-id->offer ^ByteBuffer out-gone-id ^ByteBuffer out-gone-fate ^ints out-n-gone]
  (check! handle (apply #(Native/stateMatchOffers handle %&) args) "cook_state_match_offers")
  (let [ids (.asLongBuffer out-gone-id)
        gone (for [i (range (aget out-n-gone 0))]
               [(offer-id->offer (.get ids (int i))) (.get out-gone-fate (int i))])]
    {:used (->> gone (filter #(= 1 (second %))) (map first) (group-by :hostname-code))
     :expired (->> gone (filter #(= 2 (second %))) (mapv first))
     :single-shot (->> gone (filter #(= 3 (second %))) (mapv first))}))

(defn rebalance-offers!
  "cook_state_rebalance_offers: rebalance-derived! with each host's spare resources (view-incubating-offers) folded
   from the live offers on the device; the host table's spare columns may be nil."
  [handle args]
  (check! handle (apply #(Native/stateRebalanceOffers handle %&) args) "cook_state_rebalance_offers"))

(defn exchange-usage!
  "§8e: after a pool's match round; `comm` from Native/commInit (rank 0's Native/commUniqueId bytes travel
   over Cook's own control plane).  Returns the [world n-pad] table as a DoubleBuffer."
  [handle comm world n-pad out]
  (check! handle (Native/exchangeUsage handle comm world n-pad out) "cook_exchange_usage")
  (.asDoubleBuffer ^ByteBuffer out))

(defn exchange-usage-batch!
  "§8e, once per cycle: the usage deltas of ALL pools this scheduler instance matched (handles in pool
   order, `n-slots` = most pools any instance owns) in one all-gather.  Returns [world n-slots n-pad]."
  [handles comm world n-pad n-slots out]
  (check! (first handles) (Native/exchangeUsageBatch (long-array handles) comm world n-pad n-slots out)
          "cook_exchange_usage_batch")
  (.asDoubleBuffer ^ByteBuffer out))

;; ---------------------------------------------------------------------------------------------
;; the periodic killers over resident pools (cancelled-task-killer, lingering-task-killer, straggler-handler)
(defn- longs-buf ^ByteBuffer [xs]
  (let [b (direct (* 8 (count xs)))] (doseq [[i x] (map-indexed vector xs)] (.putLong b (int (* 8 i)) (long x))) b))
(defn- ints-buf ^ByteBuffer [xs]
  (let [b (direct (* 4 (count xs)))] (doseq [[i x] (map-indexed vector xs)] (.putInt b (int (* 4 i)) (int x))) b))
(defn- bytes-buf ^ByteBuffer [xs]
  (let [b (direct (count xs))] (doseq [[i x] (map-indexed vector xs)] (.put b (int i) (byte (if x 1 0)))) b))
(defn- doubles-buf ^ByteBuffer [xs]
  (let [b (direct (* 8 (count xs)))] (doseq [[i x] (map-indexed vector xs)] (.putDouble b (int (* 8 i)) (double x))) b))

(defn task-facts!
  "The killers' facts of live running instances, from the tx-report tap: `facts` is [{:task-id :max-runtime-ms
   (-1: the job has none) :cancelled? :unknown?}]; every row must carry all three."
  [handle facts]
  (check! handle (Native/stateTaskFacts handle (count facts) (longs-buf (map :task-id facts))
                                        (longs-buf (map :max-runtime-ms facts)) (bytes-buf (map :cancelled? facts))
                                        (bytes-buf (map :unknown? facts)))
          "cook_state_task_facts"))

(defn task-reason!
  "The reason fact of live running instances, from the tx-report tap: `reasons` is [{:task-id :reason-code}], the
   code the :reason/code of the instance's :instance/reason (-1: none).  The tap forwards every :instance/reason datom
   whose instance is running or unknown (a killer's reason written before the backend confirms the kill); an upsert or
   a launch of the row writes -1."
  [handle reasons]
  (check! handle (Native/stateTaskReason handle (count reasons) (longs-buf (map :task-id reasons))
                                         (ints-buf (map :reason-code reasons)))
          "cook_state_task_reason"))

(defn reason-datoms
  "The tap's half of task-reason!: from a tx-report's datoms, the [{:task-id :reason-code}] of the asserted
   :instance/reason values whose instance `running?` holds (running or unknown in the resident state).  `reason-attr`
   is the attribute's entity id in the tx's db; `reason-code` maps a :reason entity id to its :reason/code."
  [datoms reason-attr running? reason-code]
  (vec (for [d datoms
             :when (and (= reason-attr (.a d)) (.added d) (running? (.e d)))]
         {:task-id (.e d) :reason-code (reason-code (.v d))})))

(defn finish!
  "Status updates of instances that left running or unknown: [{:task-id :end-ms :success?}].  The rows leave as a
   removal delta takes them; a success leaves its runtime per group for the straggler handler."
  [handle done]
  (check! handle (Native/stateFinish handle (count done) (longs-buf (map :task-id done)) (longs-buf (map :end-ms done))
                                     (bytes-buf (map :success? done)))
          "cook_state_finish"))

(defn finish-history!
  "finish!, and while the handle's history is on, the rows that started at or after its horizon are kept as finished
   instances for instance-stats!: [{:task-id :end-ms :success? :reason-code}], fed by the tap's terminal status datoms
   (the status, the reason and the end time arrive in one transaction, scheduler.clj:274-292).  A :reason-code of nil
   on every row keeps each row's reason fact (task-reason!, the previous-reason of scheduler.clj:281)."
  [handle done]
  (check! handle (Native/stateFinishHistory handle (count done) (longs-buf (map :task-id done))
                                            (longs-buf (map :end-ms done)) (bytes-buf (map :success? done))
                                            (when (some :reason-code done) (ints-buf (map #(or (:reason-code %) -1) done))))
          "cook_state_finish_history"))

;; cook_state_status' outcomes, by COOK_JOB_* code
(def ^:private job-outcomes [:completed :running :waiting :waiting-unretained :no-facts])

(defn retry-config!
  "At start-up: the :reason entities [{:code :mea-culpa? :failure-limit}] (:failure-limit nil: the global one) and
   :scheduler.config/mea-culpa-failure-limit (5 when unset; -1 unlimited), as :job/reasons->attempts-consumed reads
   them (schema.clj:1154-1172)."
  [handle mea-culpa-limit reasons]
  (check! handle (Native/stateRetryConfig handle (int mea-culpa-limit) (count reasons) (ints-buf (map :code reasons))
                                          (bytes-buf (map :mea-culpa? reasons))
                                          (ints-buf (map #(or (:failure-limit %) -2) reasons)))
          "cook_state_retry_config"))

(defn retry-facts!
  "At start-up and on a leadership change after the load, and for each submitted job: [{:job-id :max-retries
   :disable-mea-culpa? :completed? :done-reasons}], :done-reasons the :reason/code of each done (success or failed)
   instance, nil for none (cycle.py's retry_facts).  A launch of such a job parks its pending row for status!."
  [handle facts]
  (let [lens (map (comp count :done-reasons) facts)]
    (check! handle (Native/stateRetryFacts handle (count facts) (longs-buf (map :job-id facts))
                                           (ints-buf (map :max-retries facts))
                                           (bytes-buf (map #(bit-or (if (:disable-mea-culpa? %) 1 0)
                                                                    (if (:completed? %) 2 0)) facts))
                                           (ints-buf (reductions + 0 lens))
                                           (ints-buf (map #(or % -1) (mapcat :done-reasons facts))))
            "cook_state_retry_facts")))

(defn status!
  "finish-history!, and each row's job decided as :instance/update-state decides it (schema.clj:1242-1300), one
   status at a time in order: [{:task-id :end-ms :success? :reason-code :preempted?}] from the tap's terminal status
   datoms.  A waiting job whose row is parked is requeued on the device; returns one {:outcome :attempts} per row,
   :outcome one of :completed :running :waiting :waiting-unretained (upsert the row, as before) :no-facts."
  [handle done]
  (let [n (count done)
        out (direct (* 4 (max n 1)))
        att (direct (* 4 (max n 1)))]
    (check! handle (Native/stateStatus handle n (longs-buf (map :task-id done)) (bytes-buf (map :success? done))
                                       (longs-buf (map :end-ms done))
                                       (when (some :reason-code done) (ints-buf (map #(or (:reason-code %) -1) done)))
                                       (bytes-buf (map :preempted? done)) out att)
            "cook_state_status")
    (let [ob (.asIntBuffer out) ab (.asIntBuffer att)]
      (mapv (fn [i] {:outcome (job-outcomes (.get ob (int i))) :attempts (.get ab (int i))}) (range n)))))

(defn history-seed!
  "At start-up and on a leadership change, after the reset and the load and before the tap resumes: the finished
   instances of the pool with start >= since-ms, read once from Datomic, [{:task-id :user :start-ms :end-ms :cpus :mem
   :success? :reason-code}].  Turns the history on at horizon since-ms."
  [handle since-ms rows]
  (check! handle (Native/stateHistorySeed handle (long since-ms) (count rows)
                                          (object-array [(i64-col (map :task-id rows)) (i32-col (map :user rows))
                                                         (i64-col (map :start-ms rows)) (i64-col (map :end-ms rows))
                                                         (f64-col (map :cpus rows)) (f64-col (map :mem rows))
                                                         (u8-col (map :success? rows))
                                                         (i32-col (map #(or (:reason-code %) -1) rows))]))
          "cook_state_history_seed"))

(defn history-advance!
  "Periodically, with now - retention (the shim's setting, default 32 days: every window task-stats-handler accepts
   that ends by now): the horizon rises and the rows that started before it leave."
  [handle since-ms]
  (check! handle (Native/stateHistoryAdvance handle (long since-ms)) "cook_state_history_advance"))

(defn group-runtimes!
  "After a reset or a leadership change: the successes of the tracked groups' jobs that finished before their rows
   were resident, [[group-code runtime-seconds]], and the group codes no longer tracked."
  [handle seeds forget]
  (check! handle (Native/stateGroupRuntimes handle (count seeds) (ints-buf (map first seeds)) (ints-buf (map second seeds))
                                            (count forget) (ints-buf forget))
          "cook_state_group_runtimes"))

(defn sweep!
  "One trigger of a killer over `handles` (one device): `kinds` a subset of #{:linger :cancel :straggler}; `groups`
   [{:kind :none|:quantile-deviation :quantile :multiplier :n-jobs}] by group code; `n-rows` / `n-entries` the live
   running rows and their group entries (the shim's counts).  Returns {:linger [[task-id handle-index]] :cancel [...]
   :straggler [[group task-id handle-index]]}, each to be killed with :max-runtime-exceeded, :reason-killed-by-user and
   :straggler by the shim as the reference does.  The timeouts are derived from the hours as kill-lingering-tasks does."
  [handles kinds now-ms default-timeout-ms max-timeout-ms groups n-rows n-entries]
  (let [want (fn [k n bytes] (when (kinds k) (direct (* bytes (max 1 n)))))
        lists [(want :linger n-rows 8) (want :linger n-rows 4) (want :cancel n-rows 8) (want :cancel n-rows 4)
               (want :straggler n-entries 4) (want :straggler n-entries 8) (want :straggler n-entries 4)]
        out-n (int-array 3)
        gcols (object-array [(ints-buf (map #(if (= :quantile-deviation (:kind %)) 1 0) groups))
                             (doubles-buf (map #(:quantile % 0.0) groups)) (doubles-buf (map #(:multiplier % 0.0) groups))
                             (ints-buf (map :n-jobs groups))])]
    (check! (first handles)
            (Native/stateSweep (long-array handles) (long-array [now-ms default-timeout-ms max-timeout-ms])
                               (count groups) gcols (int-array [n-rows n-entries]) (object-array lists) out-n nil)
            "cook_state_sweep")
    (let [l (fn [^ByteBuffer b i w] (if (= w 8) (.getLong b (int (* 8 i))) (.getInt b (int (* 4 i)))))
          rows (fn [n cols] (vec (for [i (range n)] (mapv (fn [[b w]] (l b i w)) cols))))]
      (cond-> {}
        (kinds :linger) (assoc :linger (rows (aget out-n 0) [[(lists 0) 8] [(lists 1) 4]]))
        (kinds :cancel) (assoc :cancel (rows (aget out-n 1) [[(lists 2) 8] [(lists 3) 4]]))
        (kinds :straggler) (assoc :straggler (rows (aget out-n 2) [[(lists 4) 4] [(lists 5) 8] [(lists 6) 4]]))))))

;; ---------------------------------------------------------------------------------------------
;; /unscheduled_jobs over a resident pool: the device half of reasons (unscheduled.clj:172-200)
(def ^:const unsched-ahead 10)

(defn unscheduled!
  "The queried job ids of one pool's handle: [{:status (:absent :waiting :running) :usage {:count :cpus :mem :gpus}
   (waiting: the user's running jobs plus the job) :position :ahead [job ids] :plugin-deferred?}] by query.  The
   handler compares :usage with the user's quota and share in the pool (strict >, only the keys present) and assembles
   the reasons in the reference's order, as cook_b200/cycle.py's unscheduled_reasons does."
  [handle job-ids]
  (let [n (count job-ids)
        st (direct (max 1 n)) us (direct (* 32 (max 1 n))) pos (direct (* 4 (max 1 n))) na (direct (* 4 (max 1 n)))
        ah (direct (* 8 unsched-ahead (max 1 n))) pl (direct (max 1 n))]
    (check! handle (Native/stateUnscheduled handle n (longs-buf job-ids) st us pos na ah pl nil)
            "cook_state_unscheduled")
    (vec (for [i (range n)]
           (let [k (.getInt ^ByteBuffer na (int (* 4 i)))]
             {:status ([:absent :waiting :running] (.get ^ByteBuffer st (int i)))
              :usage (zipmap [:count :cpus :mem :gpus] (for [c (range 4)] (.getDouble ^ByteBuffer us (int (* 8 (+ (* 4 i) c))))))
              :position (.getInt ^ByteBuffer pos (int (* 4 i)))
              :ahead (vec (for [j (range k)] (.getLong ^ByteBuffer ah (int (* 8 (+ (* unsched-ahead i) j))))))
              :plugin-deferred? (= 1 (.get ^ByteBuffer pl (int i)))})))))

;; ---------------------------------------------------------------------------------------------
;; /usage over resident pools: the device half of get-user-usage (api.clj:2946-2969)
(defn user-usage!
  "The running usage of the user codes `users` (nil: every user) over `handles` (one device; a pool per handle).
   `n-rows` is the live running rows over the handles (the shim's count, which bounds the queried users' rows).
   Returns [{:user :scope (-1 or the handle index) :group (-2 total, -1 ungrouped, else the group code) :jobs :cpus :mem
   :gpus :job-ids (group segments with by-group?)}] in (user, scope, group) order; the handler builds the reference's
   response (zero maps, pool names, group uuids and names, job uuids) as cook_b200/cycle.py's usage_response does."
  [handles users per-pool? by-group? n-rows]
  (let [L (* (if per-pool? 2 1) (if by-group? 2 1))
        seg-cap (* L n-rows) job-cap (if by-group? (* (if per-pool? 2 1) n-rows) 0)
        m (max 1 seg-cap)
        segs [(direct (* 4 m)) (direct (* 4 m)) (direct (* 4 m)) (direct (* 8 m)) (direct (* 8 m)) (direct (* 8 m))
              (direct (* 8 m)) (when by-group? (direct (* 4 m)))]
        jids (when by-group? (direct (* 8 (max 1 job-cap))))
        out-n (int-array 2)]
    (check! (first handles)
            (Native/stateUserUsage (long-array handles) (count users) (when users (ints-buf users)) (if per-pool? 1 0)
                                   (if by-group? 1 0) (int-array [seg-cap job-cap]) (object-array segs) jids out-n nil)
            "cook_state_user_usage")
    (let [i32 (fn [^ByteBuffer b d] (.getInt b (int (* 4 d))))
          f64 (fn [^ByteBuffer b d] (.getDouble b (int (* 8 d))))]
      (vec (for [d (range (aget out-n 0))]
             (let [g (i32 (segs 2) d) jobs (.getLong ^ByteBuffer (segs 3) (int (* 8 d)))]
               (cond-> {:user (i32 (segs 0) d) :scope (i32 (segs 1) d) :group g :jobs jobs
                        :cpus (f64 (segs 4) d) :mem (f64 (segs 5) d) :gpus (f64 (segs 6) d)}
                 (and by-group? (not= g -2))
                 (assoc :job-ids (let [o (i32 (segs 7) d)]
                                   (vec (for [j (range jobs)] (.getLong ^ByteBuffer jids (int (* 8 (+ o j))))))))))))))))

;; ---------------------------------------------------------------------------------------------
;; /stats/instances over resident pools: the device half of task-stats/get-stats (task_stats.clj), for status running
;; or unknown (the running rows) and success or failed (the finished-instance histories) without a name filter; the
;; handler keeps the Datomic path for a name filter and for a window that starts before a history's horizon.  Pools on
;; several devices are answered by one call: the other devices' rows are gathered to the first handle's device
(def ^:private instance-stats-leaders 10)
(defn instance-stats!
  "Instance stats over `handles` (one device or several): `status` :running or :unknown (the live running rows, one `now-ms`) or
   :success or :failed (the handles' histories, history-seed!; now-ms unused), the window [start-ms, end-ms), the
   entity-id bounds [task-id-lo, task-id-hi) (d/entid-at of start - 1 h and end + 1 h).  `n-rows` sizes the segments:
   the live running rows over the handles (the shim's count); for a history, a capacity the call may refuse with the
   count it needs (cook_state_history_stats' COOK_E_TOO_LARGE), and the handler retries with that count.  A name
   filter or a window before a history's horizon keep the Datomic path.  Returns {:segments [{:kind 0|1|2 (overall, reason, user and
   reason) :user :reason (-1: none) :count :totals [run cpu mem] :percentiles [[p50 p75 p95 p99 p100] x3]}]
   :leaders-cpu [[user total]] :leaders-mem [[user total]]}; the handler builds the response (user names, reason
   strings, the nil reason's key) as cook_b200/cycle.py's instance_stats_response does."
  [handles status now-ms start-ms end-ms task-id-lo task-id-hi n-rows]
  (let [cap (+ 1 (* 2 n-rows))
        segs [(direct (* 4 cap)) (direct (* 4 cap)) (direct (* 4 cap)) (direct (* 8 cap)) (direct (* 24 cap))
              (direct (* 120 cap))]
        leaders [(direct (* 4 2 instance-stats-leaders)) (direct (* 8 2 instance-stats-leaders))]
        out-n (int-array 2)]
    (check! (first handles)
            (Native/stateInstanceStats (long-array handles) (long-array [now-ms start-ms end-ms task-id-lo task-id-hi])
                                       (case status :running 0 :unknown 1 :success 2 :failed 3) (int cap)
                                       (object-array segs)
                                       (object-array leaders) out-n nil)
            "cook_state_instance_stats")
    (let [i32 (fn [^ByteBuffer b d] (.getInt b (int (* 4 d))))
          f64 (fn [^ByteBuffer b d] (.getDouble b (int (* 8 d))))
          lead (fn [k] (vec (for [i (range (aget out-n 1))]
                              [(i32 (leaders 0) (+ (* k instance-stats-leaders) i))
                               (f64 (leaders 1) (+ (* k instance-stats-leaders) i))])))]
      {:segments (vec (for [d (range (aget out-n 0))]
                        {:kind (i32 (segs 0) d) :user (i32 (segs 1) d) :reason (i32 (segs 2) d)
                         :count (.getLong ^ByteBuffer (segs 3) (int (* 8 d)))
                         :totals (vec (for [m (range 3)] (f64 (segs 4) (+ (* 3 d) m))))
                         :percentiles (vec (for [m (range 3)]
                                             (vec (for [j (range 5)] (f64 (segs 5) (+ (* 15 d) (* 5 m) j))))))}))
       :leaders-cpu (lead 0)
       :leaders-mem (lead 1)})))

;; ---------------------------------------------------------------------------------------------
;; /list and /jobs over resident pools: the device half of get-active-jobs-by-user-and-state (tools.clj:445-466) for
;; the waiting and running states (completed, success and failed: list-completed below); a name filter and a non-zero
;; missing count keep the Datomic path
(defn list-facts!
  "The attributes the listing filters on, from the tx-report tap with each job upsert (which clears them), pending or
   running: [{:job-id :submit-ms :submit-pool (code, nil: none) :custom-executor (true, false or nil)}].  They never
   change over a job's life, so a launch and a requeue keep them."
  [handle jobs]
  (check! handle (Native/stateListFacts handle (count jobs) (longs-buf (map :job-id jobs))
                                        (longs-buf (map :submit-ms jobs)) (ints-buf (map #(or (:submit-pool %) -1) jobs))
                                        (ints-buf (map #(case (:custom-executor %) true 1 false 0 -1) jobs)))
          "cook_state_list_facts"))

(defn list-jobs
  "`user`'s jobs in `states` (#{:waiting :running}) over `handles` (one device) submitted in [start-ms, end-ms), with
   entity ids in [job-id-lo, job-id-hi) (d/entid-at of start - 1 h and end + 1 h), in pool `pool-code` (-1: any;
   `handle-pools` each handle's pool code), only false custom executors unless `include-custom-executor?`, each state
   cut to `limit`.  The call is made with `cap` entries and, when it needs more, once more with the count it reports.
   Returns {:waiting [job-id] :running [job-id] :submit-ms {job-id ms} :missing n}, each state in entity-id order, for
   fetch-job-map; a non-zero :missing keeps the Datomic path.  The handler merges and orders the states as
   cook_b200/cycle.py's list_jobs_response does."
  [handles user states start-ms end-ms job-id-lo job-id-hi pool-code handle-pools include-custom-executor? limit cap]
  (loop [cap (max cap 1) tries 2]
    (let [outs [(direct (* 4 cap)) (direct (* 8 cap)) (direct (* 8 cap)) (direct (* 4 cap))]
          out-n (int-array 2)
          rc (Native/stateListJobs (long-array handles) (long-array [start-ms end-ms job-id-lo job-id-hi])
                                   (int-array [user (+ (if (states :waiting) 1 0) (if (states :running) 2 0)) pool-code
                                               (if include-custom-executor? 1 0) limit cap])
                                   (when (not= pool-code -1) (ints-buf handle-pools)) (object-array outs) out-n nil)]
      (if (and (= rc -7) (> tries 1))
        (recur (aget out-n 0) (dec tries))
        (do (check! (first handles) rc "cook_state_list_jobs")
            (let [n (aget out-n 0)
                  at (fn [i] {:state (.getInt ^ByteBuffer (outs 0) (int (* 4 i)))
                              :job-id (.getLong ^ByteBuffer (outs 1) (int (* 8 i)))
                              :submit-ms (.getLong ^ByteBuffer (outs 2) (int (* 8 i)))})
                  es (mapv at (range n))]
              {:waiting (vec (for [e es :when (= 1 (:state e))] (:job-id e)))
               :running (vec (for [e es :when (= 2 (:state e))] (:job-id e)))
               :submit-ms (into {} (map (juxt :job-id :submit-ms)) es)
               :missing (aget out-n 1)}))))))

;; The completed, success and failed states from each handle's completed-job log.  The tap sends completed-record!
;; one record per job per transaction, its columns read from the db-after entity, its stamp the transaction's t:
;;   :job/state becomes :job.state/completed      -> :success or :failed, by tools/job-ent->state
;;   :job/state leaves :job.state/completed       -> :reopened (:job/ensure-not-completed, :job/update-retry-count)
;;   a completed job gains a successful instance  -> :success
;;   a listed attribute of a completed job changes (user, submit time, submit pool, custom executor) -> a new record
;; The listing handler sends a completed-family state to list-completed when there is no name filter, every handle's
;; log is on and start >= every horizon, the request's pools on one device or several; otherwise the Datomic path.
(def ^:private completed-kinds {:success 1 :failed 2 :reopened 3})
(defn- completed-cols [rows]
  (object-array [(longs-buf (map :job-id rows)) (longs-buf (map :stamp rows)) (ints-buf (map :user rows))
                 (longs-buf (map :submit-ms rows)) (ints-buf (map #(or (:submit-pool %) -1) rows))
                 (ints-buf (map #(case (:custom-executor %) true 1 false 0 -1) rows))
                 (let [b (direct (count rows))]
                   (doseq [[i r] (map-indexed vector rows)] (.put b (int i) (byte (completed-kinds (:kind r)))))
                   b)]))

(defn completed-seed!
  "At start-up and on a leadership change, after the reset and the load and before the tap resumes: the pool's
   completed jobs with submit >= since-ms, read once from one database value, [{:job-id :stamp (its basis t) :user
   (code) :submit-ms :submit-pool (code, nil: none) :custom-executor (true, false or nil) :kind (:success or
   :failed)}].  Turns the log on at horizon since-ms."
  [handle since-ms rows]
  (check! handle (Native/stateCompletedSeed handle (long since-ms) (count rows) (completed-cols rows))
          "cook_state_completed_seed"))

(defn completed-record!
  "The tap's records of one transaction, as completed-seed!'s rows with :kind also :reopened; those submitted before
   the horizon are skipped by the call."
  [handle rows]
  (check! handle (Native/stateCompletedRecord handle (count rows) (completed-cols rows)) "cook_state_completed_record"))

(defn completed-advance!
  "Periodically, with now - retention (the shim's setting, default 32 days): the horizon rises and the records of
   jobs submitted before it leave."
  [handle since-ms]
  (check! handle (Native/stateCompletedAdvance handle (long since-ms)) "cook_state_completed_advance"))

(defn list-completed
  "`user`'s jobs whose latest record over `handles` (one device or several) is in `state` (:success, :failed or :completed),
   submitted in [start-ms, end-ms), with entity ids in [job-id-lo, job-id-hi), in pool `pool-code` (-1: any;
   `handle-pools` each handle's pool code), only false custom executors unless `include-custom-executor?`, cut to
   `limit` in entity-id order.  The call is made with `cap` entries and, when it needs more, once more with the count
   it reports.  Returns {:job-ids [job-id] :submit-ms {job-id ms}}, the handler's completed part of
   list_jobs_response."
  [handles user state start-ms end-ms job-id-lo job-id-hi pool-code handle-pools include-custom-executor? limit cap]
  (loop [cap (max cap 1) tries 2]
    (let [outs [(direct (* 8 cap)) (direct (* 8 cap)) (direct (* 4 cap))]
          out-n (int-array 1)
          rc (Native/stateListCompleted (long-array handles) (long-array [start-ms end-ms job-id-lo job-id-hi])
                                        (int-array [user ({:success 1 :failed 2 :completed 3} state) pool-code
                                                    (if include-custom-executor? 1 0) limit cap])
                                        (when (not= pool-code -1) (ints-buf handle-pools)) (object-array outs) out-n nil)]
      (if (and (= rc -7) (> tries 1))
        (recur (aget out-n 0) (dec tries))
        (do (check! (first handles) rc "cook_state_list_completed")
            (let [n (aget out-n 0)
                  ids (mapv #(.getLong ^ByteBuffer (outs 0) (int (* 8 %))) (range n))]
              {:job-ids ids
               :submit-ms (zipmap ids (map #(.getLong ^ByteBuffer (outs 1) (int (* 8 %))) (range n)))}))))))

;; ---------------------------------------------------------------------------------------------
;; the match-cycle metrics of a resident pool (handle-match-cycle-metrics scheduler.clj:1210-1280, the unmatched
;; tracking :1399-1486), called after the match and before the launches
(def ^:private jf-gpus 1) (def ^:private jf-disk 2) (def ^:private jf-disk-request 4) (def ^:private jf-disk-limit 8)
(def ^:private jf-uris 16)
(defn job-facts!
  "The stats keys of live pending jobs, from the tx-report tap after each pending upsert (which clears them): `jobs` is
   [{:job-id :resources (tools/job-ent->resources) :gpu-model (the job's COOK_GPU_MODEL or nil)}]; the model and disk
   type names are coded through `gpu-models` and `disk-types` (dictionary)."
  [handle gpu-models disk-types jobs]
  (let [facts (for [{:keys [resources]} jobs
                    :let [{:keys [gpus disk uris]} resources]]
                (cond-> 0
                  gpus (bit-or jf-gpus)
                  disk (bit-or jf-disk)
                  (some? (:request disk)) (bit-or jf-disk-request)
                  (some? (:limit disk)) (bit-or jf-disk-limit)
                  (seq uris) (bit-or jf-uris)))]
    (check! handle (Native/stateJobFacts handle (count jobs) (longs-buf (map :job-id jobs))
                                         (let [b (direct (count jobs))]
                                           (doseq [[i f] (map-indexed vector facts)] (.put b (int i) (byte f))) b)
                                         (ints-buf (map #(code! gpu-models (:gpu-model %)) jobs))
                                         (doubles-buf (map #(or (get-in % [:resources :disk :request]) 0.0) jobs))
                                         (doubles-buf (map #(or (get-in % [:resources :disk :limit]) 0.0) jobs))
                                         (ints-buf (map #(code! disk-types (get-in % [:resources :disk :type])) jobs)))
            "cook_state_job_facts")))

(def ^:private mm-first 10)
(defn match-metrics!
  "The metrics of the last resident match on `handle`: `dropped` are the considerable positions whose matches
   filter-matches-for-ratelimit dropped.  With more keys than `key-cap` the call reports the count and the round stays
   uncounted, so this retries once with it.  Returns {:counts [considerable matched head-job-id head-matched uris
   uris-position keys too-long first] :amounts [total-cpus total-mem p50 p95 p100 (cpus) p50 p95 p100 (mem)]
   :rows [{:ints [job-id position user ports facts gpu-model disk-type] :amounts [cpus mem gpus disk-request
   disk-limit]} x3 (head, largest by cpus, largest by mem)] :first [[job-id cycles]] :users [[considerable matched]]
   :keys [[kind code total]]}; the handler builds the log maps and the warning as cook_b200/cycle.py's
   match_cycle_metrics_response does."
  [handle n-users dropped unmatched-warn-cycles key-cap]
  (loop [cap (max 1 key-cap) tries 0]
    (let [outs [(direct (* 8 9)) (direct (* 8 8)) (direct (* 8 21)) (direct (* 8 15)) (direct (* 8 mm-first))
                (direct (* 4 mm-first)) (direct (* 4 n-users)) (direct (* 4 n-users)) (direct (* 4 cap))
                (direct (* 4 cap)) (direct (* 8 cap))]
          rc (Native/stateMatchMetrics handle n-users (count dropped) (when (seq dropped) (ints-buf dropped))
                                       unmatched-warn-cycles cap (object-array outs) nil)
          i64 (fn [^ByteBuffer b d] (.getLong b (int (* 8 d))))
          i32 (fn [^ByteBuffer b d] (.getInt b (int (* 4 d))))
          f64 (fn [^ByteBuffer b d] (.getDouble b (int (* 8 d))))
          n-keys (i64 (outs 0) 6)]
      (if (and (= rc -7) (zero? tries) (> n-keys cap))
        (recur (int n-keys) 1)
        (do
          (check! handle rc "cook_state_match_metrics")
          {:counts (vec (for [i (range 9)] (i64 (outs 0) i)))
           :amounts (vec (for [i (range 8)] (f64 (outs 1) i)))
           :rows (vec (for [r (range 3)] {:ints (vec (for [i (range 7)] (i64 (outs 2) (+ (* 7 r) i))))
                                          :amounts (vec (for [i (range 5)] (f64 (outs 3) (+ (* 5 r) i))))}))
           :first (vec (for [i (range (i64 (outs 0) 8))] [(i64 (outs 4) i) (i32 (outs 5) i)]))
           :users (vec (for [u (range n-users)] [(i32 (outs 6) u) (i32 (outs 7) u)]))
           :keys (vec (for [d (range n-keys)] [(i32 (outs 8) d) (i32 (outs 9) d) (f64 (outs 10) d)]))})))))
