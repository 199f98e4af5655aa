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

(defn rebalance-derived!
  "cook_state_rebalance_derived: the rebalancer over the resident rows with the groups' cotask lists derived on the
   device over the host table in `args` (Native/stateRebalance's arguments after the handle)."
  [handle args]
  (check! handle (apply #(Native/stateRebalanceDerived handle %&) args) "cook_state_rebalance_derived"))

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
