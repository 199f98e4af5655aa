/*
 * cook_gpu.h — C ABI of libcookgpu.so: the H100-native replacement for Cook's
 * per-cycle scheduling hot path (DRU rank -> constraint-and-fit match ->
 * rebalancer preemption search).
 *
 * There is NO existing FFI for this path in the reference (SURVEY.md §8b): the
 * seams are JVM-level.  Each entry point below names the reference function it
 * replaces (paths relative to /root/reference/scheduler/src/cook/).
 *
 * Conventions
 *  - Plain C: pointers + sizes, caller owns every input and output buffer
 *    (JVM direct ByteBuffers / numpy arrays / malloc).  The library owns device
 *    memory and the CUDA context.
 *  - Every function returns int32: 0 = COOK_OK, negative = error.  Nothing
 *    throws or aborts across the boundary; on error no output is valid.
 *    cook_last_error() returns the message of the last failure on the handle.
 *  - A cook_pool handle is per Cook pool; calls on one handle must be
 *    serialised by the caller (exactly where Cook has `(locking fenzo ...)`,
 *    scheduler/scheduler.clj:665).  Different handles may be used concurrently
 *    and may live on different GPUs.
 *  - All "id"/"idx" columns are dense int32 dictionary codes built by the host
 *    shim; -1 means "absent / nil" unless stated otherwise.
 *  - All resource amounts are IEEE f64, exactly as Datomic's :resource/amount
 *    (:db.type/double).  Bit-exact parity with the JVM path is guaranteed when
 *    amounts lie on a binary grid (multiples of 2^-10 below 2^40), see DESIGN.md.
 *
 * The CPU oracle (oracle/cook_oracle.cpp, TEST INFRASTRUCTURE ONLY) exports the
 * same signatures with the prefix `oracle_` so tests can diff the two.
 */
#ifndef COOK_GPU_H
#define COOK_GPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ errors */
enum {
  COOK_OK = 0,
  COOK_E_BADARG = -1,
  COOK_E_CUDA = -2,
  COOK_E_NCCL = -3,
  COOK_E_OOM = -4,
  COOK_E_UNSUPPORTED_CONSTRAINT = -5,
  COOK_E_NO_DEVICE = -6,
  COOK_E_TOO_LARGE = -7   /* a table exceeds what the kernels keep on chip (e.g. a constraint pool of more
                             than ~130k offers: its verdict-bit rows live in the resolver's shared memory);
                             split the pool - nothing was computed */
};

typedef struct cook_ctx cook_ctx;   /* process-wide: devices (+ NCCL comm)   */
typedef struct cook_pool cook_pool; /* one per Cook pool, pinned to a device */

/* -------------------------------------------------------------- lifetime */
/* Called once per leadership (replaces per-pool make-fenzo-state,
 * scheduler/scheduler.clj:2301-2324, wired at mesos.clj:193). */
typedef struct {
  int32_t n_devices;          /* 0 => use current device only            */
  const int32_t* device_ids;  /* may be NULL when n_devices == 0         */
} cook_gpu_config;

int32_t cook_gpu_init(const cook_gpu_config* cfg, cook_ctx** out);
int32_t cook_gpu_shutdown(cook_ctx* ctx);

/* dru_mode: 0 = :pool.dru-mode/default, 1 = :pool.dru-mode/gpu (pool.clj:64-85) */
int32_t cook_pool_open(cook_ctx* ctx, const char* pool_name, int32_t dru_mode,
                       int32_t device, cook_pool** out);
int32_t cook_pool_close(cook_pool* pool);
/* Copies the last error text (NUL terminated) for this pool handle. */
int32_t cook_last_error(cook_pool* pool, char* buf, int32_t len);
/* Library identification: "cook_b200 <ver> sm_90a". */
const char* cook_gpu_version(void);

/* ------------------------------------------------------------- data model */

/* Tasks for ranking: running instances and synthetic tasks of pending jobs
 * (tools.clj:582-588 create-task-ent).  Feature vector = tools.clj:614-632:
 * [-priority, start-time, task :db/id, job :db/id].                        */
typedef struct {
  int32_t n;
  const int32_t* user;       /* index into cook_user_table                    */
  const int32_t* priority;   /* :job/priority (default 50)                    */
  const int64_t* start_time; /* ms; pending => INT64_MAX (Date Long/MAX)      */
  const int64_t* task_id;    /* task :db/id; pending => -1 (nil sorts first)  */
  const int64_t* job_id;     /* job :db/id                                    */
  const double* cpus;
  const double* mem;
  const double* gpus;        /* 0.0 when the job has no :gpus resource        */
} cook_tasks_soa;

/* Per-user tables (dense, indexed by user code).
 * divisors: share.clj:189-210 (user share, else "default" user's, else
 * Double/MAX_VALUE).  quota: quota.clj:272-295 (missing key => 0, as
 * tools.clj:876-881 below-quota? does).  usage/tokens are only read by
 * cook_match (scheduler.clj:711-727, tools.clj:940-959).                   */
typedef struct {
  int32_t n_users;
  const int32_t* name_rank;  /* rank of the user name in ascending string order
                                (dru.clj:123 `(sort-by first)`); unique       */
  const double* div_mem;
  const double* div_cpus;
  const double* div_gpus;
  const double* quota_count;
  const double* quota_cpus;
  const double* quota_mem;
  const double* quota_gpus;
  const double* usage_count; /* match only; may be NULL for rank             */
  const double* usage_cpus;
  const double* usage_mem;
  const double* usage_gpus;
  const int32_t* tokens;     /* match only: launch-rate tokens left          */
} cook_user_table;

/* Global pool quota / quota-group quota (tools.clj:917-933); enabled == 0
 * means `(nil? quota)` => no filtering.                                     */
typedef struct {
  int32_t enabled;
  double count, cpus, mem, gpus;
} cook_pool_quota;

typedef struct {
  int32_t max_over_quota_jobs; /* config.clj:413-416, default 100            */
  int32_t filter_offensive;    /* scheduler.clj:2198-2229                    */
  double offensive_max_mem_mb; /* (* 1024.0 max-memory-gb)                   */
  double offensive_max_cpus;
} cook_rank_params;

/* R1-R7: one call per rank cycle per pool.  Replaces
 * sort-jobs-by-dru-helper (scheduler.clj:2073-2091) + filter-based-on-quota
 * (:2134-2157) + filter-offensive-jobs (:2198-2229).
 *   group_usage[4] = {count,cpus,mem,gpus} aggregate running usage of the
 *   pool's quota group (aggregate-quota-groups :2125-2132); ignored when
 *   group_quota->enabled == 0.
 * Outputs:
 *   out_ranked_idx[<= pending->n]  pending indices in final queue order
 *   out_n                          number of entries written
 *   out_dru[running->n + pending->n]  DRU per task (running first, then
 *       pending, in input order); NaN for tasks cut by limit-over-quota-jobs
 *   out_order[running->n + pending->n] the full merged order (task indices,
 *       running 0..R-1, pending R..R+J-1) before pending/quota filtering;
 *       out_order_n entries.  May be NULL.                                   */
int32_t cook_rank(cook_pool* pool, const cook_tasks_soa* running,
                  const cook_tasks_soa* pending, const cook_user_table* users,
                  const cook_pool_quota* pool_quota,
                  const cook_pool_quota* group_quota, const double* group_usage,
                  const cook_rank_params* params, int32_t* out_ranked_idx,
                  int32_t* out_n, double* out_dru, int32_t* out_order,
                  int32_t* out_order_n);

/* Pending jobs as the matcher sees them (TaskRequestAdapter,
 * scheduler.clj:456-509) + the closed, data-driven encoding of Cook's
 * JobConstraint records (constraints.clj:459-464).  Any pointer in the
 * constraint section may be NULL => that constraint is absent for all jobs. */
typedef struct {
  int32_t n;
  const int32_t* user;
  const double* cpus;
  const double* mem;
  const double* gpus;           /* 0.0 => none                                */
  const int32_t* ports;         /* :job/ports count (may be NULL => 0)        */
  const uint8_t* allowed;       /* tools.clj:572-580 job-allowed-to-start?    */
  const uint8_t* plugin_accept; /* plugins/launch.clj:136-140                 */
  /* --- constraints ------------------------------------------------------- */
  /* novel-host (constraints.clj:68-94): CSR of hostname ids to avoid       */
  const int32_t* novel_off;     /* [n+1]                                      */
  const int32_t* novel_host;
  /* gpu-host (constraints.clj:122-157): model id requested (-1 when gpus==0)*/
  const int32_t* gpu_model;
  /* disk-host (constraints.clj:164-199): request < 0 => constraint not built*/
  const double* disk_request;
  const int32_t* disk_type;
  /* user-defined EQUALS (constraints.clj:355-383): CSR of (attr column, value
   * id); value id -1 => pattern not in the host dictionary (never matches)  */
  const int32_t* attr_off;      /* [n+1]                                      */
  const int32_t* attr_col;
  const int32_t* attr_val;
  /* estimated-completion (constraints.clj:385-431): end time ms, -1 => none */
  const int64_t* est_end_ms;
  /* checkpoint-locality (constraints.clj:201-240): location id, -1 => none  */
  const int32_t* ckpt_location;
  /* rebalancer-reservation (constraints.clj:242-252, scheduler.clj:645-653):
   * hostname id reserved FOR this job, -1 => none                           */
  const int32_t* reserved_host;
  /* group membership (:group/_job): CSR of group indices                    */
  const int32_t* group_off;     /* [n+1]                                      */
  const int32_t* group_idx;
} cook_jobs_soa;

/* One entry per assignable VM = all live leases merged per hostname
 * (VirtualMachineLeaseAdapter offer.clj:48-72; get-offer-attr-map :31-46).  */
typedef struct {
  int32_t n;
  const int32_t* hostname_id;  /* global hostname dictionary code             */
  const int32_t* name_rank;    /* byte-order rank of hostname among the n
                                  offers; unique. Tie-break of equal fitness  */
  const double* cpus;          /* Σ lease cpuCores                            */
  const double* mem;           /* Σ lease memoryMB                            */
  /* Fenzo's task-assigner state for the host (scheduler.clj:877-881):       */
  const double* run_cpus;      /* Σ cpus of running tasks Fenzo tracks there  */
  const double* run_mem;
  const int32_t* run_count;
  /* port ranges CSR (offer.clj:70-72); may be NULL => no ports              */
  const int32_t* port_off;     /* [n+1]                                       */
  const int32_t* port_begin;
  const int32_t* port_end;     /* inclusive                                   */
  /* attributes                                                              */
  const uint8_t* is_k8s;       /* "compute-cluster-type" == "kubernetes"      */
  const int32_t* location;     /* COOK_COMPUTE_CLUSTER_LOCATION id, -1 nil    */
  const int32_t* gpu_off;      /* CSR of "gpus" model->count map; NULL => {}  */
  const int32_t* gpu_model;
  const double* gpu_count;
  const int32_t* disk_off;     /* CSR of "disk" type->MiB map; NULL => {}     */
  const int32_t* disk_type;
  const double* disk_space;
  const int32_t* max_tasks;    /* COOK_MAX_TASKS_PER_HOST, -1 absent          */
  const int32_t* num_tasks;    /* COOK_NUM_TASKS_ON_HOST                      */
  const int64_t* host_start_time; /* "host-start-time" seconds, -1 absent     */
  int32_t n_attr_cols;
  const int32_t* attr;         /* [n_attr_cols][n] value ids, 0 => absent     */
  const uint8_t* reserved;     /* hostname in (vals job-uuid->reserved-host)  */
} cook_offers_soa;

/* Group host-placement constraints (constraints.clj:568-655).  cot_* lists,
 * per group, the cotasks Fenzo's tracker knows as running
 * (get-cotasks-from-tracker-state :539-552): their hostname id and the value
 * id of the group's attribute on that host's lease (0 => nil).              */
enum { COOK_GROUP_UNIQUE = 0, COOK_GROUP_BALANCED = 1, COOK_GROUP_ATTR_EQUALS = 2 };
typedef struct {
  int32_t n_groups;
  const int32_t* kind;
  const int32_t* attr_col;     /* balanced / attribute-equals                 */
  const int32_t* minimum;      /* :host-placement.balanced/minimum            */
  const int32_t* cot_off;      /* [n_groups+1]                                */
  const int32_t* cot_hostname_id;
  const int32_t* cot_attr_val;
} cook_groups;

typedef struct {
  int32_t num_considerable;      /* scheduler.clj:750 `(take num-considerable)` */
  int32_t enforce_rate_limit;    /* ratelimit/enforce? (tools.clj:942)          */
  int32_t host_lifetime_mins;    /* estimated-completion config                 */
  int32_t fitness_kind;          /* 0 = cpuMemBinPacker (config.clj:108)        */
  double good_enough_fitness;    /* must be >= 1.0 (deterministic mode, F3)     */
  int32_t reuse_resident;        /* 1: inputs are unchanged since the previous
                                    cook_match on this handle and still in HBM:
                                    skip the upload stage (columnar-mirror mode,
                                    SURVEY §8f-1); error if nothing is resident */
  int32_t max_ctas;              /* 0 = the whole GPU.  > 0: the matcher kernel uses at
                                    most this many thread blocks (one per SM), so several
                                    pools of one GPU can run their cycles side by side
                                    (Cook's pools are independent, scheduler.clj:2425-2466);
                                    results do not depend on it                           */
} cook_match_params;

enum { /* out_fail_reason codes (first failing check on the LAST VM evaluated
          is not meaningful on a parallel machine; we report the most
          permissive class seen) */
  COOK_FAIL_NONE = 0, COOK_FAIL_RESOURCES = 1, COOK_FAIL_CONSTRAINT = 2,
  COOK_FAIL_NO_OFFERS = 3
};

typedef struct {
  int32_t n_considerable;
  int32_t n_matched;
  int32_t head_matched;   /* scheduler.clj:1613-1651 scale-back feedback       */
  int32_t n_offers_used;
  int64_t evals;          /* n_considerable x n_offers (SURVEY §8d)            */
  int64_t n_fast;         /* jobs resolved by the speculative fast path        */
  int64_t n_chunk_rescan; /* chunk re-evaluations in the serial phase          */
  int64_t n_full_rescan;  /* jobs that needed a full-row re-evaluation         */
  double ms_considerable; /* device time per phase (CUDA events)               */
  double ms_match;
  double ms_h2d;
  double ms_d2h;
  double ms_match_kernel; /* the persistent matcher kernel alone               */
  int64_t h2d_bytes;      /* bytes uploaded by this call                       */
  int64_t d2h_bytes;      /* bytes downloaded by this call                     */
  int32_t n_launches;     /* kernels launched by this call                     */
  int32_t reserved0;
} cook_match_stats;

/* M0-M6: one call per match cycle per pool.  Replaces
 * pending-jobs->considerable-jobs (scheduler.clj:729-762) +
 * TaskScheduler.scheduleOnce (:665-671, Fenzo 0.10.0).
 *   ranked_idx[n_ranked]: queue order = indices into jobs (cook_rank output).
 * Outputs (caller-allocated, capacity num_considerable each unless stated):
 *   out_considerable[k]  job index of the k-th considerable job
 *   out_assign[k]        offer index it was placed on, or -1
 *   out_ports[k*max_ports + p] assigned port numbers (may be NULL; max_ports
 *                        = max over jobs of ports)
 *   out_fail_reason[k]   COOK_FAIL_* for unplaced jobs (may be NULL)         */
int32_t cook_match(cook_pool* pool, const int32_t* ranked_idx, int32_t n_ranked,
                   const cook_jobs_soa* jobs, const cook_offers_soa* offers,
                   const cook_groups* groups, const cook_user_table* users,
                   const cook_pool_quota* pool_quota,
                   const cook_match_params* params, int32_t* out_considerable,
                   int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                   uint8_t* out_fail_reason, cook_match_stats* out_stats);

/* Placement-failure summaries (SURVEY §8f-3; fenzo_utils.clj:21-89, unscheduled.clj:77-107).
 * For each requested considerable job k (index into the out_considerable order of the LAST cook_match
 * on this handle) counts, over all offers, why the job could not go there AT ITS TURN - the VM
 * state after every earlier job of the cycle was placed, exactly what Fenzo's TaskAssignmentResults
 * of that scheduleOnce describe:
 *   counts[COOK_FAILC_CPUS], counts[COOK_FAILC_MEM]  VMs whose cpus / mem did not suffice (a VM
 *       short of both counts in both, like Fenzo's one AssignmentFailure per resource)
 *   counts[COOK_FAILC_FIRST_CONSTRAINT + i]          VMs with enough resources whose FIRST failing
 *       hard constraint was i, in Cook's evaluation order (constraints.clj:459-495):
 *       checkpoint-locality, estimated-completion, user-defined, disk-host, gpu-host, novel-host,
 *       max-tasks-per-host, rebalancer-reservation, unique / balanced / attribute-equals group
 *   n_passed   VMs that failed nothing (0 for a job that stayed unplaced; ports shortage is a
 *       resource failure without a message in Fenzo and is counted in n_ports only)            */
enum { COOK_FAILC_CPUS = 0, COOK_FAILC_MEM = 1, COOK_FAILC_FIRST_CONSTRAINT = 2, COOK_FAILC_N = 13 };
typedef struct {
  int32_t n_vms;
  int32_t n_passed;
  int32_t n_ports;
  int32_t counts[COOK_FAILC_N];
} cook_failure_counts;
int32_t cook_match_failures(cook_pool* pool, const int32_t* k_idx, int32_t n, cook_failure_counts* out);

/* ---------------------------------------------------------------- rebalance */
/* Running tasks with placement for the rebalancer (rebalancer.clj:222-266).  */
typedef struct {
  cook_tasks_soa t;
  const int32_t* host;       /* index into cook_host_table                    */
} cook_running_soa;

/* Hosts known to the rebalancer: union of hosts of running tasks and hosts
 * with spare resources (view-incubating-offers scheduler.clj:1537-1546),
 * attributes from the agent-attributes cache (tools.clj:713-716).           */
typedef struct {
  int32_t n;
  const int32_t* hostname_id;
  const int32_t* name_rank;    /* `(sort-by first)` rebalancer.clj:383        */
  const uint8_t* has_spare;    /* host present in host->spare-resources       */
  const double* spare_cpus;
  const double* spare_mem;
  const double* spare_gpus;
  const uint8_t* is_k8s;
  const int32_t* location;
  const int32_t* gpu_off;
  const int32_t* gpu_model;
  const double* gpu_count;
  const int32_t* disk_off;
  const int32_t* disk_type;
  const double* disk_space;
  const int64_t* host_start_time;
  int32_t n_attr_cols;
  const int32_t* attr;
} cook_host_table;

typedef struct {
  int32_t max_preemption;     /* rebalancer.clj:434 */
  double min_dru_diff;
  double safe_dru_threshold;
  int32_t host_lifetime_mins;
} cook_rebalance_params;

typedef struct {
  int32_t pending_idx;   /* job this decision makes room for                  */
  int32_t host;          /* index into cook_host_table                        */
  int32_t victim_begin;  /* slice of out_victims                              */
  int32_t victim_count;
  double dru, mem, cpus, gpus; /* rebalancer.clj:384-397 aggregation          */
} cook_decision;

/* B1-B6: one call per rebalance cycle per pool.  Replaces init-state
 * (rebalancer.clj:222-266) + rebalance (:434-467).  `pending` holds the
 * first jobs of the ranked queue that pass job-allowed-to-start?
 * (:588-590), in order.  out_victims entries are indices into `running`
 * (>= running->t.n  means the synthetic task of decision
 * (idx - running->t.n)), stored per decision in ASCENDING dru order (K22).
 * Capacity: out_decisions[max_preemption], out_victims[running->t.n +
 * max_preemption].                                                          */
int32_t cook_rebalance(cook_pool* pool, const cook_running_soa* running,
                       const cook_jobs_soa* pending,
                       const int64_t* pending_job_id,
                       const int32_t* pending_priority,
                       const cook_host_table* hosts,
                       const cook_groups* groups,
                       const cook_user_table* users,
                       const cook_rebalance_params* params,
                       cook_decision* out_decisions, int32_t* out_victims,
                       int32_t* out_n);

/* Diagnostic twin of cook_rebalance: the same walk, plus the rebalancer STATE the reference's own
 * tests read (test/cook/test/rebalancer.clj:115-196 compute-pending-default-job-dru, :813-988
 * next-state, :1368-1397 job-below-quota).  `forced` decisions are applied with next-state instead
 * of being searched, as those tests hand compute-next-state a decision.  All pointers optional.  */
typedef struct {
  int32_t n_forced;
  const cook_decision* forced;    /* pending_idx, host, victim slice, dru/mem/cpus/gpus            */
  const int32_t* forced_victims;  /* running-task indices, in selection (descending dru) order     */
  double* pending_dru;            /* [pending->n]; untouched for jobs the walk did not reach      */
  double* task_dru;               /* [running->t.n + max_preemption] after the last transition    */
  uint8_t* task_alive;            /* same length                                                  */
  int32_t* order;                 /* task->scored-task key order (priority map) afterwards        */
  int32_t* n_order;
  uint8_t* has_spare;             /* [hosts->n] host->spare-resources afterwards                  */
  double *spare_mem, *spare_cpus, *spare_gpus;
  int32_t forced_only;            /* 1: walk only the forced jobs; 0: forced jobs take their given
                                     decision, every other pending job is searched as usual       */
  uint8_t* below_quota;           /* [pending->n] job-below-quota for the jobs the walk reached   */
} cook_reb_trace;
int32_t cook_rebalance_trace(cook_pool* pool, const cook_running_soa* running,
                             const cook_jobs_soa* pending, const int64_t* pending_job_id,
                             const int32_t* pending_priority, const cook_host_table* hosts,
                             const cook_groups* groups, const cook_user_table* users,
                             const cook_rebalance_params* params, cook_decision* out_decisions,
                             int32_t* out_victims, int32_t* out_n, const cook_reb_trace* trace);

/* ------------------------------------------------------ resident pool state */
/* §8f-1, device half: the pool's pending jobs and running tasks stay on the device between cycles and
 * change by deltas, as Cook's own state changes by transactions (monitor-tx-report-queue,
 * scheduler.clj:378-448).  rank-jobs (:2262-2284) ranks them in place and the match cycles between two
 * ranks take from that queue, which loses only what the caller's launch deltas remove
 * (remove-matched-jobs-from-pending-jobs :790-795).  Nothing that scales with the pool is uploaded or
 * scanned on the host per cycle.
 *
 * One batch of changes, applied all or nothing:
 *   reset               drop every row first (new leadership)
 *   pending             upserts keyed by pending_job_id: the columns of cook_jobs_soa, CSR lists over
 *                       the delta rows, plus pending_priority.  A pending row ranks with start_time =
 *                       INT64_MAX and task_id = -1.  Required: user, cpus, mem, pending_priority,
 *                       pending_job_id; a NULL column takes its "absent" value (gpus 0, ports 0, allowed
 *                       and plugin_accept 1, gpu_model / disk_type / ckpt_location / reserved_host -1,
 *                       disk_request -1, est_end_ms -1, empty lists).  An upsert of a known id replaces
 *                       the row.
 *   pending_rm_job_id   removals
 *   running             running-task upserts keyed by task_id (all cook_tasks_soa columns but gpus)
 *   running_rm_task_id  removals
 *   running_hostname_id the host of each running upsert: a code of the global hostname dictionary (the
 *                       code space of cook_offers_soa.hostname_id and cook_host_table.hostname_id).  NULL
 *                       stores -1, "host unknown"; cook_state_rebalance, cook_state_usage and
 *                       cook_state_cotasks read it.
 *   running_group_off   the group list of each running upsert, its job's groups (:group/_job): CSR
 *   running_group_idx   offsets [running.n + 1] over the upserts and group codes.  NULL stores empty lists.
 *                       Only cook_state_cotasks reads them.
 * An upsert of a known id replaces the row with its lists; a removal or reset drops them.
 * A launch can be one batch (remove pending job j, upsert its running task with j's group list);
 * cook_state_launch does the same from job ids without re-sending the rows.  An upsert of a pending row gives
 * it a new generation, so it leaves the last rank's queue; cook_state_patch changes the match-time columns
 * without that.
 * COOK_E_BADARG, state unchanged: an unknown id in a removal, an id twice in one table of the batch, a
 * malformed CSR offset column, a negative user / attr_col / group (pending or running) / novel hostname
 * code, a reserved_host or running_hostname_id below -1.
 * Codes are checked here, when they enter; their maxima are kept on the host, and rank / match reject a
 * user, offer or group table too small for them.  Group codes and attribute value codes must therefore
 * come from stable, append-only dictionaries (INTEGRATION.md §3b).
 * Uploads exactly: every non-NULL column of the delta (n rows; CSR offsets n+1, lists their length)
 * plus one int32 slot per upserted or removed row.  Statistics: cook_last_stats(COOK_PHASE_STATE).   */
typedef struct {
  int32_t reset;
  cook_jobs_soa pending;
  const int32_t* pending_priority;
  const int64_t* pending_job_id;
  int32_t n_pending_rm;
  const int64_t* pending_rm_job_id;
  cook_tasks_soa running;
  int32_t n_running_rm;
  const int64_t* running_rm_task_id;
  const int32_t* running_hostname_id;
  const int32_t* running_group_off;
  const int32_t* running_group_idx;
} cook_state_delta;
int32_t cook_state_apply(cook_pool* pool, const cook_state_delta* delta);

/* Launches by job id: live pending job job_id[i] becomes running task task_id[i], started at start_time[i] on
 * hostname_id[i] (a code of the global hostname dictionary; a NULL column stores -1, "host unknown").  User,
 * priority, job id, cpus, mem and gpus are copied on the device from the pending row.  Leaves exactly the
 * state cook_state_apply leaves after the batch pending_rm_job_id = job_id plus the running upserts built
 * from those rows with running_hostname_id = hostname_id and, as running_group_off / running_group_idx, the
 * pending rows' group lists: the job leaves the last rank's queue, its counts and reservation leave with the
 * row, its group list moves to the task (copied on the device, in launch order) while its other list
 * entries leave, and the list arenas compact by the same rule.
 * COOK_E_BADARG, before any change: n < 0; a NULL job_id, task_id or start_time while n > 0; a job id that
 * is not live or appears twice; a task id that appears twice or is already live; a hostname code below -1.
 * Uploads exactly n * (4 + 4 + 8 + 8) bytes (pending slot, running slot, task id, start time), plus 4 * n
 * when hostname_id is not NULL.  Statistics: cook_last_stats(COOK_PHASE_STATE).                        */
int32_t cook_state_launch(cook_pool* pool, int32_t n, const int64_t* job_id, const int64_t* task_id,
                          const int64_t* start_time, const int32_t* hostname_id);

/* The columns Cook reads from live state at match time, written in place on live pending rows:
 * allowed (job-allowed-to-start?), plugin_accept (the launch-filter plugin) and reserved_host (the
 * rebalancer's reservation map); a NULL column is left unchanged.  Unlike an upsert, a patch keeps the
 * row's live flag and generation: the job keeps its place in the last rank's queue, and the next
 * cook_state_match and cook_state_rebalance read the new values.  clear_reservations != 0 first sets
 * reserved_host = -1 on every live row that holds one, then writes the batch: reserve-hosts! replacing the
 * whole map.  Priority is not patchable: the order changes only at the next rank (an upsert, as before).
 * COOK_E_BADARG, before any change: n < 0; a NULL job_id while n > 0; a job id that is not live or appears
 * twice; a reserved_host below -1.
 * Uploads exactly: when n > 0 and some column is given, n * (4 + [allowed] 1 + [plugin_accept] 1 +
 * [reserved_host] 4) bytes (a slot per row plus each non-NULL column); when clearing, 4 bytes per live row
 * that held a reservation.  Statistics: cook_last_stats(COOK_PHASE_STATE).                              */
int32_t cook_state_patch(cook_pool* pool, int32_t n, const int64_t* job_id, const uint8_t* allowed,
                         const uint8_t* plugin_accept, const int32_t* reserved_host, int32_t clear_reservations);

/* cook_rank over the live rows (running = live running tasks, pending = live pending jobs).  The ranked
 * queue stays on the device as the handle's resident queue; out_ranked_job_id[<= #pending] (may be
 * NULL) receives it as job ids, *out_n its length.  Rank is a total order on (user, -priority, start,
 * task id, job id) over unique ids, so the result does not depend on where rows are stored.  Uploads
 * only the user table's rank columns; cook_last_stats(COOK_PHASE_RANK) as after cook_rank.          */
int32_t cook_state_rank(cook_pool* pool, const cook_user_table* users, const cook_pool_quota* pool_quota,
                        const cook_pool_quota* group_quota, const double* group_usage,
                        const cook_rank_params* params, int64_t* out_ranked_job_id, int32_t* out_n);

/* cook_state_rank plus the jobs filter-offensive-jobs (scheduler.clj:2198-2229) puts on offensive-jobs-ch: the jobs
 * that survived the rank's quota filters (limit-over-quota, pool and group quota) and are offensive (mem >
 * offensive_max_mem_mb or cpus > offensive_max_cpus), in rank order, as job ids in
 * out_offensive_job_id[*out_n_offensive].  Empty when params->filter_offensive is 0; a job a quota cut first is not
 * listed.  The queue, out_ranked_job_id and *out_n are bit-identical to cook_state_rank's.  COOK_E_BADARG, before
 * any device work: every case cook_state_rank rejects, a NULL out_offensive_job_id or out_n_offensive, and
 * offensive_cap < the number of live pending rows.  Transfers: cook_state_rank's, plus 4 bytes (the count, when a
 * row is live) and 8 per offensive job down.  Statistics: cook_last_stats(COOK_PHASE_RANK).                     */
int32_t cook_state_rank_offensive(cook_pool* pool, const cook_user_table* users, const cook_pool_quota* pool_quota,
                                  const cook_pool_quota* group_quota, const double* group_usage,
                                  const cook_rank_params* params, int64_t* out_ranked_job_id, int32_t* out_n,
                                  int64_t* out_offensive_job_id, int32_t offensive_cap, int32_t* out_n_offensive);

/* cook_match with ranked_idx = the resident queue minus every job removed or replaced since that
 * cook_state_rank, reading the rows' current columns (what cook_state_patch wrote since the rank counts).
 * Outputs as cook_match, with the job id of the k-th considerable job in out_considerable_job_id[k];
 * afterwards cook_match_failures and cook_exchange_usage(_batch) work on this round, their k being
 * positions in out_considerable_job_id.  Uploads only the offers, the users' match columns and the
 * groups.  COOK_E_BADARG before any cook_state_rank and with params->reuse_resident set;
 * COOK_E_TOO_LARGE exactly as cook_match.  stats->ms_h2d covers the upload and the gathering of the
 * queue's rows into the matcher's columns.                                                        */
int32_t cook_state_match(cook_pool* pool, const cook_offers_soa* offers, const cook_groups* groups,
                         const cook_user_table* users, const cook_pool_quota* pool_quota,
                         const cook_match_params* params, int64_t* out_considerable_job_id,
                         int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                         uint8_t* out_fail_reason, cook_match_stats* out_stats);

/* cook_rebalance over the resident rows, as rebalancer.clj reads them: init-state (:222-266) takes every
 * live running task on its host, and jobs-to-make-room-for (:588-590) the first max_preemption jobs of the
 * last cook_state_rank's queue that are still live, still hold their generation (not removed or replaced
 * since the rank) and are allowed to start, in queue order.  A running row's host is the index in `hosts`
 * whose hostname_id equals the row's running_hostname_id.
 * Outputs as cook_rebalance, except: pending_idx is the job's position among the jobs the walk took and
 * out_decision_job_id[d] its job id; victims are task ids in out_victim_task_id (a synthetic victim, the
 * task of the job an earlier decision e of the same walk placed, as -1 - e).  Capacity:
 * out_decisions[max_preemption], out_decision_job_id[max_preemption], out_victim_task_id[victim_cap].
 * Changes nothing resident: the caller applies the decisions through deltas, as transact-preemption! does.
 * COOK_E_BADARG, before any device work and with the handle unchanged: no cook_state_rank yet, a null
 * required argument, victim_cap < live running rows + max_preemption, a live running row whose hostname is
 * -1 or a code no entry of `hosts` carries, a hostname_id twice (or negative) in `hosts`, a resident user
 * code >= n_users, a pending group code >= n_groups, a pending attribute column >= max(1, n_attr_cols).
 * COOK_E_UNSUPPORTED_CONSTRAINT in GPU DRU mode.  COOK_OK with *out_n = 0 where cook_rebalance returns
 * early: max_preemption <= 0, hosts->n == 0, no job taken.  Uploads only the host table, the users'
 * rebalance columns and the groups; cook_last_stats(COOK_PHASE_REBALANCE), ms_device including the gathers. */
int32_t cook_state_rebalance(cook_pool* pool, const cook_host_table* hosts, const cook_groups* groups,
                             const cook_user_table* users, const cook_rebalance_params* params,
                             cook_decision* out_decisions, int64_t* out_decision_job_id,
                             int64_t* out_victim_task_id, int32_t victim_cap, int32_t* out_n);

/* Running usage read from the live running rows (generate-user-usage-map scheduler.clj:711-727,
 * task-ents->usage :2118-2123, Fenzo's tracker state per host :877-881).  Every output may be NULL.
 *   out_user_usage[4][n_users]  rows count, cpus, mem, gpus: pass out, out+n_users, ... straight
 *                               into cook_user_table.usage_*; users without a live row get 0
 *   out_pool_usage[4]           count, cpus, mem, gpus over every live running row: one pool's entry
 *                               of aggregate-quota-groups, i.e. one term of cook_state_rank's group_usage
 *   hostname_id[n_hosts]        codes of the global hostname dictionary, e.g. offers->hostname_id
 *   out_run_cpus/_mem/_count[n_hosts]  sums over the live running rows whose running_hostname_id is
 *                               hostname_id[h]: cook_offers_soa.run_* for that offer table.  A row whose
 *                               host is -1 or not listed counts for its user and the pool only; a listed
 *                               host without rows gets 0.
 * Fold order: each sum is a left fold in ascending task id (DESIGN.md §2); count is the number of rows
 * as a double, and a row without gpus adds 0.0.  The result does not depend on where rows are stored.
 * Changes nothing resident; needs no cook_state_rank.  COOK_E_BADARG before any device work: n_users
 * <= a live running row's user code (when out_user_usage is given), n_hosts < 0, a NULL hostname_id
 * with n_hosts > 0, or a hostname_id that is negative or appears twice.  Uploads exactly 4 * n_hosts
 * bytes (nothing when no running row is live: every output is then 0 without device work).
 * Statistics: cook_last_stats(COOK_PHASE_USAGE).                                                     */
int32_t cook_state_usage(cook_pool* pool, int32_t n_users, double* out_user_usage, double* out_pool_usage,
                         int32_t n_hosts, const int32_t* hostname_id, double* out_run_cpus,
                         double* out_run_mem, int32_t* out_run_count);

/* Each group's running cotasks, read from the live running rows: the lists cook_groups.cot_* takes, for
 * cook_state_match and cook_state_rebalance.  A group's cotasks are the running instances of its jobs
 * (group->running-task-set, group.clj:47-57) that Fenzo's tracker knows, i.e. that are assigned to a host
 * (get-cotasks-from-tracker-state, constraints.clj:539-552).
 *   Entries     one per (live running row, group in its running_group_idx list) whose running_hostname_id is
 *               not -1.
 *   Order       grouped by group code; within a group, ascending task id (DESIGN.md §2).
 *               out_cot_off[n_groups + 1] is the CSR over groups; a group without entries has an empty range.
 *   Values      out_cot_hostname_id[k]: the row's running_hostname_id.  out_cot_attr_val[k]:
 *               hosts->attr[attr_col[g]][h], h the index in `hosts` whose hostname_id is the row's host; 0 (nil)
 *               when that host is not listed, when hosts is NULL, or when attr_col is NULL or attr_col[g] == -1.
 *               An unlisted host keeps its entry and hostname code, so unique groups still see it.  Only n,
 *               hostname_id, n_attr_cols and attr of `hosts` are read: for a match, point them at the offer
 *               table's columns; for a rebalance, pass the host table given to cook_state_rebalance.
 * Size query: with out_cot_hostname_id NULL only *out_n is written, the required capacity (known on the host,
 * no device work).  Otherwise *out_n receives the number of entries and the capacity of the two value outputs is
 * cap.
 * COOK_E_BADARG, before any device work and with nothing written: a NULL out_n, or (not a size query) a NULL
 * out_cot_off or out_cot_attr_val; n_groups < 0 or <= a live running row's group code; cap < the required size
 * (not a size query); attr_col[g] outside [-1, hosts->n_attr_cols) (read only when hosts is given); hosts->n < 0,
 * a NULL hostname_id with hosts->n > 0, a hostname_id that is negative or appears twice; a NULL hosts->attr when
 * some group names a column and hosts->n > 0.
 * No state, or no live running row with a known host and a group: every offset is 0, *out_n = 0, no device work.
 * Transfers exactly: up 4 * hosts->n (the hostname codes) + 4 * hosts->n per distinct column the groups name
 * + 4 * n_groups; down 4 * (n_groups + 1) + 8 * *out_n.  Nothing proportional to the running table moves, and
 * nothing when there is no device work.  Changes nothing resident; needs no cook_state_rank.
 * Statistics: cook_last_stats(COOK_PHASE_COTASKS).                                                          */
int32_t cook_state_cotasks(cook_pool* pool, int32_t n_groups, const int32_t* attr_col, const cook_host_table* hosts,
                           int32_t cap, int32_t* out_cot_off, int32_t* out_cot_hostname_id, int32_t* out_cot_attr_val,
                           int32_t* out_n);

/* cook_state_match with its running-side inputs read from the live running rows as they are at the call, on the
 * device, without a round trip: the resident match cycle in one call.  These fields are not read (may be NULL):
 *   users->usage_count/_cpus/_mem/_gpus   = what cook_state_usage(n_users, ...) returns now
 *   offers->run_cpus/_mem/_count          = what cook_state_usage(..., offers->n, offers->hostname_id, ...) returns
 *   groups->cot_off/_hostname_id/_attr_val (when groups has groups) = what cook_state_cotasks(groups->n_groups,
 *                                           groups->attr_col, <the offers' n, hostname_id, n_attr_cols, attr>, ...)
 *                                           returns now
 * Every other input is read as cook_state_match reads it, and the outputs are bit-identical to cook_state_match fed
 * by those calls (same kernels, same fold orders), fail reasons and ports included; cook_match_failures and
 * cook_exchange_usage(_batch) work on the round as after cook_state_match.  Edges: no live running row gives zero
 * sums and empty lists without a derivation kernel; no live queue row returns as cook_state_match does.
 * COOK_E_BADARG, before the build, with nothing written and the handle unchanged: every case cook_state_match
 * rejects except NULL cot_* lists; a live running row's user code >= n_users; and, when a queue row is left to
 * match, a NULL offers->hostname_id with offers->n > 0, an offers->hostname_id that is negative or appears twice,
 * and (groups with groups) a live running row's group code >= n_groups, an attr_col outside [-1, n_attr_cols) or
 * a NULL offers->attr while some group names a column and offers->n > 0.
 * Transfers exactly: up = the equivalent cook_state_match's upload minus 32 * n_users (usage), minus 20 *
 * offers->n (run columns), minus 4 * (n_groups + 1) + 8 * max(1, entries) (the lists, when a pending row has a
 * group list); nothing is added.  Down = cook_state_match's.  The derivation counts into COOK_PHASE_MATCH and
 * stats->ms_h2d with the queue gathers; COOK_PHASE_USAGE and COOK_PHASE_COTASKS are left as they were.        */
int32_t cook_state_match_derived(cook_pool* pool, const cook_offers_soa* offers, const cook_groups* groups,
                                 const cook_user_table* users, const cook_pool_quota* pool_quota,
                                 const cook_match_params* params, int64_t* out_considerable_job_id,
                                 int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                                 uint8_t* out_fail_reason, cook_match_stats* out_stats);

/* cook_state_rebalance with groups->cot_off/_hostname_id/_attr_val (not read, may be NULL) derived on the device
 * from the live running rows over `hosts`: what cook_state_cotasks(groups->n_groups, groups->attr_col, hosts, ...)
 * returns now.  Outputs bit-identical to cook_state_rebalance fed by that call.  COOK_E_BADARG, before any device
 * work with nothing written: every case cook_state_rebalance rejects except NULL cot_* lists; and (groups with
 * groups) a live running row's group code >= n_groups, an attr_col outside [-1, hosts->n_attr_cols) or a NULL
 * hosts->attr while some group names a column.  COOK_E_UNSUPPORTED_CONSTRAINT in GPU DRU mode.  Upload =
 * cook_state_rebalance's minus 4 * (n_groups + 1) + 8 * max(1, entries) when a pending row has a group list; the
 * derivation counts into COOK_PHASE_REBALANCE with the gathers.                                                */
int32_t cook_state_rebalance_derived(cook_pool* pool, const cook_host_table* hosts, const cook_groups* groups,
                                     const cook_user_table* users, const cook_rebalance_params* params,
                                     cook_decision* out_decisions, int64_t* out_decision_job_id,
                                     int64_t* out_victim_task_id, int32_t victim_cap, int32_t* out_n);

/* M0 over the resident queue without a match: pending-jobs->considerable-jobs (scheduler.clj:729-762; the jobs
 * handle-kubernetes-scheduler-pool :1749-1800 launches) or, with quota_only, filter-pending-jobs-for-quota
 * (tools.clj:961-973; what handle-resource-offers-autoscaling-helper :1283-1335 takes).
 *   Queue    the queue cook_state_match reads: the last cook_state_rank's, minus every entry whose slot was removed or
 *            replaced since, and minus the entries an earlier consuming call took.  Each row's current allowed and
 *            plugin_accept are read (cook_state_patch counts).
 *   Result   out_job_id[*out_n] (room for num_considerable) in take order: bit-identical to the considerable set of
 *            cook_match on host tables holding the same rows, in queue order, with an empty offer table (quota_only:
 *            allowed and plugin_accept all ones).  Folds as there: per user a left fold in queue order, the pool
 *            quota over users 0 .. n_users - 1 of the selected usage.  Does not depend on slot layout.
 *   Usage    usage_source: COOK_USAGE_GIVEN reads users->usage_*; COOK_USAGE_DERIVED folds them on the device from
 *            the live running rows (what cook_state_usage(n_users, ...) returns now; usage_* not read);
 *            COOK_USAGE_LAST_MATCH takes the [4][n_users] usage the last cook_match / cook_state_match(_derived) on
 *            this handle read (usage_* not read): the cycle-start usage the autoscaling helper reuses after the
 *            match's launches.
 *   Consume  consume != 0: the returned entries leave the queue until the next cook_state_rank, which brings back
 *            those still pending; their rows stay live and unchanged (counts, usage, cotasks, cook_state_launch).
 * Reads users' quota_* (and tokens when enforcing) always.  Builds no match plan: cook_match_failures,
 * cook_exchange_usage(_batch) and COOK_USAGE_LAST_MATCH still refer to the last match.
 * COOK_E_BADARG, before any device work with the queue unchanged and nothing written: no cook_state_rank yet; a NULL
 * users, params, out_job_id, out_n or quota_* column (usage_* too for GIVEN); a live pending row's user code >=
 * n_users (and a live running row's for DERIVED); LAST_MATCH with no match on the handle or one with another
 * n_users; an unknown usage_source.  num_considerable <= 0 or an empty queue: *out_n = 0 without device work.
 * Transfers exactly: up 32 * n_users (quotas) + 4 * n_users (tokens, when enforcing and given) + 32 * n_users (usage,
 * GIVEN only); down 4 (the live queue's length) and, when that is not 0, 4 (*out_n) + 8 * *out_n.
 * Statistics: cook_last_stats(COOK_PHASE_CONSIDERABLE); all zero after a call without device work.            */
enum { COOK_USAGE_GIVEN = 0, COOK_USAGE_DERIVED = 1, COOK_USAGE_LAST_MATCH = 2 };
typedef struct {
  int32_t num_considerable;   /* take N; <= 0 => *out_n = 0, no device work                                        */
  int32_t enforce_rate_limit; /* as cook_match_params                                                              */
  int32_t quota_only;         /* 1: filter-pending-jobs-for-quota only (autoscaling): allowed and plugin_accept are
                                 not read.  0: pending-jobs->considerable-jobs                                       */
  int32_t usage_source;       /* COOK_USAGE_*: where users->usage_* come from                                      */
  int32_t consume;            /* 1: the returned jobs leave the resident queue until the next cook_state_rank
                                 (handle-kubernetes-scheduler-pool)                                                */
} cook_considerable_params;
int32_t cook_state_considerable(cook_pool* pool, const cook_user_table* users, const cook_pool_quota* pool_quota,
                                const cook_considerable_params* params, int64_t* out_job_id, int32_t* out_n);

/* ------------------------------------------------------------ phase timing */
/* Device-side timing of the last call of each kind on this handle (CUDA events on the
 * pool's stream): what bench.py's `phases` block and roofline lines are computed from.
 * COOK_PHASE_STATE: the last cook_state_apply, cook_state_launch or cook_state_patch (upload, then the
 * scatter / move / compaction kernels).  COOK_PHASE_USAGE: the last cook_state_usage (upload of the
 * hostname list, the compaction, sorts and folds, the download of the sums).  COOK_PHASE_COTASKS: the last
 * cook_state_cotasks (upload of the host codes, attribute columns and group map, the compaction, expansion and
 * sort, the download of the lists; all zero after a call without device work).  COOK_PHASE_CONSIDERABLE: the last
 * cook_state_considerable (upload of the user columns, the queue compaction and gathers, the usage fold when derived,
 * the considerable pass and the consumption, the download of the ids). */
enum { COOK_PHASE_RANK = 0, COOK_PHASE_MATCH = 1, COOK_PHASE_REBALANCE = 2, COOK_PHASE_EXCHANGE = 3,
       COOK_PHASE_STATE = 4, COOK_PHASE_USAGE = 5, COOK_PHASE_COTASKS = 6, COOK_PHASE_CONSIDERABLE = 7 };
typedef struct {
  double ms_h2d;      /* upload stage                                              */
  double ms_device;   /* kernels (for the exchange: delta kernels + the collective) */
  double ms_d2h;      /* result download                                           */
  int64_t h2d_bytes;
  int64_t d2h_bytes;
  int32_t n_launches;
  int32_t reserved0;
} cook_phase_stats;
int32_t cook_last_stats(cook_pool* pool, int32_t phase, cook_phase_stats* out);

/* ----------------------------------------------------------------- multi-GPU */
/* §8e: after a pool's match round every rank contributes its pools' usage
 * deltas {count,cpus,mem,gpus} per user; one ncclAllGather over NVLink makes
 * all ranks consistent (reference analogue: reading one Datomic snapshot,
 * scheduler.clj:2125-2157).  `comm` is an ncclComm_t created by the host
 * (torch.distributed or ncclCommInitRank); `stream` a cudaStream_t (0 ok).
 * local/out are DEVICE pointers: local[n_doubles], out[world*n_doubles].    */
int32_t cook_allgather_usage(void* nccl_comm, void* stream, const double* local_dev,
                             double* out_dev, int64_t n_doubles);

/* Communicator plumbing for hosts without their own NCCL binding (the JVM): rank 0 calls
 * cook_comm_unique_id, ships the 128 bytes to every rank over its own control plane (Cook:
 * ZooKeeper / the leader's REST endpoint; bench.py: torch.distributed broadcast), every rank
 * calls cook_comm_init (ncclCommInitRank on `device`).                                      */
int32_t cook_comm_unique_id(uint8_t out_id[128]);
int32_t cook_comm_init(const uint8_t id[128], int32_t rank, int32_t world, int32_t device,
                       void** out_comm);
int32_t cook_comm_destroy(void* comm);

/* The exchange step as one call.  Computes, ON THE DEVICE, the per-user usage delta
 * {count,cpus,mem,gpus} of the jobs the last cook_match on this handle placed (left fold per
 * user in queue order: same association as generate-user-usage-map scheduler.clj:711-727
 * would produce for those tasks), then all-gathers it over `comm` on the pool's stream and
 * copies the result to the host:
 *   out_all[world][n_pad]   n_pad >= 4 * n_users doubles per rank ([user][4], zero padded)
 * A handle that has not matched yet contributes zeros.  world == 1 (or comm == NULL) skips
 * the collective.  Every rank must call it the same number of times with the same n_pad.   */
int32_t cook_exchange_usage(cook_pool* pool, void* comm, int32_t world, int32_t n_pad,
                            double* out_all);

/* The same for ALL the pools a rank ran in the cycle, with ONE all-gather per cycle instead of one
 * per pool: pools placed on GPUs by LPT balance the SUM of a rank's pools, a collective per pool
 * slot would make every slot as long as its slowest rank.  pools[i] fills slot i, slots
 * n_pools .. n_slots-1 stay zero (ranks own different numbers of pools; n_slots is the same on
 * every rank).  out_all[world][n_slots][n_pad].  The result feeds the NEXT cycle's cook_rank
 * (group_usage), as aggregate-quota-groups scheduler.clj:2125-2132 does per cycle.  The handles
 * of one call live on one device and are idle (their cook_match calls have returned).       */
int32_t cook_exchange_usage_batch(cook_pool* const* pools, int32_t n_pools, void* comm, int32_t world,
                                  int32_t n_pad, int32_t n_slots, double* out_all);

#ifdef __cplusplus
}
#endif
#endif /* COOK_GPU_H */
