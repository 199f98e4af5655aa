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
 * priority, job id, cpus, mem, gpus and the list facts (cook_state_list_facts) are copied on the device from the
 * pending row.  Leaves exactly the
 * state cook_state_apply leaves after the batch pending_rm_job_id = job_id plus the running upserts built
 * from those rows with running_hostname_id = hostname_id and, as running_group_off / running_group_idx, the
 * pending rows' group lists: the job leaves the last rank's queue, its counts and reservation leave with the
 * row, its group list moves to the task (copied on the device, in launch order) while its other list
 * entries leave, and the list arenas compact by the same rule.  A job with retry facts (cook_state_retry_facts)
 * parks its pending slot instead: the same state for every reader, but the slot keeps its columns and lists for
 * cook_state_status and stays off the free list; the compaction keeps its entries (one more launch while some slot
 * is parked).
 * COOK_E_BADARG, before any change: n < 0; a NULL job_id, task_id or start_time while n > 0; a job id that
 * is not live or appears twice; a task id that appears twice or is already live; a hostname code below -1.
 * Uploads exactly n * (4 + 4 + 8 + 8) bytes (pending slot, running slot, task id, start time), plus 4 * n
 * when hostname_id is not NULL, plus 4 * n when some job of the batch parks (the parked and the freed slots).
 * Statistics: cook_last_stats(COOK_PHASE_STATE).                                                        */
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
 * task id, job id) over unique ids, and the pool quota's start value (the pool's running usage) is the
 * live running rows folded in ascending task id, equal to cook_state_usage's pool total bit for bit, so
 * the result does not depend on where rows are stored.  Uploads only the user table's rank columns;
 * cook_last_stats(COOK_PHASE_RANK) as after cook_rank.                                             */
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

/* The live offers: Fenzo's leases (scheduler.clj:617-687, :2301-2324), kept on the device between match cycles.
 * cook_state_offers_add takes one row per offer as it arrives, not merged: offers->n rows of hostname_id, cpus, mem,
 * the port CSR, is_k8s, location, the gpu and disk maps, max_tasks, num_tasks, host_start_time and n_attr_cols / attr
 * (columns past a row's n_attr_cols are absent, 0); name_rank, run_* and reserved are not read.  A NULL column takes
 * its absent value (is_k8s 0, location -1, max_tasks -1, num_tasks 0, host_start_time -1, empty lists).
 * offer_id[n] names each offer; single_shot[n] (NULL: none) marks offers that never outlive a match attempt
 * (Kubernetes, :674-678); offer_gpus[n] is the lease's "gpus" scalar (NULL: 0).  hostname / hostname_off[n + 1]: each
 * row's hostname bytes as a CSR (NULL hostname_off: all empty); a row may give an empty name when the handle already
 * knows its code.  Every row is stamped received = now_ms and takes the next arrival number (calls in sequence,
 * rows in order).
 * COOK_E_BADARG with nothing changed: an offer id that is live or twice in the batch, a negative code, a new code
 * without a name, a code whose name differs from the one the handle holds, two codes with one name, a malformed CSR.
 * cook_state_apply with reset drops the live offers (the names stay known).  Uploads: the non-NULL columns, the
 * lists with their offsets, 8 bytes (arrival number) plus 4 (slot) per row, and the attribute rows as one more list
 * (4 * n_attr_cols values and 4 bytes of offset per row); statistics: cook_last_stats(COOK_PHASE_STATE). */
int32_t cook_state_offers_add(cook_pool* pool, const cook_offers_soa* offers, const int64_t* offer_id,
                              const uint8_t* single_shot, const double* offer_gpus, const char* hostname,
                              const int32_t* hostname_off, int64_t now_ms);

/* One Fenzo scheduleOnce over the resident queue and the live offers, in four steps:
 *   (a) expiry       offers with now_ms - received >= incubate_ms leave, fate COOK_OFFER_EXPIRED.  The boundary is
 *                    this library's rule (Fenzo's own is not in the reference); a shim converts
 *                    offer-incubate-time-ms as max(seconds, 1) * 1000.
 *   (b) merge        one VM per hostname with a live offer, VMs in memcmp order of the hostname bytes (the equal
 *                    fitness tie-break).  cpus and mem are left folds over the host's offers in arrival order, port
 *                    ranges concatenated in arrival order, every other column from the host's newest offer.  The
 *                    attribute matrix is as wide as the widest live offer row, the largest column a pending row
 *                    names and the largest group attr_col, whichever is largest.  reserved marks the hosts some
 *                    live pending row has as reserved_host (present when some row has one).  is_k8s, max_tasks and
 *                    the gpu and disk maps are present when some VM's value is not absent, the port lists when some
 *                    live offer has a range; location, num_tasks and host_start_time always.
 *   (c) match        cook_state_match_derived over that table; out_assign_hostname_id gets the VM's hostname code
 *                    or -1.  cook_match_failures, cook_exchange_usage(_batch) and COOK_USAGE_LAST_MATCH then refer
 *                    to this round.
 *   (d) consumption  every offer of a host with an assignment leaves, fate COOK_OFFER_USED; every remaining
 *                    single-shot offer leaves, fate COOK_OFFER_SINGLE_SHOT.
 * (a) and (d) also run when no queue row is left.  out_gone_offer_id / out_gone_fate [*out_n_gone]: the offers that
 * left, in arrival order; gone_cap must be at least the live offers before the call.  An error returned after the
 * expiry still writes the offers that had left by then.
 * COOK_E_BADARG before any device work or offer change: every case of cook_state_match_derived, incubate_ms <= 0,
 * gone_cap too small, a NULL gone output, params->reuse_resident.
 * Transfers: up = cook_state_match_derived's over the merged table, without that table's columns, plus 4 bytes per VM
 * (its hostname code), 4 per reserved pending row (when the table has reserved) and 4 per offer that left; down =
 * cook_state_match_derived's.  Statistics: stats and cook_last_stats(COOK_PHASE_MATCH). */
enum { COOK_OFFER_USED = 1, COOK_OFFER_EXPIRED = 2, COOK_OFFER_SINGLE_SHOT = 3 };
int32_t cook_state_match_offers(cook_pool* pool, int64_t now_ms, int64_t incubate_ms, const cook_groups* groups,
                                const cook_user_table* users, const cook_pool_quota* pool_quota,
                                const cook_match_params* params, int64_t* out_considerable_job_id,
                                int32_t* out_assign_hostname_id, int32_t* out_ports, int32_t max_ports,
                                uint8_t* out_fail_reason, int64_t* out_gone_offer_id, uint8_t* out_gone_fate,
                                int32_t gone_cap, int32_t* out_n_gone, cook_match_stats* out_stats);

/* cook_state_rebalance_derived with hosts->has_spare / spare_cpus / spare_mem / spare_gpus (not read, may be NULL)
 * derived from the live offers as view-incubating-offers (scheduler.clj:1537-1546) gives them: has_spare is set for a
 * host with at least one live offer, and the spare values are left folds in arrival order of its offers' cpus, mem
 * and offer_gpus.  Nothing expires here (getVmCurrentStates does not expire either); the attributes still come from
 * the caller's table (the agent-attributes cache).
 * COOK_E_BADARG, before any device work: every case of cook_state_rebalance_derived, and a host with a live offer
 * that is not in `hosts`.  Transfers: cook_state_rebalance_derived's minus 25 bytes per host (the spare columns).
 * Statistics: cook_last_stats(COOK_PHASE_REBALANCE). */
int32_t cook_state_rebalance_offers(cook_pool* pool, const cook_host_table* hosts, const cook_groups* groups,
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

/* ---------------------------------------------------------- auditing a resident pool */
/* The read side of the resident state: a fingerprint a host can restate from its own source of truth (the
 * database the deltas came from), a bucketed form of it that localises a difference, the rows themselves in a
 * form cook_state_apply takes back, and the live queue.  None of these calls changes anything resident, needs a
 * cook_state_rank (the queue parts report empty) or touches the queue or the last match: cook_state_match,
 * cook_match_failures, cook_exchange_usage(_batch) and COOK_USAGE_LAST_MATCH behave after them as before.
 *
 * Row hash (64 bit; all arithmetic mod 2^64):
 *   mix(z)       = the splitmix64 finaliser: z ^= z >> 30; z *= 0xbf58476d1ce4e5b9; z ^= z >> 27;
 *                  z *= 0x94d049bb133111eb; z ^= z >> 31
 *   absorb(h, w) = mix((h ^ w) + 0x9e3779b97f4a7c15)
 *   A row starts from its table's tag (1 pending, 2 running), absorbs its id (job id / task id), then every data
 *   column as one 64-bit word each (int32 sign-extended, uint8 zero-extended, a double by its bit pattern as
 *   stored, so -0.0 differs from 0.0; a column the delta left NULL by its documented absent value), then each
 *   list: its length, then its entries in order (attribute-equals: column, then value; each sign-extended).
 *     pending: user, priority, cpus, mem, gpus, ports, allowed, plugin_accept, gpu_model, disk_request, disk_type,
 *              est_end_ms, ckpt_location, reserved_host; lists novel_host, (attr_col, attr_val), group_idx
 *     running: user, priority, start_time, job_id, cpus, mem, gpus, running_hostname_id; list running_group_idx
 *   Where a row is stored (slot, generation, list offsets) is layout and is not hashed.
 * Set fingerprint: sum = the sum of the row hashes, xr = their xor, n = their number.  Both are commutative, so
 *   the result does not depend on slot or arena layout, grid size or the order of atomics.
 * Queue fingerprint: over the entries cook_state_match would read now, p the position among them:
 *   row hash = absorb(absorb(3, p), job id).  Zero with n = 0 before any cook_state_rank.
 * Buckets: n_buckets is 0 or a power of two up to 65536; bucket(id) = mix(id) & (n_buckets - 1).               */
typedef struct { uint64_t sum, xr; int64_t n; } cook_fp;

/* What the host side of the state mirrors of the device rows, recounted from them by cook_state_digest: live rows
 * per table, live entries per list arena (+ 0 novel hosts, 1 attribute-equals, 2 pending groups, 3 running
 * groups), pending rows holding a non-absent value per kind (+ 0 gpus, 1 ports, 2 not allowed, 3 not
 * plugin-accepted, 4 gpu_model, 5 disk_request, 6 est_end_ms, 7 ckpt_location, 8 reserved_host), the reserved
 * rows, the running rows with a known host and a group list and their entries, and the largest code per kind
 * (-1: none).  first_mismatch is one of these.                                                                 */
enum {
  COOK_AUDIT_PENDING_ROWS = 0, COOK_AUDIT_RUNNING_ROWS = 1, COOK_AUDIT_ENTRIES = 2, COOK_AUDIT_FLAGS = 6,
  COOK_AUDIT_RESERVED_ROWS = 15, COOK_AUDIT_COT_ROWS = 16, COOK_AUDIT_COT_ENTRIES = 17,
  COOK_AUDIT_MAX_USER_PENDING = 18, COOK_AUDIT_MAX_USER_RUNNING = 19, COOK_AUDIT_MAX_GROUP_PENDING = 20,
  COOK_AUDIT_MAX_GROUP_RUNNING = 21, COOK_AUDIT_MAX_ATTR_COL = 22, COOK_AUDIT_MAX_HOSTNAME_RUNNING = 23,
  COOK_AUDIT_N = 24
};
typedef struct {
  cook_fp pending, running;   /* the live rows of each table                                               */
  cook_fp queue;              /* the live queue, order-sensitive                                           */
  int64_t entries[4];         /* live list entries: novel hosts, attribute-equals, pending groups, running groups */
  int32_t consistent;         /* 1: every host-side count equals its recount from the device rows          */
  int32_t first_mismatch;     /* the first COOK_AUDIT_* count that differed, -1 when consistent            */
} cook_state_digest_out;

/* Fingerprints and recount in one pass per table.  out_pending_bucket / out_running_bucket [n_buckets] receive the
 * fingerprint of each table's rows per bucket (their sums, xors and counts add up to the table's); both are
 * required when n_buckets > 0.
 * COOK_E_BADARG, before any device work with nothing written: a NULL out; n_buckets negative, not a power of two
 * or above 65536; n_buckets > 0 with a NULL bucket output, or a bucket output with n_buckets == 0.
 * No state, or no live row in either table: all zero, consistent = 1, no device work.
 * Transfers exactly: up nothing; down 72 (the three fingerprints) + 8 * COOK_AUDIT_N (the recount) + 2 * 24 *
 * n_buckets.  Statistics: cook_last_stats(COOK_PHASE_AUDIT).                                                   */
int32_t cook_state_digest(cook_pool* pool, int32_t n_buckets, cook_state_digest_out* out,
                          cook_fp* out_pending_bucket, cook_fp* out_running_bucket);

/* The comparison cook_state_digest makes after its download: *out_first = the first index k < COOK_AUDIT_N with
 * host[k] != device[k], or -1.  A pure host function.  COOK_E_BADARG on a NULL argument.                        */
int32_t cook_state_counts_compare(const int64_t* host, const int64_t* device, int32_t* out_first);

/* The rows as a delta: cook_state_delta's columns with writable pointers.  A NULL column is skipped; a list is
 * written when its offsets column is given, and then needs its value column(s).                                 */
typedef struct {
  int32_t* user; double* cpus; double* mem; double* gpus; int32_t* ports; uint8_t* allowed; uint8_t* plugin_accept;
  int32_t* novel_off; int32_t* novel_host; int32_t* gpu_model; double* disk_request; int32_t* disk_type;
  int32_t* attr_off; int32_t* attr_col; int32_t* attr_val; int64_t* est_end_ms; int32_t* ckpt_location;
  int32_t* reserved_host; int32_t* group_off; int32_t* group_idx;
} cook_jobs_rows;
typedef struct {
  int32_t* user; int32_t* priority; int64_t* start_time; int64_t* task_id; int64_t* job_id;
  double* cpus; double* mem; double* gpus;
} cook_tasks_rows;
typedef struct {
  cook_jobs_rows pending;
  int32_t* pending_priority;
  int64_t* pending_job_id;
  cook_tasks_rows running;
  int32_t* running_hostname_id;
  int32_t* running_group_off;
  int32_t* running_group_idx;
} cook_state_rows;
typedef struct {
  int32_t pending, running;   /* rows per table                                                             */
  int32_t entries[4];         /* entries per list: novel hosts, attribute-equals, pending groups, running groups */
} cook_state_sizes;

/* Every live row or, with bucket_mask[n_buckets], those whose bucket b has bucket_mask[b] != 0: pending rows in
 * ascending job id, running rows in ascending task id, the lists rebuilt as CSR over that order ([rows + 1]
 * offsets).  *out_n receives the rows and entries; `cap` is the capacity of the columns of `out`.
 * Round trip: the arrays, passed as one cook_state_delta with reset = 1 to a fresh handle, give a state with the
 * same digest; without reset, to a handle that lacks or mis-holds those rows, they repair them.  Generations and
 * the queue are not exported: repaired rows leave the queue until the next rank, as after any upsert.
 * Size query: out == NULL writes only *out_n; without a mask from the host-side counts (no device work), with one
 * by the count pass.
 * COOK_E_BADARG with nothing written: a NULL out_n, or a NULL cap with out given; n_buckets as for
 * cook_state_digest; a mask with n_buckets == 0; an offsets column without its value column(s); a capacity below
 * the required size (without a mask before any device work, with one after the count pass).
 * No state, or no live row in either table: *out_n all zero, each given offsets column gets its one 0, no device
 * work.
 * Transfers exactly (when there is device work): up n_buckets bytes with a mask, else nothing; down 24 (the
 * counts) + 8 with a mask (the row counts, ahead of the sort) and, unless a size query, for each non-NULL column
 * its element size times the rows, per given list 4 * (rows + 1) for the offsets and 4 (attribute-equals 8) per
 * entry.  Statistics: cook_last_stats(COOK_PHASE_AUDIT).                                                        */
int32_t cook_state_export(cook_pool* pool, int32_t n_buckets, const uint8_t* bucket_mask,
                          const cook_state_sizes* cap, const cook_state_rows* out, cook_state_sizes* out_n);

/* The live queue now: the job ids cook_state_match would read, in order (the last cook_state_rank's queue minus
 * the launched, removed, replaced and consumed jobs).  out_job_id == NULL is a size query: only *out_n.
 * COOK_E_BADARG with nothing written: before any cook_state_rank, a NULL out_n, cap < the live entries.
 * Transfers exactly: down 4 (the length; nothing for an empty ranked queue: no device work) + 8 * *out_n unless a
 * size query.  Statistics: cook_last_stats(COOK_PHASE_AUDIT).                                                   */
int32_t cook_state_queue(cook_pool* pool, int32_t cap, int64_t* out_job_id, int32_t* out_n);

/* ------------------------------------------------------------ phase timing */
/* Device-side timing of the last call of each kind on this handle (CUDA events on the
 * pool's stream): what bench.py's `phases` block and roofline lines are computed from.
 * COOK_PHASE_STATE: the last cook_state_apply, cook_state_launch, cook_state_patch, cook_state_task_facts,
 * cook_state_task_reason, cook_state_finish, cook_state_finish_history, cook_state_history_seed,
 * cook_state_history_advance or cook_state_group_runtimes (upload, then the scatter / move / record / compaction kernels).  COOK_PHASE_USAGE: the last cook_state_usage (upload of the
 * hostname list, the compaction, sorts and folds, the download of the sums).  COOK_PHASE_COTASKS: the last
 * cook_state_cotasks (upload of the host codes, attribute columns and group map, the compaction, expansion and
 * sort, the download of the lists; all zero after a call without device work).  COOK_PHASE_CONSIDERABLE: the last
 * cook_state_considerable (upload of the user columns, the queue compaction and gathers, the usage fold when derived,
 * the considerable pass and the consumption, the download of the ids).  COOK_PHASE_AUDIT: the last
 * cook_state_digest, cook_state_export or cook_state_queue (upload of the bucket mask, the passes over the tables,
 * the compaction, sort and gathers, the download of the fingerprints, rows or ids; all zero after a call without
 * device work).  cook_state_user_stats reports through its own out_stats argument. */
enum { COOK_PHASE_RANK = 0, COOK_PHASE_MATCH = 1, COOK_PHASE_REBALANCE = 2, COOK_PHASE_EXCHANGE = 3,
       COOK_PHASE_STATE = 4, COOK_PHASE_USAGE = 5, COOK_PHASE_COTASKS = 6, COOK_PHASE_CONSIDERABLE = 7,
       COOK_PHASE_AUDIT = 8 };
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

/* ------------------------------------------------------ the monitor over resident pools */
/* The monitor's per-user stats and user counts (set-stats-counters!, monitor.clj:177-207) read from the live rows of
 * one pool or of a quota group, and the queue lengths (jobs->queue-lengths, queue_limit.clj:64-90) as the waiting
 * state of single-pool calls.
 *   Rows     the union of the live rows of pools[0, n_pools): one handle gives a pool's stats; the handles of the pools
 *            a quota-group name maps to give that name's (job-ent-in-pool :35-38).  The handles are idle, each call
 *            serialised with each of them by the caller, on one device or several (the gather step, DESIGN.md §9a);
 *            the work runs on pools[0]'s stream and scratch, and the answer is the bits of one device.
 *   Folds    get-job-stats (:40-57) per user, each sum a left fold in a fixed order (DESIGN.md §2): waiting over the
 *            live pending rows in ascending job id, running over the live running rows in ascending task id; an id
 *            several handles hold, in the order of pools.  jobs is the number of rows.
 *   Outputs  for each state s (COOK_STATS_*) and user code u < n_users, out_jobs / out_cpus / out_mem[s * n_users +
 *            u]; bit s of out_member[u] says whether u is in state s.  A user outside a state has zeros there.
 *     running  the user has a live running row: their running fold.
 *     waiting  the user has a live pending row: their waiting fold.
 *     starved  (waiting users, get-starved-job-stats :69-90) run_cpus < share_cpus and run_mem < share_mem, the shares
 *              being users->div_cpus / div_mem filled as share/get-shares fills them (the user's share, else the
 *              default user's, else Double/MAX_VALUE); a user with no running row has usage 0.0.  cpus = min(share -
 *              run, wait), mem likewise; jobs = min(run_jobs, wait_jobs) when the user runs, else wait_jobs: :jobs is
 *              only in the running map, so (merge-with - share running) passes it through unchanged.
 *     wuq      (waiting users, get-waiting-under-quota-job-stats :92-116) run_jobs < quota_count, run_cpus <
 *              quota_cpus, run_mem < quota_mem and quota_rest_ok[u] != 0: the caller's verdict that every other key
 *              of the user's quota map is > 0.0 (gpus always, plus the default user's :launch-rate-* for users
 *              without a quota of their own, quota.clj:82-111, 272-295); NULL means all 1.  jobs, cpus, mem =
 *              min(max(quota - run, 0), wait), quota_count an integral value.  The map's other keys pass through
 *              from the quota unchanged; they are host values and not computed here.
 *   Totals   out_all_jobs / _cpus / _mem[s]: the "all" entry of state s (add-aggregated-stats :59-67), a left fold
 *            over the state's users in ascending user code (any association only where the grid rule holds).
 *            out_users[COOK_USERS_*]: total = |running u waiting|, starved, wuq, hungry = waiting - starved,
 *            satisfied = running - waiting.
 * Changes nothing resident: no row, queue, match plan or COOK_USAGE_LAST_MATCH usage.
 * COOK_E_BADARG, before any device work and with nothing written: a NULL pools, users or out_* array; n_pools <= 0;
 * a NULL handle or a handle listed twice; n_users <= 0; a NULL div_cpus, div_mem, quota_count, quota_cpus or quota_mem;
 * a live row's user code >= n_users.  An OOM or CUDA error on another handle's device is returned on pools[0], with
 * nothing written.
 * No live row in any handle: every output zero, no device work.
 * Transfers exactly: up 40 * n_users (the five user columns) + n_users (quota_rest_ok, when given), none per device;
 * down 97 * n_users (the three [4][n_users] arrays and out_member) + 136 (the totals); 36 B a live row between devices.
 * Statistics: out_stats (may be NULL) receives the call's own cook_phase_stats: upload of the user columns, the
 * compactions, sorts and folds of both tables (launches on every device), the classification and totals, the download,
 * timed on pools[0]; all zero without device work.  No cook_last_stats slot is written: each phase reports its own.
 * Outputs are plain caller arrays, like cook_state_usage's, rather than one result struct: every struct of this
 * header has a field-for-field ctypes mirror (cook_b200/abi.py), and arrays need none.                          */
enum { COOK_STATS_RUNNING = 0, COOK_STATS_WAITING = 1, COOK_STATS_STARVED = 2, COOK_STATS_WUQ = 3 };
enum { COOK_USERS_TOTAL = 0, COOK_USERS_STARVED = 1, COOK_USERS_WUQ = 2, COOK_USERS_HUNGRY = 3,
       COOK_USERS_SATISFIED = 4, COOK_USERS_N = 5 };
int32_t cook_state_user_stats(cook_pool* const* pools, int32_t n_pools, const cook_user_table* users,
                              const uint8_t* quota_rest_ok, int64_t* out_jobs, double* out_cpus, double* out_mem,
                              uint8_t* out_member, int64_t* out_all_jobs, double* out_all_cpus, double* out_all_mem,
                              int64_t* out_users, cook_phase_stats* out_stats);

/* ------------------------------------------ the periodic killers over resident pools */
/* What the cancelled-task killer (killable-cancelled-tasks, scheduler.clj:1988-2016), the lingering-task killer
 * (get-lingering-tasks :1888-1953) and the straggler handler (handle-stragglers :1955-1986, find-stragglers
 * :quantile-deviation, group.clj:17-45) read, kept on the resident rows, and the three lists swept on the device.
 * All times are ms since the epoch, as cook_tasks_soa.start_time.
 *
 * Facts on live running rows, by task id: max_runtime_ms[i] (the job's :job/max-runtime, -1: none), cancelled[i]
 * (:instance/cancelled) and unknown[i] (status unknown rather than running); a NULL column is left unchanged.  Like
 * cook_state_patch, the row keeps its live flag and generation.  Every running upsert of cook_state_apply and every
 * cook_state_launch writes the absent facts (no max-runtime, not cancelled, running), so an upsert of a known running id
 * resets them.  The facts are not part of cook_state_digest or cook_state_export: after a resync the caller sends them
 * again.
 * COOK_E_BADARG, before any change: n < 0; a NULL task_id while n > 0; a task id that is not live or appears twice;
 * a max_runtime_ms below -1.  Uploads exactly, when n > 0 and some column is given: n * (4 + [max_runtime_ms] 8 +
 * [cancelled or unknown] 1) bytes.  Statistics: cook_last_stats(COOK_PHASE_STATE).                                */
int32_t cook_state_task_facts(cook_pool* pool, int32_t n, const int64_t* task_id, const int64_t* max_runtime_ms,
                              const uint8_t* cancelled, const uint8_t* unknown);

/* The reason fact of live running rows, by task id: reason_code[i] is the instance's :instance/reason as the caller's
 * dictionary of :reason/code values, -1 for none.  A running or unknown instance carries one only when a killer wrote
 * it before the backend confirmed the kill (:reason-killed-by-user from the cancelled-task killer, scheduler.clj:2012,
 * and from the tx-report job-completion kill, :439); :instance/update-state writes none.  Written in place like
 * cook_state_task_facts (live flag and generation kept); every running upsert of cook_state_apply and every
 * cook_state_launch writes -1.  Not part of cook_state_digest or cook_state_export: after a resync the caller sends it
 * again.  cook_state_instance_stats reads it.
 * COOK_E_BADARG, before any change: n < 0; a NULL task_id or reason_code while n > 0; a task id that is not live or
 * appears twice; a reason code below -1.  Uploads exactly 8 * n bytes (the slots and the codes).
 * Statistics: cook_last_stats(COOK_PHASE_STATE).                                                                  */
int32_t cook_state_task_reason(cook_pool* pool, int32_t n, const int64_t* task_id, const int32_t* reason_code);

/* Finished tasks by id.  Leaves exactly the state cook_state_apply with running_rm_task_id = task_id leaves for every
 * other call (rows, list arenas, counts, digest, export, queue).  In addition, each row with success[i] != 0 appends one
 * runtime record (group code, runtime_s) per entry of its group list to the handle's record table, runtime_s =
 * (end_time_ms[i] - start) / 1000 truncated (Joda's in-seconds of the interval), computed on the device from the row's
 * start time.  success NULL: no row succeeded (end_time_ms may then be NULL).  A reset through cook_state_apply drops
 * every record; cook_state_digest and cook_state_export do not cover them: after a resync the caller seeds them again
 * (cook_state_group_runtimes).
 * COOK_E_BADARG, before any change: n < 0; a NULL task_id while n > 0; success without end_time_ms; a task id that is
 * not live or appears twice; a successful row whose end is before its start (the reference's interval throws; this
 * error is ours) or whose runtime is 2^31 s or more.  COOK_E_TOO_LARGE: more than 2^31 - 1 records.
 * Uploads exactly, when n > 0: 4 * n (the slots) + 9 * n when success is given (success, end_time_ms).
 * Statistics: cook_last_stats(COOK_PHASE_STATE).                                                                  */
int32_t cook_state_finish(cook_pool* pool, int32_t n, const int64_t* task_id, const int64_t* end_time_ms,
                          const uint8_t* success);

/* ------------------------------------------------------- finished-instance history */
/* A handle's history: a device table of its finished instances, 49 B per row (task id i64, user i32, start and end
 * i64 ms, cpus and mem f64, reason code i32 with -1 for none, success u8), in arrival order.  Capacity doubles with
 * device-to-device copies; rows leave only by a stable compaction.  The history is off until seeded; while it is off,
 * no other call changes its behaviour or cost.  The handle keeps a horizon since_ms: every finished instance of this
 * pool whose start is >= since_ms is in the table, and a finishing row whose start is before it is not kept.  Not part
 * of cook_state_digest or cook_state_export; a reset through cook_state_apply empties it and turns it off.
 * cook_state_history_stats reads it.
 * Fixed choices:
 *   Horizon  on start time.  Rows with start < the horizon are neither kept nor selectable; a window before it is
 *            refused (cook_state_history_stats), never answered partially.
 *   Reason   a finished row's reason is the caller's final reason (reason_code) or, with reason_code NULL, the running
 *            row's cook_state_task_reason fact.
 *   Interval end before start is COOK_E_BADARG (the reference's interval throws; this error is ours).
 *
 * cook_state_history_seed: replaces the history with rows [0, n), sets the horizon to since_ms and turns the history
 * on (the start-up and leadership-change path: the finished instances with start >= since_ms, read once).  n = 0
 * starts an empty history at that horizon.
 * COOK_E_BADARG, before any change: n < 0; a NULL array while n > 0; a row with start < since_ms or end < start; a
 * negative user; a reason below -1; cpus or mem negative, -0.0 or not finite (the stats rely on equal values being
 * equal bits); a task id listed twice, or live in the handle's running table.
 * Uploads exactly 49 * n bytes, copied straight into the table.  Statistics: cook_last_stats(COOK_PHASE_STATE). */
int32_t cook_state_history_seed(cook_pool* pool, int64_t since_ms, int32_t n, const int64_t* task_id,
                                const int32_t* user, const int64_t* start_ms, const int64_t* end_ms, const double* cpus,
                                const double* mem, const uint8_t* success, const int32_t* reason_code);

/* Exactly cook_state_finish(pool, n, task_id, end_time_ms, success), straggler records included; in addition, while
 * the history is on, each row whose start is >= the horizon is appended to it in batch order, on the device from the
 * running row before its removal (user, start, cpus, mem), with end_time_ms[i], success[i] != 0 (1 success, 0 failed)
 * and reason_code[i] (NULL: the running row's reason fact).  The append costs O(n), not O(history).  While the
 * history is off this is cook_state_finish plus the checks below.
 * COOK_E_BADARG, before any change: everything cook_state_finish rejects; a NULL end_time_ms or success while n > 0;
 * any row, failed ones included, whose end is before its start; a reason below -1.  COOK_E_TOO_LARGE: more than
 * 2^31 - 1 records, or history rows.
 * Uploads exactly cook_state_finish's 13 * n, plus 4 * n (reason_code) when reason_code is given and a row is appended.
 * Statistics: cook_last_stats(COOK_PHASE_STATE).                                                                  */
int32_t cook_state_finish_history(cook_pool* pool, int32_t n, const int64_t* task_id, const int64_t* end_time_ms,
                                  const uint8_t* success, const int32_t* reason_code);

/* Raises the horizon to since_ms and drops the rows with start < since_ms in one stable device compaction (into new
 * columns of the same capacity, the old ones then freed).  The caller calls it periodically with now - retention; the
 * retention is the caller's configuration.
 * COOK_E_BADARG: the history is off; since_ms below the current horizon.
 * Uploads nothing; downloads 4 bytes (the rows kept) when the table holds a row and since_ms is above the horizon,
 * else nothing.  Statistics: cook_last_stats(COOK_PHASE_STATE).                                                 */
int32_t cook_state_history_advance(cook_pool* pool, int64_t since_ms);

/* ------------------------------------------------------------- retries */
/* A failed task whose job has retries left returns the job to the queue without a row re-sent: the decision of
 * :instance/update-state (scheduler/src/cook/schema.clj:1242-1300) taken per status on the host from per-job retry
 * facts, and the requeue done on the device from the job's parked pending slot.
 * Fixed choices:
 *   Parking   cook_state_launch of a job with retry facts parks its pending slot instead of freeing it: the live flag is
 *             cleared and the generation bumped as by a removal (the job leaves the queue and every reader, all of
 *             which test the live flag), the columns and the three lists are kept, and the slot stays off the free
 *             list, so parked slots count against the pending table's capacity.  The host's counts drop the row as a
 *             launch does; the list compaction keeps the parked slots' entries and counts them as kept.  A job without
 *             retry facts launches exactly as before, and while no job of a handle has retry facts no call changes its
 *             behaviour, launches, transfers or cost.  Parked copies and facts are outside cook_state_digest and
 *             cook_state_export: a resync does not repair them (the caller sends the facts again; a job whose copy is
 *             gone answers COOK_JOB_WAITING_UNRETAINED and is upserted).
 *   Decision  one status at a time, in batch order (Cook writes each status in its own transaction).  The attempts
 *             consumed are reasons->attempts-consumed (:1154-1172) over the job's done instances, this one included:
 *             a reason counts once per instance, -1 (nil) or a code outside the dictionary as a plain failure, a
 *             success's reason too; a mea-culpa reason is free up to its limit (its failure limit, the global limit
 *             when -2, 0 under COOK_RF_DISABLE_MEA_CULPA; -1 unlimited).  Then, in order: the job is COOK_RF_COMPLETED
 *             -> COOK_JOB_COMPLETED (no change); a success, or no other live instance and attempts >= max_retries ->
 *             COOK_JOB_COMPLETED; another live running or unknown instance of the job -> COOK_JOB_RUNNING; else
 *             COOK_JOB_WAITING with a parked copy, COOK_JOB_WAITING_UNRETAINED without one (a job whose tasks came in
 *             through running upserts: the caller upserts the row as before).
 *   Requeue   the parked slot becomes live with a new generation, so it enters the queue at the next cook_state_rank as
 *             an upsert would; reserved_host becomes -1 (the reservation was consumed at launch), the job facts of
 *             cook_state_job_facts are cleared as by an upsert, allowed and plugin_accept stay.  The failed instance's
 *             hostname code is appended to the novel-host list (novel-host-constraint, constraints.clj:68-94) unless
 *             it is -1, the instance was preempted, or the list holds it.  A list that gains an entry moves to the
 *             arena's tail on the device (an order-wide scan of the new lengths, then a warp per row); the others stay
 *             in place.  The state then equals, for every reader, cook_state_finish_history followed by a
 *             cook_state_apply upsert of that row with the appended list and reserved_host = -1.
 *   Freeing   a parked copy is freed (its entries dead, its slot back on the free list) by a COOK_JOB_COMPLETED
 *             decision; by cook_state_retry_facts with COOK_RF_COMPLETED while the job has no live instance; by a
 *             pending upsert of its job id (the caller's row wins); by cook_state_finish or cook_state_finish_history
 *             of the job's last live instance; by a reset.  A pending upsert or removal of a job id drops its facts;
 *             so do a COOK_JOB_COMPLETED decision and a finish of the last live instance when the job has no live
 *             pending row.
 *
 * cook_state_retry_config: the reason dictionary (reason_code[i], whether it is mea culpa, its failure limit: -2 none,
 * use mea_culpa_limit; -1 unlimited) and the global mea-culpa limit (-1 unlimited), replacing the previous ones.  A
 * fresh handle has limit 5 and an empty dictionary.  Host only: no transfer, no device work, no statistics.
 * COOK_E_BADARG, with nothing changed: n_reasons < 0; a NULL array while n_reasons > 0; a negative or repeated code; a
 * failure limit below -2; mea_culpa_limit below -1.                                                              */
enum { COOK_RF_DISABLE_MEA_CULPA = 1, COOK_RF_COMPLETED = 2 };
enum { COOK_JOB_COMPLETED = 0, COOK_JOB_RUNNING = 1, COOK_JOB_WAITING = 2, COOK_JOB_WAITING_UNRETAINED = 3,
       COOK_JOB_NO_FACTS = 4 };
int32_t cook_state_retry_config(cook_pool* pool, int32_t mea_culpa_limit, int32_t n_reasons, const int32_t* reason_code,
                                const uint8_t* mea_culpa, const int32_t* failure_limit);

/* The retry facts of jobs the handle holds (a live pending row, a parked copy or a live running instance), replacing
 * earlier ones: max_retries[i] (:job/max-retries), flags[i] (COOK_RF_*: :job/disable-mea-culpa-retries, the job is
 * completed) and the reason codes done_reason[done_off[i], done_off[i + 1]) of its earlier done (success or failed)
 * instances, -1 for none; done_off NULL: no done instance.  The facts survive launch and requeue.  A job given
 * COOK_RF_COMPLETED while it has no live instance loses its parked copy and its facts.
 * COOK_E_BADARG, before any change: n < 0; a NULL job_id, max_retries or flags while n > 0; malformed CSR offsets; a
 * reason code below -1; a negative max_retries; unknown flag bits; a job id the handle does not hold or listed twice.
 * Uploads exactly 4 bytes per parked copy freed, else nothing.  Statistics: cook_last_stats(COOK_PHASE_STATE).   */
int32_t cook_state_retry_facts(cook_pool* pool, int32_t n, const int64_t* job_id, const int32_t* max_retries,
                               const uint8_t* flags, const int32_t* done_off, const int32_t* done_reason);

/* Terminal statuses by task id: exactly cook_state_finish_history(pool, n, task_id, end_time_ms, success, reason_code)
 * (the removal, the straggler records, the history append, the same checks), and in addition each row's job decided
 * as above, in batch order: out_outcome[i] (COOK_JOB_*) and out_attempts[i] (the attempts consumed after this instance;
 * -1 with COOK_JOB_NO_FACTS, the job having no facts, when nothing else happens).  The reason is reason_code[i] or,
 * with reason_code NULL, the row's cook_state_task_reason fact; preempted[i] != 0 (:instance/preempted?) keeps the host
 * off the novel-host list; NULL: none preempted.  Requeues and frees as above, on the device.
 * COOK_E_BADARG, before any change: everything cook_state_finish_history rejects; a NULL out_outcome or out_attempts
 * while n > 0.  COOK_E_TOO_LARGE: as cook_state_finish_history.
 * Uploads exactly cook_state_finish_history's, plus 4 per requeued row (its slot), 8 per requeued row whose list gains
 * a host (its slot and the code) and 4 per parked copy freed.  Downloads nothing.
 * Statistics: cook_last_stats(COOK_PHASE_STATE).                                                                  */
int32_t cook_state_status(cook_pool* pool, int32_t n, const int64_t* task_id, const uint8_t* success,
                          const int64_t* end_time_ms, const int32_t* reason_code, const uint8_t* preempted,
                          int32_t* out_outcome, int32_t* out_attempts);

/* The record table by hand: first every record of the groups forget_group[0, n_forget) leaves (groups the caller no
 * longer tracks), then n_add records (group[i], runtime_s[i]) are appended: the successes that finished before the
 * rows were resident (after a reset or a leadership change).
 * COOK_E_BADARG, before any change: a negative size; a NULL array with its size > 0; a negative group code or
 * runtime.  COOK_E_TOO_LARGE: more than 2^31 - 1 records.  Uploads exactly 4 * (the distinct codes of forget_group)
 * + 8 * n_add bytes.  Statistics: cook_last_stats(COOK_PHASE_STATE).                                           */
int32_t cook_state_group_runtimes(cook_pool* pool, int32_t n_add, const int32_t* group, const int32_t* runtime_s,
                                  int32_t n_forget, const int32_t* forget_group);

/* The three kill lists over the union of the live running rows of pools[0, n_pools): the handles follow
 * cook_state_user_stats' rules (one device, idle, the work on pools[0]'s stream and scratch).  Each list comes with
 * the index in pools of the handle that holds the row.  A NULL task-id array skips that sweep and its kernels.
 *   Lingering  (out_linger_*) every row, running or unknown, with now_ms - start > min(max_runtime, max_timeout_ms),
 *              max_runtime the row's max_runtime_ms or default_timeout_ms when it has none; int64, strict (a row whose
 *              boundary equals now_ms is not lingering).  The caller derives both timeouts from its hours as
 *              kill-lingering-tasks does (:1912-1918).
 *   Cancelled  (out_cancel_*) every row with the cancelled fact, running or unknown.
 *   Stragglers (out_straggler_*) for each group g < n_groups with group_kind[g] == COOK_SWEEP_QUANTILE_DEVIATION:
 *              idx = (int)((double)(n_jobs[g] - 1) * quantile[g]) (truncated toward zero; n_jobs[g] counts the group's
 *              jobs in every state); when the group has more than idx live records, limit = (double)(its idx-th
 *              smallest runtime_s) * multiplier[g], and every row of status running (not unknown) with g in its group
 *              list and (double)((now_ms - start) / 1000) > limit is a straggler of g.  A row in several groups is
 *              judged once per group.  COOK_SWEEP_NONE yields nothing; so does idx < 0 (n_jobs 0 with quantile 1,
 *              where the reference's nth throws).
 * Orders (the reference returns sets): lingering and cancelled by ascending task id, a task id several handles hold
 * by pool index; stragglers by ascending (group, task id, pool index).  *out_n_* gets each list's length.
 * Capacities: row_cap >= the live running rows (lingering, cancelled), entry_cap >= the live running rows' group
 * entries (stragglers).  Changes nothing resident.
 * COOK_E_BADARG, before any device work and with nothing written: cook_state_user_stats' handle cases; a list without
 * its pool column or count; n_groups < 0; (stragglers) a NULL group_kind, quantile, multiplier or n_jobs with
 * n_groups > 0, an unknown kind, a quantile outside [0, 1] for a checked group, a negative n_jobs, a live running
 * row's group or a record's group >= n_groups; a capacity below the required size.  COOK_E_BADARG after the sweep
 * and with nothing written: a running row of a checked group that starts after now_ms (the reference's interval
 * throws and aborts the sweep; this error is ours).
 * No live row to judge: empty lists without device work.
 * Transfers exactly: up 24 * n_groups (the four group columns) when the stragglers are swept over some group entry;
 * down 16 (the counts) + 12 per lingering and per cancelled row + 16 per straggler.  Nothing that scales with the
 * running table crosses the bus.
 * Statistics: out_stats (may be NULL), as cook_state_user_stats; no cook_last_stats slot is written.  The parameters
 * are plain arguments, like cook_state_user_stats' outputs: every struct of this header has a ctypes mirror. */
enum { COOK_SWEEP_NONE = 0, COOK_SWEEP_QUANTILE_DEVIATION = 1 };
int32_t cook_state_sweep(cook_pool* const* pools, int32_t n_pools, int64_t now_ms, int64_t default_timeout_ms,
                         int64_t max_timeout_ms, int32_t n_groups, const int32_t* group_kind, const double* quantile,
                         const double* multiplier, const int32_t* n_jobs, int32_t row_cap, int64_t* out_linger_task_id,
                         int32_t* out_linger_pool, int32_t* out_n_linger, int64_t* out_cancel_task_id,
                         int32_t* out_cancel_pool, int32_t* out_n_cancel, int32_t entry_cap,
                         int32_t* out_straggler_group, int64_t* out_straggler_task_id, int32_t* out_straggler_pool,
                         int32_t* out_n_straggler, cook_phase_stats* out_stats);

/* ------------------------------------------------ why a resident pool's job is not scheduled */
/* The device half of /unscheduled_jobs (reasons, unscheduled.clj:172-200) for n queried job ids of one handle; the
 * caller compares the usage with the user's quota and share maps and assembles the reasons (cycle.unscheduled_reasons).
 * For each job_id[i], answered independently of repeats:
 *   out_status[i]    COOK_UNSCHED_WAITING when a live pending row holds the id; else COOK_UNSCHED_RUNNING when a live
 *                    running row carries it as its job id; else COOK_UNSCHED_ABSENT (completed, or another pool's).
 * The user's running jobs are the distinct job ids of the user's live running rows (running and unknown alike), each
 * represented by its row with the greatest task id.  The job's user is its pending row's, or (RUNNING) that of the
 * job's live running row with the greatest task id.
 *   out_usage[4i..4i+3]  (WAITING) count, cpus, mem, gpus: a left fold over the user's running jobs' representatives in
 *                    ascending task id (count 1.0 each, cook_state_usage's fold when every job has one row), then plus
 *                    the job (count 1.0, its cpus, mem, gpus); zeros otherwise.
 *   out_position[i]  (WAITING, RUNNING) the number of the user's entries before the job's own, where the entries are
 *                    the representatives and the user's live pending rows in the same-user task order of cook_state_rank
 *                    (-priority, start (pending INT64_MAX), task id (pending -1), job id); -1 otherwise.  A job with a
 *                    pending row and running rows is WAITING, and its running rows still count.
 *   out_ahead_job_id[COOK_UNSCHED_AHEAD*i ..]  the job ids of the first out_n_ahead[i] = min(position, COOK_UNSCHED_AHEAD)
 *                    entries in that order, 0 after them.
 *   out_plugin_deferred[i]  (WAITING) 1 when the row's plugin_accept is 0; 0 otherwise.
 * No submit-time window and no cap on the waiting jobs: every live row counts.  Changes nothing resident (rows, queue,
 * match plan, COOK_USAGE_LAST_MATCH).
 * COOK_E_BADARG, before any device work and with nothing written: n < 0; a NULL handle, job_id or output (but
 * out_stats) while n > 0.  n == 0, or no queried job in the handle: no device work (statistics zero).
 * Transfers exactly, otherwise: up 4 * (the distinct users of the queried jobs found) + 4 * n; down 121 * n (usage 32,
 * position 4, count 4, ahead 80, plugin 1).  Nothing that scales with the tables crosses the bus.
 * Statistics: out_stats (may be NULL), as cook_state_user_stats; no cook_last_stats slot is written.             */
enum { COOK_UNSCHED_ABSENT = 0, COOK_UNSCHED_WAITING = 1, COOK_UNSCHED_RUNNING = 2, COOK_UNSCHED_AHEAD = 10 };
int32_t cook_state_unscheduled(cook_pool* pool, int32_t n, const int64_t* job_id, uint8_t* out_status,
                               double* out_usage, int32_t* out_position, int32_t* out_n_ahead,
                               int64_t* out_ahead_job_id, uint8_t* out_plugin_deferred, cook_phase_stats* out_stats);

/* ------------------------------------------------------------- users' running usage over resident pools */
/* The device half of GET /usage (get-user-usage, api.clj:2946-2969; user-usage :2894-2915) over the union of the live
 * running rows of pools[0, n_pools), for the user codes user[0, n_users) or, with user NULL (n_users 0), every user.
 * Each handle is one pool; the handles follow cook_state_user_stats' rules (one device, idle, the work on pools[0]'s
 * stream and scratch).  Pools on different GPUs: one call per device and the host's addition.  Fixed choices:
 *   Jobs      a running job is a distinct (handle, job id) over the live running rows, running and status-unknown
 *             alike; its representative is its row with the greatest task id (cook_state_unscheduled's rule).
 *   Order     every fold is a left fold from +0.0 over the segment's representatives in ascending (task id, pool
 *             index); jobs is an integer count; the job lists come in the same order.
 *   Group     a job's group is the first entry of its representative's running group list, as the delta or the
 *             launch gave it; an empty list is ungrouped.  The reference's "first of a set" is the caller's order.
 *   Segments  (user, scope, group): scope -1 is all the handles, p (per_pool != 0 only) handle p; group
 *             COOK_UU_TOTAL the scope's total, COOK_UU_UNGROUPED the jobs without a group, g >= 0 (by_group != 0 only)
 *             group code g.  A segment is emitted only when it holds a job (the host builds the zero maps), in
 *             ascending (user, scope, group): -1 before the handles, COOK_UU_TOTAL, COOK_UU_UNGROUPED, then codes.
 *   Outputs   per segment d < *out_n_seg: out_user, out_scope, out_group, out_jobs, out_cpus, out_mem, out_gpus; with
 *             by_group, out_list_off[d] (-1 for a total) is where the segment's out_jobs[d] job ids start in
 *             out_job_id[0, *out_n_job), segments in order.  Without by_group, out_list_off and out_job_id are not
 *             read and *out_n_job = 0.
 *   Sizes     with R_q the live running rows of the queried users over the handles (the library's host-side
 *             counts): seg_cap >= R_q * (1 + per_pool) * (1 + by_group), and with by_group job_cap >=
 *             R_q * (1 + per_pool).
 * Changes nothing resident (rows, queue, match plan, COOK_USAGE_LAST_MATCH).
 * COOK_E_BADARG, before any device work and with nothing written: cook_state_user_stats' handle cases; a NULL output
 * (out_list_off and out_job_id only with by_group; out_stats may be NULL); n_users < 0, or n_users != 0 with user
 * NULL; a negative user code or one listed twice; a capacity below its bound.  COOK_E_TOO_LARGE: R_q * (1 + per_pool)
 * * (1 + by_group) >= 2^31.  R_q == 0: empty results without device work (statistics zero).
 * Transfers exactly, otherwise: up 4 * n_users; down 8 (the counts) + (44 + 4 * by_group) * *out_n_seg + 8 *
 * *out_n_job.  Nothing that scales with the tables crosses the bus.
 * Statistics: out_stats (may be NULL), as cook_state_user_stats; no cook_last_stats slot is written.  The outputs are
 * plain arrays, like cook_state_user_stats' outputs: every struct of this header has a ctypes mirror. */
enum { COOK_UU_TOTAL = -2, COOK_UU_UNGROUPED = -1 };
int32_t cook_state_user_usage(cook_pool* const* pools, int32_t n_pools, const int32_t* user, int32_t n_users,
                              int32_t per_pool, int32_t by_group, int32_t seg_cap, int32_t* out_user,
                              int32_t* out_scope, int32_t* out_group, int64_t* out_jobs, double* out_cpus,
                              double* out_mem, double* out_gpus, int32_t* out_list_off, int32_t job_cap,
                              int64_t* out_job_id, int32_t* out_n_seg, int32_t* out_n_job, cook_phase_stats* out_stats);

/* ------------------------------------------------------- instance stats over resident pools */
/* The device half of GET /stats/instances with status running or unknown and no name filter (task-stats/get-stats,
 * task_stats.clj) over the union of the live running rows of pools[0, n_pools); the handles follow
 * cook_state_user_stats' rules (on one device or several).  Percentiles do not compose from per-device summaries, so
 * another device sends its live running rows themselves, 45 B a row, and the answer is the bits of one device.
 *   Selection  (get-tasks) a row is selected when its status is `status` (COOK_IS_RUNNING: without the unknown fact of
 *              cook_state_task_facts; COOK_IS_UNKNOWN: with it), task_id_lo <= task id < task_id_hi (the caller's
 *              d/entid-at of start - 1 h and end + 1 h; the bound is part of the reference's semantics) and
 *              start_ms <= start < end_ms.
 *   Entries    (task->task-entry) run_time = (double)(now_ms - start) / 1000.0, cpu = run_time * cpus, mem = run_time *
 *              mem, each an f64 product; reason the row's cook_state_task_reason code (-1: none); user the row's.
 *   Segments   (generate-all-stats) kind COOK_IS_OVERALL (user -1, reason -1), COOK_IS_REASON (user -1) and
 *              COOK_IS_USER_REASON; only non-empty segments, in ascending (kind, user, reason), -1 first.  No selected
 *              row: no segment (the reference's {} overall).
 *   Outputs    per segment d < *out_n_seg: out_kind, out_user, out_reason, out_count (rows), and for metric m
 *              (COOK_IS_RUN_TIME, COOK_IS_CPU, COOK_IS_MEM) out_total[3 * d + m] and out_pct[15 * d + 5 * m + j], the
 *              nearest-rank percentiles p = 50, 75, 95, 99, 100: element ceil(p * n / 100) - 1 of the segment's n
 *              values in ascending order.  Leaders: for k = 0 (cpu) and 1 (mem), out_leader_user / out_leader_total
 *              [COOK_IS_LEADERS * k + i], i < *out_n_leader = min(COOK_IS_LEADERS, users selected): the users with the
 *              largest per-user total of that metric, totals descending.
 * Fixed choices:
 *   Now      one now_ms for the whole call (the reference calls t/now per lazily realised entry).
 *   Order    every total is a left fold from +0.0 in ascending (task id, pool index), a task id several handles hold by
 *            pool index; a user's leader total is its own fold over all its selected rows, not a sum of its per-reason
 *            totals.  The percentile sort is by value; equal values are equal bits (no value is -0.0 or NaN).
 *   Ties     leaders of equal totals go by ascending user code (the reference's order is its user map's hash order).
 * Sizes: seg_cap >= 1 + 2 * R, R the live running rows over the handles (the library's host-side counts).
 * Changes nothing resident (rows, queue, match plan, COOK_USAGE_LAST_MATCH).
 * COOK_E_BADARG, before any device work and with nothing written: cook_state_user_stats' handle cases; an unknown
 * status; end_ms <= start_ms; a NULL output (out_stats may be NULL); seg_cap below its bound.  COOK_E_TOO_LARGE: 4 * R
 * >= 2^31.  COOK_E_BADARG after the selection, with nothing written: a selected row that starts after now_ms (the
 * reference's interval throws; this error is ours).  No live row: empty results without device work (statistics
 * zero).
 * Transfers exactly: up nothing; down 8 (the selection's count and flag), and when a row is selected 8 (the counts)
 * + 164 * *out_n_seg (kind, user, reason, count, three totals, fifteen percentiles) + 24 * *out_n_leader.
 * Statistics: out_stats (may be NULL), as cook_state_user_stats; no cook_last_stats slot is written.  The outputs are
 * plain arrays, like cook_state_user_stats' outputs: every struct of this header has a ctypes mirror. */
enum { COOK_IS_RUNNING = 0, COOK_IS_UNKNOWN = 1, COOK_IS_SUCCESS = 2, COOK_IS_FAILED = 3 };
enum { COOK_IS_OVERALL = 0, COOK_IS_REASON = 1, COOK_IS_USER_REASON = 2 };
enum { COOK_IS_RUN_TIME = 0, COOK_IS_CPU = 1, COOK_IS_MEM = 2, COOK_IS_LEADERS = 10 };
int32_t cook_state_instance_stats(cook_pool* const* pools, int32_t n_pools, int64_t now_ms, int32_t status,
                                  int64_t start_ms, int64_t end_ms, int64_t task_id_lo, int64_t task_id_hi,
                                  int32_t seg_cap, int32_t* out_kind, int32_t* out_user, int32_t* out_reason,
                                  int64_t* out_count, double* out_total, double* out_pct, int32_t* out_leader_user,
                                  double* out_leader_total, int32_t* out_n_seg, int32_t* out_n_leader,
                                  cook_phase_stats* out_stats);

/* The device half of GET /stats/instances with status success or failed and no name filter, over the union of the
 * history tables (cook_state_history_seed) of pools[0, n_pools); the handles follow cook_state_user_stats' rules.
 * Outputs, segments, fold order, percentiles, leaders and their tie rule are cook_state_instance_stats', with:
 *   Selection  status COOK_IS_SUCCESS (the success flag set) or COOK_IS_FAILED (clear; only this call accepts the two),
 *              task_id_lo <= task id < task_id_hi and start_ms <= start < end_ms.
 *   Entries    run_time = (double)(end - start) / 1000.0 (task-run-time with the instance's end time), cpu = run_time *
 *              cpus, mem = run_time * mem.  There is no now.
 *   Order      every total is a left fold from +0.0 in ascending (task id, pool index, table position): the position
 *              keeps the answer deterministic when one handle holds a task id twice (a caller's divergence, not
 *              checked after the seed).  Leaders of equal totals go by ascending user code.
 * Sizes follow the selection S: every buffer after a count pass is sized by S, and only S crosses devices (48 B a row).
 * COOK_E_BADARG, before any device work and with nothing written: cook_state_user_stats' handle cases; an unknown
 * status; end_ms <= start_ms; a NULL output (out_stats may be NULL); seg_cap < 0; a handle whose history is off or
 * whose horizon is > start_ms (the caller then keeps the Datomic path).  COOK_E_TOO_LARGE: 4 * S >= 2^31, with nothing
 * written; more than seg_cap segments, with only *out_n_seg (the segments needed) written, so that the caller can
 * retry with that capacity.  No handle holds a row: empty results without device work (statistics zero).
 * Transfers exactly: up nothing; down 4 * H (one count per handle holding a row, whichever device counts it), plus,
 * when a row is selected, 8 (the counts), plus, when *out_n_seg <= seg_cap, 164 * *out_n_seg + 24 * *out_n_leader.
 * Statistics: out_stats (may be NULL), as cook_state_instance_stats.  Changes nothing resident.                    */
int32_t cook_state_history_stats(cook_pool* const* pools, int32_t n_pools, int32_t status, int64_t start_ms,
                                 int64_t end_ms, int64_t task_id_lo, int64_t task_id_hi, int32_t seg_cap,
                                 int32_t* out_kind, int32_t* out_user, int32_t* out_reason, int64_t* out_count,
                                 double* out_total, double* out_pct, int32_t* out_leader_user,
                                 double* out_leader_total, int32_t* out_n_seg, int32_t* out_n_leader,
                                 cook_phase_stats* out_stats);

/* ------------------------------------------------- match-cycle metrics of resident pools */
/* What handle-match-cycle-metrics (scheduler.clj:1210-1280) and the unmatched tracking (:1399-1486) read after each
 * match, before the launches, computed from the resident rows of the last match round.
 *
 * Job facts: the keys jobs->resource-maps (:511-545) reads, which are not the matcher's columns (P_GPU_MODEL and the
 * disk constraint carry pool and config defaults).  On live pending rows, by job id, in place like
 * cook_state_task_facts (live flag and generation kept); a NULL column is left unchanged.
 *   flags[i]         COOK_JF_* bits: GPUS the job has a gpus resource (an amount of 0.0 counts: `(if gpus ...)`), DISK
 *                    a disk resource, DISK_REQUEST / DISK_LIMIT its request / limit is present (needs DISK), URIS at
 *                    least one uri
 *   gpu_model[i]     the code of the job's COOK_GPU_MODEL environment value, -1: unspecified-gpu-model
 *   disk_request[i], disk_limit[i]   the amounts, read under their bits
 *   disk_type[i]     the code of :resource.disk/type, -1: unspecified-disk-type
 * The gpus amount is the row's gpus column.  Every pending upsert of cook_state_apply writes flags 0 (no facts).  The
 * facts are not part of cook_state_digest or cook_state_export: after a resync the caller sends them again.
 * COOK_E_BADARG, before any change: n < 0; a NULL job_id while n > 0; a job id that is not live or appears twice; an
 * unknown flag bit, or DISK_REQUEST / DISK_LIMIT without DISK; a gpu model or disk type code below -1; a NaN amount.
 * Uploads exactly, when n > 0 and some column is given: n * (4 + [flags] 1 + [gpu_model] 4 + [disk_request] 8 +
 * [disk_limit] 8 + [disk_type] 4) bytes.  Statistics: cook_last_stats(COOK_PHASE_STATE).                       */
enum { COOK_JF_GPUS = 1, COOK_JF_DISK = 2, COOK_JF_DISK_REQUEST = 4, COOK_JF_DISK_LIMIT = 8, COOK_JF_URIS = 16 };
int32_t cook_state_job_facts(cook_pool* pool, int32_t n, const int64_t* job_id, const uint8_t* flags,
                             const int32_t* gpu_model, const double* disk_request, const double* disk_limit,
                             const int32_t* disk_type);

/* The metrics of the last cook_state_match, cook_state_match_derived or cook_state_match_offers on the handle: its
 * considerable jobs in take order and their assignments.  dropped[n_dropped]: the considerable positions whose
 * matches the launch-rate filter dropped (filter-matches-for-ratelimit :887-924); they count as unmatched.
 *   Counts      out_counts[COOK_MMC_*]: considerable, matched (after the drops), the head's job id (-1: none), whether
 *               the head is matched, the rows with a uri, that row's position when there is exactly one (else -1),
 *               the keyed totals, the rows unmatched too long, the first ones listed (at most 10).
 *   Per user    out_user_considerable[u], out_user_matched[u] for u < n_users (unmatched = the difference).
 *   cpus, mem   out_amounts[COOK_MMA_*]: totals, left folds in take order (the exact grid or the serial chain,
 *               DESIGN.md §2); percentiles 50, 95, 100: element ceil(p * n / 100) - 1 of the ascending values
 *               (task_stats.clj's exact p/100); the largest rows: the LAST row of maximal value in take order (sort-by
 *               is stable and `last` takes the last).
 *   Keyed       one total per (kind, code) some considerable row carries, kind COOK_MM_GPUS (code: gpu model),
 *               COOK_MM_DISK_REQUEST or COOK_MM_DISK_LIMIT (code: disk type), -1 being the unspecified value, in
 *               ascending (kind, code): the left fold in take order of the rows that carry the key (merge-with +).
 *               More keys than key_cap: only out_counts[COOK_MMC_KEYS] is written, COOK_E_TOO_LARGE, the round stays uncounted,
 *               so the caller can retry with a larger cap.
 *   Rows        the head, the largest by cpus and the largest by mem (COOK_MM_HEAD, _LARGEST_CPUS, _LARGEST_MEM): row r's
 *               integers in out_row_int[COOK_MMR_NI * r + COOK_MMR_*] (job id, position, user, ports, COOK_JF_* facts,
 *               gpu model, disk type; -1: unspecified) and its amounts in out_row_amount[COOK_MMR_NF * r + COOK_MMR_*]
 *               (cpus, mem, gpus, disk request, disk limit; an absent disk amount is 0.0): :head-resources and
 *               :largest-by without a job-entity read, except for the uri strings.
 *   Uris        with two or more such rows, jobs->stats is "Error collecting job stats" (merge-with + adds two
 *               vectors and throws); with one, its resource map keeps :uris.
 *   Unmatched   every job has a cycle count, keyed by job id: after the call it is the previous count + 1 for a
 *               considerable job that is unmatched (dropped ones included) and 0 for every other job, as the
 *               reference's map rebuilt each cycle.  The counts live on the device as the last counted round's
 *               unmatched (job id, count) pairs, so an upsert of a pending id, or its removal and return, keeps its
 *               count.  COOK_MMC_TOO_LONG counts the rows with count > unmatched_warn_cycles (strictly);
 *               out_first_job_id / out_first_cycles [10] list the first ten in TAKE ORDER (-1 and 0 past them), a fixed
 *               choice: the reference takes them in hash-map order, which is
 *               unspecified.  The fraction test of the warning stays with the caller.
 * Call it after the match and before the launches, once per round.  A reset through cook_state_apply drops the round
 * and the counts.
 * Empty round (no considerable job): out_counts gets zeros (the head's job id and the uri position -1), the
 * unmatched counts are zeroed, nothing else is written, no device work.
 * COOK_E_BADARG, with nothing written and no count changed: no resident round on the handle (none yet, or another
 * match ran on it since); the round was already counted; a considerable row upserted or removed since the match;
 * a pending row's user code >= n_users, or n_users <= 0; a dropped position out of [0, n_considerable), repeated or
 * holding no assignment; a NULL output (out_stats may be NULL), n_dropped < 0, a NULL dropped while n_dropped > 0,
 * unmatched_warn_cycles < 0, key_cap < 0.  The first two of the dropped position rules and the ones before are
 * checked before any device work, the others on the device before anything is written.
 * Transfers exactly: up 4 * n_dropped; down 32 (the counts), plus 4 * n_considerable when a pending row was upserted
 * or removed since the match (the rows' slots, for the check), plus 440 (the counts, amounts, rows and first ten as
 * one block), then, unless COOK_E_TOO_LARGE, 8 * n_users + 16 * n_keys.  Nothing moves in an empty round.
 * Statistics: out_stats (may be NULL) receives the call's own cook_phase_stats, as cook_state_user_stats; no
 * cook_last_stats slot is written.  The match keeps its outputs, launches and transfers: it records the round with
 * one device-to-device copy of its rows' slots.                                                               */
enum { COOK_MM_GPUS = 0, COOK_MM_DISK_REQUEST = 1, COOK_MM_DISK_LIMIT = 2 };
enum { COOK_MMC_CONSIDERABLE = 0, COOK_MMC_MATCHED = 1, COOK_MMC_HEAD_JOB_ID = 2, COOK_MMC_HEAD_MATCHED = 3,
       COOK_MMC_URIS = 4, COOK_MMC_URIS_POSITION = 5, COOK_MMC_KEYS = 6, COOK_MMC_TOO_LONG = 7, COOK_MMC_FIRST = 8,
       COOK_MMC_N = 9 };
enum { COOK_MMA_TOTAL_CPUS = 0, COOK_MMA_TOTAL_MEM = 1, COOK_MMA_PCT_CPUS = 2, COOK_MMA_PCT_MEM = 5, COOK_MMA_N = 8 };
enum { COOK_MM_HEAD = 0, COOK_MM_LARGEST_CPUS = 1, COOK_MM_LARGEST_MEM = 2, COOK_MM_ROWS = 3, COOK_MM_FIRST_N = 10 };
enum { COOK_MMR_JOB_ID = 0, COOK_MMR_POSITION = 1, COOK_MMR_USER = 2, COOK_MMR_PORTS = 3, COOK_MMR_FACTS = 4,
       COOK_MMR_GPU_MODEL = 5, COOK_MMR_DISK_TYPE = 6, COOK_MMR_NI = 7 };
enum { COOK_MMR_CPUS = 0, COOK_MMR_MEM = 1, COOK_MMR_GPUS = 2, COOK_MMR_DISK_REQUEST = 3, COOK_MMR_DISK_LIMIT = 4,
       COOK_MMR_NF = 5 };
int32_t cook_state_match_metrics(cook_pool* pool, int32_t n_users, int32_t n_dropped, const int32_t* dropped,
                                 int32_t unmatched_warn_cycles, int32_t key_cap, int64_t* out_counts,
                                 double* out_amounts, int64_t* out_row_int, double* out_row_amount,
                                 int64_t* out_first_job_id, int32_t* out_first_cycles, int32_t* out_user_considerable,
                                 int32_t* out_user_matched, int32_t* out_key_kind, int32_t* out_key_code,
                                 double* out_key_total, cook_phase_stats* out_stats);

/* ------------------------------------------------- job listing over resident pools */
/* The device half of GET /list and the list form of GET /jobs for the waiting and running states
 * (get-active-jobs-by-user-and-state, tools.clj:445-466): one user's jobs in a submit window, read from the resident
 * rows instead of a walk of every job in the state.
 *
 * List facts: the three job attributes the listing filters on, which never change over a job's life.  By job id, on
 * the job's live pending row and on each of its live running rows, in place like cook_state_job_facts (live flag and
 * generation kept); a NULL column is left unchanged.
 *   submit_ms[i]        :job/submit-time in ms since the epoch
 *   submit_pool[i]      the code of :job/submit-pool-name (the caller's pool dictionary), -1: none
 *   custom_executor[i]  :job/custom-executor, -1 nil, 0 false, 1 true (the filters tell the three apart)
 * A row has facts once custom_executor has been written to it; the other two are read only then, so the caller sends
 * the three together.  Every pending and every running upsert of cook_state_apply writes "no facts" (inside the
 * scatter it already runs: apply's launches and transfers are unchanged).  cook_state_launch copies the pending row's
 * facts to the new running row on the device (no upload).  A parked copy (cook_state_retry_facts) and the in-place
 * requeue of cook_state_status keep them: unlike the job facts, which a requeue clears, these attributes are fixed
 * when the job is submitted.  Not part of cook_state_digest or cook_state_export: after a resync the caller sends
 * them again.  The columns add 13 B per pending row and 13 B per running row (submit 8, pool 4, executor and the
 * facts-present state 1), about 130 MB at 10 M jobs.
 * COOK_E_BADARG, before any change: n < 0; a NULL job_id while n > 0; a job id that is neither live-pending nor
 * live-running, or that appears twice; a custom_executor outside {-1, 0, 1}; a submit pool code below -1.
 * Uploads exactly, when n > 0 and some column is given: (P + R) * (4 + [submit_ms] 8 + [submit_pool] 4 +
 * [custom_executor] 1) bytes, P the listed jobs with a live pending row and R their live running rows (a slot and
 * each non-NULL column per row written; the executor goes up as its one-byte stored code).  Statistics: cook_last_stats(COOK_PHASE_STATE).                        */
int32_t cook_state_list_facts(cook_pool* pool, int32_t n, const int64_t* job_id, const int64_t* submit_ms,
                              const int32_t* submit_pool, const int32_t* custom_executor);

/* The listing over the union of the live rows of pools[0, n_pools); the handles follow cook_state_user_stats' rules
 * (one device, idle, the work on pools[0]'s stream and scratch).  states: COOK_LJ_WAITING and/or COOK_LJ_RUNNING.
 *   Rows       waiting: the live pending rows (committed jobs only, so `(remove uncommitted?)` holds by
 *              construction); running: the distinct (handle, job id) over the live running rows, running and unknown
 *              alike, represented by the row with the greatest task id (cook_state_unscheduled's rule).
 *   Selection  an entry is selected when its user is `user`, its (representative's) facts are present, start_ms <=
 *              submit < end_ms (job-submitted-in-range?), job_id_lo <= job id < job_id_hi (the caller's d/entid-at of
 *              start - 1 h and end + 1 h: the bound is part of the reference's semantics), the pool check passes
 *              (check-pool-for-listing, pool.clj:22-42: pool_code == -1, or handle_pool[k] == pool_code, or the submit
 *              pool == pool_code; a job without :job/pool lives in the default pool's handle) and the executor check
 *              passes (include_custom_executor 0 keeps custom_executor == 0 only, the reference's `false?`, so nil is
 *              dropped; 1 keeps every entry).
 *   Order      within each state ascending (job id, pool index), the reference's entity-id traversal; each state keeps
 *              its first `limit` entries, as its `(take limit)` before the merge.  Waiting entries first, then running.
 *   Outputs    entry e < *out_n: out_state[e] (COOK_LJ_*), out_job_id, out_submit_ms, out_pool (the index in pools).
 *              *out_n_missing: the rows of `user` in a requested state inside the id window without facts; when it is
 *              not 0 the caller keeps the Datomic path.
 * Changes nothing resident.
 * COOK_E_BADARG, before any device work and with nothing written: cook_state_user_stats' handle cases; states 0 or
 * with unknown bits; a negative user; pool_code below -1, or handle_pool NULL while pool_code != -1;
 * include_custom_executor outside {0, 1}; limit < 0 or cap < 0; a NULL output (out_stats may be NULL).
 * COOK_E_TOO_LARGE: more than 2^31 - 1 rows of `user` in a state over the handles, with nothing written; more than
 * cap entries, with only *out_n (the entries needed) written, so that the caller can retry with that capacity.
 * No row of `user` in a requested state: empty results without device work (statistics zero).
 * Transfers exactly: up nothing; down 12 (the two states' entry counts and the missing count), plus, unless
 * COOK_E_TOO_LARGE, 20 * *out_n (job id, submit time, pool index; the states are known on the host).  Nothing that
 * scales with the tables crosses the bus.
 * Statistics: out_stats (may be NULL), as cook_state_user_stats; no cook_last_stats slot is written.             */
enum { COOK_LJ_WAITING = 1, COOK_LJ_RUNNING = 2 };
int32_t cook_state_list_jobs(cook_pool* const* pools, int32_t n_pools, int32_t user, int32_t states, int64_t start_ms,
                             int64_t end_ms, int64_t job_id_lo, int64_t job_id_hi, int32_t pool_code,
                             const int32_t* handle_pool, int32_t include_custom_executor, int32_t limit, int32_t cap,
                             int32_t* out_state, int64_t* out_job_id, int64_t* out_submit_ms, int32_t* out_pool,
                             int32_t* out_n, int32_t* out_n_missing, cook_phase_stats* out_stats);

/* ------------------------------------------------- completed-job log and its listing */
/* The device half of GET /list and the list form of GET /jobs for the completed, success and failed states
 * (get-completed-jobs-by-user, tools.clj:393-434), read from a per-handle log of job-state records instead of a walk
 * of every job the user submitted in the window.
 *
 * A handle's log: a device table of job-state records, 34 B per row (job id i64, stamp i64, submit ms i64, user i32,
 * submit pool code i32 with -1 for none, custom executor i8 with -1 nil / 0 false / 1 true, kind u8), in arrival
 * order.  Capacity doubles with device-to-device copies; rows leave only by a stable compaction.  The host keeps each
 * row's user and submit time too (12 B per row), so that the listing is sized without a transfer.  The log is off
 * until seeded; while it is off, no other call changes its behaviour or cost.  Not part of cook_state_digest or
 * cook_state_export (after a resync the caller seeds it again); a reset through cook_state_apply empties it and turns
 * it off.  No other call writes it: cook_state_apply, _launch, _status and _finish_history keep their columns,
 * launches and transfers.
 * Fixed choices:
 *   Kinds    COOK_CJ_SUCCESS and COOK_CJ_FAILED: the job is completed, its state success when an instance succeeded
 *            (job-ent->state); COOK_CJ_REOPENED: the job left the completed state (:job/ensure-not-completed,
 *            :job/update-retry-count, reached from /retry).
 *   Latest   a job's state is its record with the greatest stamp over the handles asked; equal stamps go to the greater
 *            handle index, then the later row.  The stamp is the Datomic t of the transaction that made the change, so
 *            a record sent twice changes nothing, and a job that moved pools between a reopen and a second completion
 *            is answered once.  A job whose latest record is REOPENED is not completed.
 *   Horizon  on submit time: every completed job of the pool submitted at or after since_ms is in the log, and a
 *            record submitted before it is not kept.  A listing that starts before a handle's horizon is refused,
 *            never answered partially.
 *
 * cook_state_completed_seed: replaces the log with rows [0, n), sets the horizon to since_ms and turns the log on (the
 * start-up and leadership-change path: the pool's completed jobs submitted at or after now - retention, read once
 * from one database value, its basis t as their stamp; the order is reset, load, seed, then resume the tap).
 * COOK_E_BADARG, before any change: n < 0; a NULL array while n > 0; a row submitted before since_ms; a negative user
 * or stamp; a kind outside COOK_CJ_*; a custom_executor outside {-1, 0, 1}; a submit pool code below -1; a job id
 * listed twice.
 * Uploads exactly 34 * n bytes, copied straight into the table (the executor as its byte).
 * Statistics: cook_last_stats(COOK_PHASE_STATE).                                                                  */
enum { COOK_CJ_SUCCESS = 1, COOK_CJ_FAILED = 2, COOK_CJ_REOPENED = 3 };
int32_t cook_state_completed_seed(cook_pool* pool, int64_t since_ms, int32_t n, const int64_t* job_id,
                                  const int64_t* stamp, const int32_t* user, const int64_t* submit_ms,
                                  const int32_t* submit_pool, const int32_t* custom_executor, const uint8_t* kind);

/* Appends the batch's records in order, skipping (on the host) those submitted before the horizon.  The append costs
 * O(n), not O(log).  COOK_E_BADARG, before any change: the log is off; every row check of cook_state_completed_seed
 * except the horizon; a job id twice in the batch.  COOK_E_TOO_LARGE: more than 2^31 - 1 rows.
 * Uploads exactly 34 * (the rows kept) bytes.  Statistics: cook_last_stats(COOK_PHASE_STATE).                      */
int32_t cook_state_completed_record(cook_pool* pool, int32_t n, const int64_t* job_id, const int64_t* stamp,
                                    const int32_t* user, const int64_t* submit_ms, const int32_t* submit_pool,
                                    const int32_t* custom_executor, const uint8_t* kind);

/* Raises the horizon to since_ms and drops the rows submitted before it in one stable device compaction (into new
 * columns of the same capacity, the old ones then freed).  The caller calls it periodically with now - retention.
 * COOK_E_BADARG: the log is off; since_ms below the current horizon.
 * Uploads nothing; downloads 4 bytes (the rows kept) when the log holds a row and since_ms is above the horizon, else
 * nothing.  Statistics: cook_last_stats(COOK_PHASE_STATE).                                                       */
int32_t cook_state_completed_advance(cook_pool* pool, int64_t since_ms);

/* The listing over the union of the logs of pools[0, n_pools); the handles follow cook_state_user_stats' rules, on one
 * device or several.  A job that moved pools has records on two handles, so the records themselves cross: a handle on
 * another device sends all of `user`'s records it holds (the job-id bounds and filters are applied on pools[0]), 29
 * bytes per record (job id, stamp, submit time, pool index, the filters' verdict), and the latest record per job and
 * the `limit` cut are those of one device.
 * state: COOK_LC_SUCCESS, COOK_LC_FAILED or COOK_LC_COMPLETED (both).
 *   Records    those of `user` with job_id_lo <= job id < job_id_hi (the caller's d/entid-at of start - 1 h and
 *              end + 1 h; user and job id never change over a job's life).  Each job is its latest record; a REOPENED
 *              one drops it.
 *   Selection  the kind matches `state`, and on the latest record: start_ms <= submit < end_ms
 *              (job-submitted-in-range?), the pool check and the executor check of cook_state_list_jobs.
 *   Order      ascending job id, the reference's entity-id traversal, cut to `limit` after the filters (its
 *              `(take limit)`).
 *   Outputs    entry e < *out_n: out_job_id, out_submit_ms, out_pool (the index in pools of the latest record).
 * Changes nothing resident.
 * COOK_E_BADARG, before any device work and with nothing written: cook_state_list_jobs' handle and argument cases
 * (except `states` and handles on different devices); state outside COOK_LC_*; a handle whose log is off; a handle
 * whose horizon is > start_ms (the caller then keeps the Datomic path); a NULL output (out_stats may be NULL).
 * COOK_E_TOO_LARGE: more than 2^31 - 1 records of `user` over the handles, with nothing written; more than cap
 * entries, with only *out_n (the entries needed) written, so that the caller can retry with that capacity.
 * No record of `user`: empty results without device work (statistics zero).
 * Transfers exactly: up nothing; down 4 (the entry count), plus, unless COOK_E_TOO_LARGE, 20 * *out_n (job id,
 * submit time, pool index).
 * Statistics: out_stats (may be NULL), as cook_state_user_stats; no cook_last_stats slot is written.             */
enum { COOK_LC_SUCCESS = 1, COOK_LC_FAILED = 2, COOK_LC_COMPLETED = 3 };
int32_t cook_state_list_completed(cook_pool* const* pools, int32_t n_pools, int32_t user, int32_t state,
                                  int64_t start_ms, int64_t end_ms, int64_t job_id_lo, int64_t job_id_hi,
                                  int32_t pool_code, const int32_t* handle_pool, int32_t include_custom_executor,
                                  int32_t limit, int32_t cap, int64_t* out_job_id, int64_t* out_submit_ms,
                                  int32_t* out_pool, int32_t* out_n, cook_phase_stats* out_stats);

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
