// common.cuh — handles, error plumbing and the device arena of libcookgpu.so.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/cook_gpu.h"

struct cook_ctx {
  std::vector<int> devices;
};

// Grow-only device arena: one cudaMalloc per high-water mark, carved per call by carve() below.
struct Arena {
  char* base = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (base) cudaFree(base);
    base = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 4 + (1 << 20);
    cudaError_t e = cudaMalloc(&base, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (base) cudaFree(base);
    base = nullptr;
    cap = 0;
  }
};

// One pass over a call's device buffers (see carve()).  While measuring (base == nullptr) every take
// returns nullptr and only advances the offset; while carving it returns the arena's memory and the
// uploads are queued on the stream.
struct Carve {
  char* base = nullptr;
  size_t cap = 0, off = 0;
  cudaStream_t st = nullptr;
  int64_t h2d = 0;                   // bytes uploaded
  cudaError_t err = cudaSuccess;     // sticky: the first take that did not fit or the first failed copy
  template <class T>
  T* take(size_t n) {
    const size_t bytes = (n * sizeof(T) + 255) & ~size_t(255);
    T* p = nullptr;
    if (base && off + bytes <= cap) p = reinterpret_cast<T*>(base + off);
    else if (base && err == cudaSuccess) err = cudaErrorMemoryAllocation;
    off += bytes;
    return p;
  }
  template <class T>
  void copy(T* dev, const T* host, size_t n) {
    if (!dev || n == 0 || err != cudaSuccess) return;
    err = host ? cudaMemcpyAsync(dev, host, n * sizeof(T), cudaMemcpyHostToDevice, st) : cudaErrorInvalidValue;
    h2d += (int64_t)(n * sizeof(T));
  }
  // a host column: null stays null (no take), an empty one gets one element
  template <class T>
  T* up(const T* host, size_t n) {
    if (!host) return nullptr;
    T* d = take<T>(n ? n : 1);
    copy(d, host, n);
    return d;
  }
  // a[0, na) followed by b[0, nb), and one spare element
  template <class T>
  T* cat(const T* a, size_t na, const T* b, size_t nb) {
    T* d = take<T>(na + nb + 1);
    copy(d, a, na);
    if (d) copy(d + na, b, nb);
    return d;
  }
  // cap_n elements that start with host[0, n).  `zero`: all cap_n are zeroed first, and a null host
  // leaves them so.
  template <class T>
  T* part(const T* host, size_t n, size_t cap_n, bool zero = false) {
    T* d = take<T>(cap_n);
    if (zero && d && err == cudaSuccess) err = cudaMemsetAsync(d, 0, cap_n * sizeof(T), st);
    if (host || !zero) copy(d, host, n);
    return d;
  }
};

// Carves one call's buffers from `a`.  body(Carve&) lists them once and runs twice: measuring, with no
// CUDA call, then (after the arena is grown to the measured size) carving.  Both runs make the same takes
// in the same order, so the arena is sized by the list it is carved by; the body therefore branches on
// host data only.  `start` (if any) is recorded on st once the arena is large enough, before the first
// upload.  Adds the uploaded bytes to *h2d (if given).
template <class Body>
inline cudaError_t carve(Arena& a, cudaStream_t st, cudaEvent_t start, int64_t* h2d, const Body& body) {
  Carve m;
  body(m);
  cudaError_t e = a.reserve(m.off);
  if (e == cudaSuccess && start) e = cudaEventRecord(start, st);
  if (e != cudaSuccess) return e;
  Carve c;
  c.base = a.base; c.cap = a.cap; c.st = st;
  body(c);
  if (h2d) *h2d += c.h2d;
  return c.err;
}

// A device-to-host copy on st whose bytes count towards *d2h.
template <class T>
inline cudaError_t download(T* host, const T* dev, size_t n, cudaStream_t st, int64_t* d2h) {
  *d2h += (int64_t)(n * sizeof(T));
  return cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, st);
}

struct cook_pool {
  cook_ctx* ctx = nullptr;
  std::string name;
  int dru_mode = 0;
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[24] = {};
  cook_phase_stats phase[8] = {};        // last rank / match / rebalance / exchange / state-apply / usage / cotasks /
                                         // considerable call
  double* xchg = nullptr;                // exchange buffers: [n_pad] local + [world * n_pad] gathered
  size_t xchg_cap = 0;
  Arena arena;
  void* match_plan = nullptr;            // MatchPlan (match.cu), resident inputs
  void (*match_plan_free)(void*) = nullptr;
  void* state = nullptr;                 // PoolState (state.cu), the resident job and task tables
  void (*state_free)(void*) = nullptr;
  char err[512] = {0};
};

// ---- the inputs of rank and match on the device, uploaded from host tables or gathered from the resident
// state (state.cu)
// Rank's task columns: running tasks [0, R) then pending jobs [R, R + J).
struct TaskCols {
  const int32_t* user;
  const int32_t* prio;
  const int64_t* start;
  const int64_t* tid;
  const int64_t* jid;
  const double* cpus;
  const double* mem;
  const double* gpus;
};

// The match's job columns in job index space (null: absent).
struct JobDev {
  const int32_t* user;
  const double* cpus;
  const double* mem;
  const double* gpus;
  const int32_t* ports;
  const uint8_t* allowed;
  const uint8_t* plugin;
  const int32_t* novel_off; const int32_t* novel_host;
  const int32_t* gpu_model;
  const double* disk_request; const int32_t* disk_type;
  const int32_t* attr_off; const int32_t* attr_col; const int32_t* attr_val;
  const int64_t* est_end_ms;
  const int32_t* ckpt_location;
  const int32_t* reserved_host;
  const int32_t* group_off; const int32_t* group_idx;
};

// Rank and match only read their device columns, so they hold them as const.  The gathers of the resident
// state are what fills columns carved for them, and write through this.
template <class T>
__host__ __device__ inline T* writable(const T* p) { return const_cast<T*>(p); }

// rank.cu: cook_rank over R running tasks and J pending jobs, from the host tables `running` and `pending`
// or from task columns already on the device (`dev`).  out_ranked_idx may be null (not downloaded).
// *queue (if given) receives the ranked pending indices on the device and their device count; they live in
// the pool's arena until it is carved again.
struct RankQueue {
  const int32_t* ranked;
  const int32_t* n;
};
// `offensive` (if given): the pending jobs that survive the quota filters and are offensive, in rank order, as job
// ids jid[pslot[pending index]] into the host's out[<= J], their number in *out_n (downloaded with the counts).
struct RankOffensive {
  const int32_t* pslot;
  const int64_t* jid;
  int64_t* out;
  int32_t* out_n;
};
int32_t rank_impl(cook_pool* pool, int R, int J, const cook_tasks_soa* running, const cook_tasks_soa* pending,
                  const TaskCols* dev, const cook_user_table* users, const cook_pool_quota* pool_quota,
                  const cook_pool_quota* group_quota, const double* group_usage, const cook_rank_params* params,
                  int32_t* out_ranked_idx, int32_t* out_n, double* out_dru, int32_t* out_order, int32_t* out_order_n,
                  RankQueue* queue, const RankOffensive* offensive = nullptr);

// The running-side inputs of a match or rebalance that the resident state derives on the device after the build:
// carved, not uploaded.  usage: the users' usage_* as one [4][n_users] block (count, cpus, mem, gpus); run: the
// offers' run_cpus, run_mem and run_count; cot: the groups' cot_* lists, sized for n_cot entries (carved where
// the plan reads the lists).
struct Derived {
  bool usage = false, run = false, cot = false;
  int64_t n_cot = 0;
};

// match.cu: what a match's plan needs to know about its jobs before it carves their columns.
struct JobShape {
  int J = 0;                      // job rows
  JobDev cols = {};               // the columns to carve (null: absent): host columns to upload when
                                  // `upload`, else the resident columns the caller gathers them from
  bool upload = false;
  int64_t n_novel = 0, n_attr = 0, n_group = 0;   // entries of each CSR list
  std::vector<int32_t> gp_off;    // [n_groups + 1] per-group member capacity offsets (empty: no groups)
  bool any_gpus_ports = false;    // some job asks for gpus or ports
  bool job_ids = false;           // carve a job id per row, and report the considerable jobs by job id
  Derived dev;                    // the users', offers' and groups' columns the caller fills on the device
};
// The carved rows of a plan whose columns the caller writes: row d is ranked[d] = d.
// The columns of shape.dev, null where not carved: usage [4][n_users]; run_* [offers->n] by input index;
// cot_off [n_groups + 1], cot_host / cot_attr [max(1, n_cot)].  What a derivation reads from the plan's uploads:
// the offers' hostname codes, their [n_attr_cols][offers->n] attribute matrix and the groups' attr_col (each
// null when not uploaded).
struct MatchRows {
  JobDev jb;
  int32_t* ranked;
  int64_t* job_id;
  double* usage;
  double* run_cpus; double* run_mem; int32_t* run_count;
  int32_t* cot_off; int32_t* cot_host; int32_t* cot_attr;
  const int32_t* hostname_id; const int32_t* attr; const int32_t* gcol;
};
// The checks of a match's offers, groups, users, params and sizes, with `who` in the messages.  The offer
// and group tables are checked when `tables`; `novel` and `grouped`: some job has novel-host or group lists.
// `cot_derived`: the groups' cot_* lists are derived on the device, so they are not required.
int32_t check_match_inputs(cook_pool* pool, const char* who, const cook_offers_soa* offers, const cook_groups* groups,
                           const cook_user_table* users, const cook_match_params* params, int32_t max_ports,
                           bool tables, bool novel, bool grouped, bool cot_derived = false);
// The pool's match plan is built for n_ranked rows of the jobs `sh` describes (ranked_idx: uploaded, null:
// the caller writes *rows before the run), then run.  A failed build leaves no valid plan.
int32_t match_build(cook_pool* pool, const int32_t* ranked_idx, int32_t n_ranked, const JobShape& sh,
                    const cook_offers_soa* offers, const cook_groups* groups, const cook_user_table* users,
                    const cook_pool_quota* pool_quota, const cook_match_params* params, int32_t max_ports,
                    MatchRows* rows);
int32_t match_run(cook_pool* pool, int32_t* out_considerable, int64_t* out_job_id, int32_t* out_assign,
                  int32_t* out_ports, uint8_t* out_fail_reason, cook_match_stats* out_stats, bool uploaded, int max_ctas);

// match.cu: M0 (pending-jobs->considerable-jobs, filter-pending-jobs-for-quota) over n job rows already on the
// device, by cook_match's own launches: the per-user folds in the order `ranked` gives, the pool-quota fold over
// users 0 .. n_users - 1, the masks (null: not read), take num_considerable.  Quotas [4] and usage [4] are count,
// cpus, mem, gpus columns of n_users (a null usage column reads 0); tokens may be null.  Scratch: pos, tmp [n + 1],
// seg_s, seg_e [n_users + 1], keep [n + 1], gf.  out_row[k] receives the row of the k-th considerable job, *out_n
// (device) their number.
struct GridFlag;
struct ConsRows {
  int n = 0, n_users = 0;
  const int32_t* ranked = nullptr;
  const int32_t* user = nullptr;
  const double *cpus = nullptr, *mem = nullptr, *gpus = nullptr;
  const uint8_t *allowed = nullptr, *plugin = nullptr;
  const double* quota[4] = {};
  const double* usage[4] = {};
  const int32_t* tokens = nullptr;
  int enforce_rate_limit = 0;
  cook_pool_quota pool_q = {0, 0, 0, 0, 0};
  int num_considerable = 0;
  int32_t *pos = nullptr, *tmp = nullptr, *seg_s = nullptr, *seg_e = nullptr;
  uint8_t* keep = nullptr;
  GridFlag* gf = nullptr;
  int32_t* out_row = nullptr;
  int32_t* out_n = nullptr;
};
cudaError_t considerable_rows(const ConsRows& r, cudaStream_t st, int* launches);
// The [4][n_users] usage columns the last match on this handle read, from its plan; false when no plan is valid or
// it was built for another n_users.
bool match_last_usage(cook_pool* pool, int n_users, const double* (&usage)[4]);

// rebalance.cu: what a rebalance needs to know about its rows before it carves their columns.
struct RebShape {
  int R = 0, P = 0;                               // running tasks, pending jobs
  // host tables to upload (cook_rebalance); a null `running`: the caller writes the carved rows (RebRows)
  const cook_running_soa* running = nullptr;
  const cook_jobs_soa* pending = nullptr;
  const int64_t* job_id = nullptr;
  const int32_t* priority = nullptr;
  int64_t n_novel = 0, n_attr = 0, n_group = 0;   // caller-written rows: entries each list may hold (0: no list)
  Derived dev;                                    // caller-written rows: only .cot applies
};
// The carved rows a caller writes before the run: running task r < R (host: index into the host table) and
// pending job p < P, with the pending lists the shape asked for.
struct RebRows {
  TaskCols t;
  const int32_t* host;
  JobDev jb;
  const int64_t* jid;
  const int32_t* prio;
  const int32_t* hostname_id;   // the host table's codes, uploaded [hosts->n]
  const int32_t* attr;          // its [n_attr_cols][hosts->n] attribute matrix (null: none uploaded)
  const int32_t* gcol;          // the groups' attr_col, uploaded (null: none)
  int32_t* cot_off; int32_t* cot_host; int32_t* cot_attr;   // sh.dev.cot and the walk reads the lists, else null
};
struct RebPlan;
struct RebPlanFree { void operator()(RebPlan* p) const; };
using RebPlanPtr = std::unique_ptr<RebPlan, RebPlanFree>;
// The build carves (and uploads the host table, the users' rebalance columns and the groups); the run is
// cook_rebalance's own, with each victim reported as its task id (a synthetic victim, the task of the job
// decision e placed, as -1 - e) and each decision's job id.  The caller checks the inputs.
int32_t rebalance_build(cook_pool* pool, const RebShape& sh, const cook_host_table* hosts, const cook_groups* groups,
                        const cook_user_table* users, const cook_rebalance_params* prm, RebPlanPtr* plan,
                        RebRows* rows);
int32_t rebalance_run(cook_pool* pool, RebPlan& plan, cook_decision* out_decisions, int64_t* out_victim_tid,
                      int64_t* out_decision_jid, int32_t* out_n);

inline int32_t set_err(cook_pool* p, int32_t code, const char* fmt, ...) {
  if (p) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(p->err, sizeof(p->err), fmt, ap);
    va_end(ap);
  }
  return code;
}

#define CK(pool, call)                                                                    \
  do {                                                                                    \
    cudaError_t _e = (call);                                                              \
    if (_e != cudaSuccess)                                                                \
      return set_err(pool, _e == cudaErrorMemoryAllocation ? COOK_E_OOM : COOK_E_CUDA,   \
                     "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
  } while (0)

// Host-side range check of an index column: a bad index from the shim must come back as
// COOK_E_BADARG, not as an illegal-address fault that poisons the CUDA context of every pool.
inline bool idx_in_range(const int32_t* col, size_t n, int32_t lo, int32_t hi_excl) {
  if (!col) return true;
  for (size_t i = 0; i < n; i++)
    if (col[i] < lo || col[i] >= hi_excl) return false;
  return true;
}

inline float ev_ms(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  cudaEventElapsedTime(&ms, a, b);
  return ms;
}

// The statistics of the last call of `phase`: its upload, device and download stages lie between the
// events up .. dev .. d2h .. end (a null `up`: no upload stage).
inline void record_phase(cook_pool* p, int phase, cudaEvent_t up, cudaEvent_t dev, cudaEvent_t d2h, cudaEvent_t end,
                         int64_t h2d_bytes, int64_t d2h_bytes, int32_t launches) {
  p->phase[phase] = {up ? ev_ms(up, dev) : 0.0, ev_ms(dev, d2h), ev_ms(d2h, end), h2d_bytes, d2h_bytes, launches, 0};
}

// ---------------------------------------------------------------------------------------------
// Exact-grid fast path for the f64 running sums of the path (DRU prefix sums, quota filters).
// The reference folds left to right (`reductions`, `reduce +`); a left fold is a serial chain.
// When every addend is a multiple of 2^-10 and the total magnitude stays below 2^43, every partial
// sum of every subset is exactly representable in f64, so ANY association produces the same bits
// as the left fold - and a parallel scan is legal.  grid_check_kernel establishes that per call on
// the device (no host round trip); the kernels take the scan path when it holds and keep the
// serial, association-preserving chain otherwise (e.g. cpus = 0.1).  Datomic amounts in Cook are
// MiB integers and cpus in halves in practice, so the fast path is the common one.
struct GridFlag {
  int bad;                      // != 0: some addend is off the 2^-10 grid (or not finite / too large)
  unsigned long long max_bits;  // bit pattern of the largest |addend| (non-negative doubles order like their bits)
};
#ifdef __CUDACC__
__device__ __forceinline__ bool grid_value_ok(double x) {
  const double y = x * 1024.0;
  return x >= 0.0 && x <= 1099511627776.0 && y == rint(y);
}
static __global__ void grid_check_kernel(const double* a, const double* b, const double* c, int n, GridFlag* f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool bad = false;
  double m = 0.0;
  if (i < n) {
    const double x = a ? a[i] : 0.0, y = b ? b[i] : 0.0, z = c ? c[i] : 0.0;
    bad = !(grid_value_ok(x) && grid_value_ok(y) && grid_value_ok(z));
    m = fmax(x, fmax(y, z));
  }
  const unsigned anyb = __ballot_sync(0xffffffffu, bad);
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) {
    if (anyb) atomicOr(&f->bad, 1);
    if (m > 0.0) atomicMax(&f->max_bits, (unsigned long long)__double_as_longlong(m));
  }
}
// the sums of `n` addends (plus a start value) are association-free
__device__ __forceinline__ bool grid_exact(const GridFlag* f, long long n, double start = 0.0) {
  if (!f || f->bad) return false;
  const double m = __longlong_as_double((long long)f->max_bits);
  return grid_value_ok(start) && ((double)(n + 1) * fmax(m, 1.0) + start) < 8796093022208.0;   // 2^43
}
template <class T>
__device__ __forceinline__ T warp_incl_scan(T x, const int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x = x + y;
  }
  return x;
}
#endif
