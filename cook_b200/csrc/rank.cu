// rank.cu — DRU fair-share ranking on the GPU (SURVEY §8a R1-R7).
//
// Replaces sort-jobs-by-dru-helper (scheduler/scheduler.clj:2073-2091),
// limit-over-quota-jobs (:2057-2071), dru/compute-task-scored-task-pairs
// (dru.clj:50-80), dru/sorted-merge (dru.clj:82-104), filter-based-on-quota
// (scheduler.clj:2134-2157) and filter-offensive-jobs (:2198-2229).
//
// Pipeline (all on the pool's stream, no host round trips):
//   K1 comparator sort by (user name rank, -priority, start, task id,
//      job id)                      -> per-user segments in tools.clj:614-641 order
//   K2 segment bounds
//   K3 warp-per-user fold           -> cumulative usage in the reference's
//      left-fold order (lane-serial shuffle chain keeps f64 association),
//      over-quota truncation, DRU = max(mem/div, cpus/div) (IEEE div.rn.f64)
//   K4 comparator sort of positions by (dru, k-way-merge tie rule); K3 wrote
//      each kept task's run of equal scores for it (merge_tie_word)
//   K5 single-warp queue filter     -> pending only, pool quota, group quota,
//      offensive filter, stable compaction.
#include "fold.cuh"
#include "sort.cuh"

namespace {

__global__ void scatter_dru_kernel(const int32_t* __restrict__ idx, const double* __restrict__ dru_at,
                                   int n, double* __restrict__ dru_task) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) dru_task[idx[p]] = dru_at[p];
}

struct UserCols {
  const double *div_mem, *div_cpus, *div_gpus;
  const double *q_count, *q_cpus, *q_mem, *q_gpus;
};

// K3: one warp per user, the running sums in the reference's left-fold order
// (fold.cuh): acc = ((acc + x0) + x1) + ... exactly as `reductions` does.
__global__ void __launch_bounds__(128) user_fold_kernel(
    const int32_t* __restrict__ idx, TaskCols t, UserCols uc, const int32_t* __restrict__ seg_start,
    const int32_t* __restrict__ seg_end, const int32_t* __restrict__ name_rank, int n_users, int dru_mode,
    int max_over_quota, double* __restrict__ dru_at, int64_t* __restrict__ tie, int32_t* n_kept_total,
    const GridFlag* gf, int n_scan) {
  if (n_scan > 0 && grid_exact(gf, n_scan)) return;   // the order-wide scans below did it
  __shared__ double stage[4][3][32];
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n_users) return;
  const int u = warp;
  const int s = seg_start[u], e = seg_end[u];
  if (e <= s) return;
  const double md = uc.div_mem[u], cd = uc.div_cpus[u], gd = uc.div_gpus[u];
  const double qn = uc.q_count[u], qc = uc.q_cpus[u], qm = uc.q_mem[u], qg = uc.q_gpus[u];
  const bool exact = grid_exact(gf, e - s);
  double acc[3] = {0.0, 0.0, 0.0};   // mem, cpus, gpus
  int over = 0;
  bool cut = false;
  int kept = 0;
  const double NaN = __longlong_as_double(0x7ff8000000000000LL);
  for (int base0 = s; base0 < e; base0 += 128) {
    // the gathers (idx -> amounts) are what a long segment waits for: four chunks in flight
    double x4[4][3];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int p = base0 + 32 * q + lane;
      x4[q][0] = x4[q][1] = x4[q][2] = 0.0;
      if (p < e) { const int ti = idx[p]; x4[q][0] = t.mem[ti]; x4[q][1] = t.cpus[ti]; x4[q][2] = t.gpus[ti]; }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int base = base0 + 32 * q;
      if (base >= e) break;
      const int p = base + lane;
      warp_fold_prefix(x4[q], acc, min(32, e - base), exact, stage[threadIdx.x >> 5]);
      const double mym = x4[q][0], myc = x4[q][1], myg = x4[q][2];
      // scheduler.clj:2057-2071: keep while #violating prefixes <= limit
      bool viol = false;
      if (p < e) {
        double cnt = (double)(p - s + 1);
        viol = !(cnt <= qn && myc <= qc && mym <= qm && myg <= qg);
      }
      unsigned vb = __ballot_sync(0xffffffffu, viol);
      int over_incl = over + __popc(vb & (0xffffffffu >> (31 - lane)));
      bool keep = (p < e) && !cut && (over_incl <= max_over_quota);
      double d = NaN;
      if (keep) {
        if (dru_mode == 0) {
          double a = mym / md, b = myc / cd;
          d = a > b ? a : b;
        } else {
          d = myg / gd;
        }
      }
      if (p < e) dru_at[p] = d;
      unsigned kb = __ballot_sync(0xffffffffu, keep);
      kept += __popc(kb);
      over += __popc(vb);
      if (over > max_over_quota) cut = true;  // later batches are all beyond the cut
    }
  }
  // the merge comparator's word of every kept task, from the scores this warp just wrote
  __syncwarp();
  const int32_t nr = name_rank[u];
  for (int p = s + lane; p < s + kept; p += 32)
    tie[p] = merge_tie_word(p, s, u, nr, dru_at[p], [&](int m) { return dru_at[m]; });
  if (lane == 0 && kept) atomicAdd(n_kept_total, kept);
}

// K3 for exact-grid amounts (fold.cuh: any association gives the left fold's bits): the per-user
// running sums are the order-wide scan of the amounts, the over-quota count is a second one over the
// violation flags.  No user, however long its list, sits on one warp.  Five launches: the two scans,
// the finish (keep / dru / kept count).
struct RankScan {
  const int32_t* user_at; const int32_t* seg_start; const int32_t* name_rank; UserCols uc;
  OrderScan<double, 3> amt;   // mem, cpus, gpus
  OrderScan<int, 1> viol;     // violating prefixes
  int n, dru_mode, max_over_quota;
  double* dru_at; int64_t* tie; int32_t* n_kept_total;
  // the score of kept position p of user u, whose list starts at s
  __device__ double score(int p, int s, int u) const {
    if (dru_mode == 0) {
      const double x = amt.segment_sum(0, p, s) / uc.div_mem[u], y = amt.segment_sum(1, p, s) / uc.div_cpus[u];
      return x > y ? x : y;
    }
    return amt.segment_sum(2, p, s) / uc.div_gpus[u];
  }
  // scheduler.clj:2057-2071: a prefix violates when (count, cpus, mem, gpus) is not within the quota
  __device__ void operator()(int p, int (&v)[1]) const {
    const int u = user_at[p], s = seg_start[u];
    const double cnt = (double)(p - s + 1);
    v[0] = !(cnt <= uc.q_count[u] && amt.segment_sum(1, p, s) <= uc.q_cpus[u] && amt.segment_sum(0, p, s) <= uc.q_mem[u] &&
             amt.segment_sum(2, p, s) <= uc.q_gpus[u]) ? 1 : 0;
  }
};

struct LoadAmounts {
  const int32_t* idx; TaskCols t;
  __device__ void operator()(int p, double (&x)[3]) const {
    const int ti = idx[p];
    x[0] = t.mem[ti]; x[1] = t.cpus[ti]; x[2] = t.gpus[ti];
  }
};

__global__ void __launch_bounds__(OS_TB) os_finish(RankScan a, const GridFlag* gf) {
  if (!grid_exact(gf, a.n)) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  bool keep = false;
  if (p < a.n) {
    const int u = a.user_at[p], s = a.seg_start[u];
    keep = a.viol.segment_sum(0, p, s) <= a.max_over_quota;
    double d = __longlong_as_double(0x7ff8000000000000LL);
    if (keep) {
      d = a.score(p, s, u);
      // the merge comparator's word: the scores before p are recomputed (same bits), not read back, since
      // other blocks write them.  A kept task's predecessors are kept.
      a.tie[p] = merge_tie_word(p, s, u, a.name_rank[u], d, [&](int m) { return a.score(m, s, u); });
    }
    a.dru_at[p] = d;
  }
  const int kept = __syncthreads_count(keep);
  if (threadIdx.x == 0 && kept) atomicAdd(a.n_kept_total, kept);
}

struct QueueFilterArgs {
  const int32_t* pos_sorted;  // positions (into user-sorted array) in merge order
  const int32_t* idx;         // sorted position -> combined task index
  const int32_t* n_kept;      // device: tasks that survived limit-over-quota-jobs
  int R;                      // running count (combined index >= R => pending)
  const double* cpus;         // combined columns
  const double* mem;
  const double* gpus;
  int filter_offensive;
  double off_mem, off_cpus;
  int32_t* out_order;         // combined task index per emitted task
  int32_t* out_ranked;        // pending indices surviving all filters
  int32_t* out_n;
  // queue-order scratch (one entry per emitted task)
  int32_t* ti_at;
  uint8_t* flag;              // pending job still in the queue after the filters so far
  double *xc, *xm, *xg;       // its request (0 for running tasks)
  int32_t* blk_cnt;           // per block of CP_BLOCK entries: survivors, then exclusive offsets
};

constexpr int QF_TB = 256;

// Σ running usage of the pool (scheduler.clj:2118-2123) in input order, on one warp.
__global__ void pool_usage_kernel(const double* cpus, const double* mem, const double* gpus, int R,
                                  double* out4, const GridFlag* gf) {
  __shared__ double stage[3][32];
  double acc[3] = {0.0, 0.0, 0.0};
  warp_fold_sum<3, 4>(acc, R, grid_exact(gf, R), [&](int i, double (&x)[3]) {
    x[0] = cpus[i]; x[1] = mem[i]; x[2] = gpus[i];
    return true;
  }, stage);
  if (threadIdx.x == 0) { out4[0] = (double)R; out4[1] = acc[0]; out4[2] = acc[1]; out4[3] = acc[2]; }
}

// K5 step 1: the merged order as task indices, with each pending job's request
// laid out in queue order so that the sequential filters below stream it.
__global__ void __launch_bounds__(QF_TB) qf_gather_kernel(QueueFilterArgs a) {
  const int i = blockIdx.x * QF_TB + threadIdx.x;
  if (i >= *a.n_kept) return;
  const int ti = a.idx[a.pos_sorted[i]];
  if (a.out_order) a.out_order[i] = ti;
  const bool pend = ti >= a.R;
  a.ti_at[i] = ti;
  a.flag[i] = pend;
  a.xc[i] = pend ? a.cpus[ti] : 0.0;
  a.xm[i] = pend ? a.mem[ti] : 0.0;
  a.xg[i] = pend ? a.gpus[ti] : 0.0;
}

// K5 step 2, once per enabled quota (pool, then quota group): tools.clj:654-668
// filter-sequential -- the usage advances for every job that reaches the filter,
// kept or not, in queue order, with the reference's left-fold association.  The
// four running sums are four independent serial chains: one thread each over a
// chunk staged in shared memory (a job that did not reach the filter adds 0.0,
// which leaves a sum unchanged); everything else is parallel.
constexpr int QF_CH = 1024;
__global__ void __launch_bounds__(QF_CH) qf_quota_kernel(QueueFilterArgs a, cook_pool_quota q,
                                                         const double* usage4, const GridFlag* gf) {
  __shared__ double s[4][QF_CH];
  const int tid = threadIdx.x, n = *a.n_kept;
  const int chain = tid >> 5;                       // chain k runs on lane 0 of warp k
  if (grid_exact(gf, n, fmax(fmax(usage4[0], usage4[1]), fmax(usage4[2], usage4[3]))) &&
      grid_value_ok(usage4[0]) && grid_value_ok(usage4[1]) && grid_value_ok(usage4[2]) && grid_value_ok(usage4[3])) {
    // every partial sum is exact: block-wide parallel scan of the four running sums, carried chunk to chunk
    __shared__ double wsum[4][32];
    const int lane = tid & 31, w = tid >> 5;
    double carry[4] = {usage4[0], usage4[1], usage4[2], usage4[3]};
    for (int base = 0; base < n; base += QF_CH) {
      const int i = base + tid;
      const bool f = i < n && a.flag[i];
      double x[4] = {f ? 1.0 : 0.0, f ? a.xc[i] : 0.0, f ? a.xm[i] : 0.0, f ? a.xg[i] : 0.0};
#pragma unroll
      for (int k = 0; k < 4; k++) { x[k] = warp_incl_scan(x[k], lane); if (lane == 31) wsum[k][w] = x[k]; }
      __syncthreads();
      if (w < 4) { const double t = warp_incl_scan(wsum[w][lane], lane); wsum[w][lane] = t; }
      __syncthreads();
      bool ok = true;
#pragma unroll
      for (int k = 0; k < 4; k++) x[k] = carry[k] + ((w ? wsum[k][w - 1] : 0.0) + x[k]);
      ok = x[0] <= q.count && x[1] <= q.cpus && x[2] <= q.mem && x[3] <= q.gpus;
      if (f && !ok) a.flag[i] = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) carry[k] = carry[k] + wsum[k][31];
      __syncthreads();
    }
    return;
  }
  double acc = (tid & 31) == 0 && chain < 4 ? usage4[chain] : 0.0;
  for (int base = 0; base < n; base += QF_CH) {
    const int i = base + tid, cnt = min(QF_CH, n - base);
    bool f = false;
    if (i < n) {
      f = a.flag[i];
      s[0][tid] = f ? 1.0 : 0.0;
      s[1][tid] = f ? a.xc[i] : 0.0;
      s[2][tid] = f ? a.xm[i] : 0.0;
      s[3][tid] = f ? a.xg[i] : 0.0;
    }
    __syncthreads();
    if ((tid & 31) == 0 && chain < 4) {
      double* row = s[chain];
#pragma unroll 8
      for (int j = 0; j < cnt; j++) { acc = acc + row[j]; row[j] = acc; }
    }
    __syncthreads();
    if (f && !(s[0][tid] <= q.count && s[1][tid] <= q.cpus && s[2][tid] <= q.mem && s[3][tid] <= q.gpus))
      a.flag[i] = 0;
    __syncthreads();
  }
}

// K5 step 3: offensive-job filter (scheduler.clj:2198-2229) and order-preserving
// compaction of the survivors.
struct QueueSurvivors {
  QueueFilterArgs a;
  __device__ bool keep(int i) const {
    return a.flag[i] && !(a.filter_offensive && (a.xm[i] > a.off_mem || a.xc[i] > a.off_cpus));
  }
  __device__ void emit(int i, int slot) const { a.out_ranked[slot] = a.ti_at[i] - a.R; }
};

// The jobs filter-offensive-jobs puts on its channel: past the quota filters and offensive, in rank order, as job
// ids (dense pending index -> slot -> job id).
struct QueueOffensive {
  QueueFilterArgs a; const int32_t* pslot; const int64_t* jid; int64_t* out;
  __device__ bool keep(int i) const { return a.flag[i] && (a.xm[i] > a.off_mem || a.xc[i] > a.off_cpus); }
  __device__ void emit(int i, int slot) const { out[slot] = jid[pslot[a.ti_at[i] - a.R]]; }
};

}  // namespace

extern "C" int32_t cook_rank(cook_pool* pool, const cook_tasks_soa* running,
                             const cook_tasks_soa* pending, const cook_user_table* users,
                             const cook_pool_quota* pool_quota, const cook_pool_quota* group_quota,
                             const double* group_usage, const cook_rank_params* params,
                             int32_t* out_ranked_idx, int32_t* out_n, double* out_dru,
                             int32_t* out_order, int32_t* out_order_n) {
  if (!pool) return COOK_E_BADARG;
  if (!running || !pending || !out_ranked_idx) return set_err(pool, COOK_E_BADARG, "cook_rank: null argument");
  return rank_impl(pool, running->n, pending->n, running, pending, nullptr, users, pool_quota, group_quota, group_usage,
                   params, out_ranked_idx, out_n, out_dru, out_order, out_order_n, nullptr);
}

int32_t rank_impl(cook_pool* pool, int R, int J, const cook_tasks_soa* running, const cook_tasks_soa* pending,
                  const TaskCols* dev, const cook_user_table* users, const cook_pool_quota* pool_quota,
                  const cook_pool_quota* group_quota, const double* group_usage, const cook_rank_params* params,
                  int32_t* out_ranked_idx, int32_t* out_n, double* out_dru, int32_t* out_order, int32_t* out_order_n,
                  RankQueue* queue, const RankOffensive* offensive, const double* d_pool_usage) {
  if (!users || !params || !out_n) return set_err(pool, COOK_E_BADARG, "cook_rank: null argument");
  const int N = R + J, U = users->n_users;
  if (R < 0 || J < 0 || U <= 0) return set_err(pool, COOK_E_BADARG, "cook_rank: bad sizes");
  // device rows had their user codes checked when they entered (state.cu)
  if (!dev && (!idx_in_range(running->user, R, 0, U) || !idx_in_range(pending->user, J, 0, U)))
    return set_err(pool, COOK_E_BADARG, "cook_rank: task user index out of range");
  *out_n = 0;
  if (out_order_n) *out_order_n = 0;
  if (offensive) *offensive->out_n = 0;
  if (N == 0) return COOK_OK;
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  TaskCols t;
  UserCols uc;
  const int32_t* d_name_rank;
  int32_t *d_idx, *d_tmp, *d_user_at, *d_pos, *d_out_order, *d_out_ranked, *d_seg_start, *d_seg_end, *d_counters;
  int64_t* d_tie;
  int32_t *d_os_pv, *d_os_bv;
  double *d_dru_at, *d_quota_usage, *d_dru_task, *d_os_pm, *d_os_pc, *d_os_pg, *d_os_b;
  GridFlag* d_gf;
  QueueFilterArgs qa;
  int64_t* d_off = nullptr;
  const int os_nb = (N + OS_TILE - 1) / OS_TILE;
  int64_t h2d = 0, d2h = 0;
  const cudaError_t carved = carve(pool->arena, st, pool->ev[8], &h2d, [&](Carve& c) {
    if (dev) {
      t = *dev;
    } else {
      t.user = c.cat(running->user, R, pending->user, J);
      t.prio = c.cat(running->priority, R, pending->priority, J);
      t.start = c.cat(running->start_time, R, pending->start_time, J);
      t.tid = c.cat(running->task_id, R, pending->task_id, J);
      t.jid = c.cat(running->job_id, R, pending->job_id, J);
      t.cpus = c.cat(running->cpus, R, pending->cpus, J);
      t.mem = c.cat(running->mem, R, pending->mem, J);
      t.gpus = c.cat(running->gpus, R, pending->gpus, J);
    }
    d_name_rank = c.up(users->name_rank, U);
    uc.div_mem = c.up(users->div_mem, U); uc.div_cpus = c.up(users->div_cpus, U); uc.div_gpus = c.up(users->div_gpus, U);
    uc.q_count = c.up(users->quota_count, U); uc.q_cpus = c.up(users->quota_cpus, U);
    uc.q_mem = c.up(users->quota_mem, U); uc.q_gpus = c.up(users->quota_gpus, U);
    d_idx = c.take<int32_t>(N + 1);
    d_tmp = c.take<int32_t>(N + 1);
    d_user_at = c.take<int32_t>(N + 1);
    d_pos = c.take<int32_t>(N + 1);
    d_out_order = c.take<int32_t>(N + 1);
    d_out_ranked = c.take<int32_t>(N + 1);
    d_dru_at = c.take<double>(N + 1);
    d_tie = c.take<int64_t>(N + 1);
    d_seg_start = c.take<int32_t>(U);
    d_seg_end = c.take<int32_t>(U);
    d_quota_usage = c.take<double>(8);   // [0, 4): the pool's running usage (unless given), [4, 8): the group's
    d_counters = c.take<int32_t>(8);  // [0]=n_kept [1]=n_out
    d_dru_task = c.take<double>(N + 1);
    d_gf = c.take<GridFlag>(1);
    d_os_pm = c.take<double>(N + 1); d_os_pc = c.take<double>(N + 1); d_os_pg = c.take<double>(N + 1);
    d_os_b = c.take<double>(3 * (os_nb + 1));
    d_os_pv = c.take<int32_t>(N + 1); d_os_bv = c.take<int32_t>(os_nb + 1);
    qa.ti_at = c.take<int32_t>(N + 1); qa.flag = c.take<uint8_t>(N + 1);
    qa.xc = c.take<double>(N + 1); qa.xm = c.take<double>(N + 1); qa.xg = c.take<double>(N + 1);
    qa.blk_cnt = c.take<int32_t>(N / CP_BLOCK + 2);
    if (offensive) d_off = c.take<int64_t>(J + 1);
  });
  CK(pool, carved);
  CK(pool, cudaMemsetAsync(d_gf, 0, sizeof(GridFlag), st));
  CK(pool, cudaMemsetAsync(d_seg_start, 0, sizeof(int32_t) * U, st));
  CK(pool, cudaMemsetAsync(d_seg_end, 0, sizeof(int32_t) * U, st));
  CK(pool, cudaMemsetAsync(d_counters, 0, sizeof(int32_t) * 8, st));

  CK(pool, cudaEventRecord(pool->ev[9], st));
  int nl = 0;
  const int TB = 256, nb = (N + TB - 1) / TB;
  grid_check_kernel<<<nb, TB, 0, st>>>(t.cpus, t.mem, t.gpus, N, d_gf);
  nl++;
  CK(pool, csort::sort_indices(d_idx, d_tmp, N, LessUserTask{t.user, t.prio, t.start, t.tid, t.jid, d_name_rank}, st, &nl));
  seg_bounds_kernel<<<nb, TB, 0, st>>>(SortedKey{d_idx, nullptr, t.user}, N, d_seg_start, d_seg_end, d_user_at);
  nl++;
  {
    RankScan os;
    os.user_at = d_user_at; os.seg_start = d_seg_start; os.name_rank = d_name_rank; os.uc = uc;
    os.amt = OrderScan<double, 3>{{d_os_pm, d_os_pc, d_os_pg}, {d_os_b, d_os_b + os_nb + 1, d_os_b + 2 * (os_nb + 1)}};
    os.viol = OrderScan<int, 1>{{d_os_pv}, {d_os_bv}};
    os.n = N; os.dru_mode = pool->dru_mode; os.max_over_quota = params->max_over_quota_jobs;
    os.dru_at = d_dru_at; os.tie = d_tie; os.n_kept_total = d_counters;
    order_scan(os.amt, LoadAmounts{d_idx, t}, N, d_gf, st, &nl);
    order_scan(os.viol, os, N, d_gf, st, &nl);
    os_finish<<<(N + OS_TB - 1) / OS_TB, OS_TB, 0, st>>>(os, d_gf);
    int warps_per_block = 4;
    int blocks = (U + warps_per_block - 1) / warps_per_block;
    user_fold_kernel<<<blocks, warps_per_block * 32, 0, st>>>(
        d_idx, t, uc, d_seg_start, d_seg_end, d_name_rank, U, pool->dru_mode, params->max_over_quota_jobs,
        d_dru_at, d_tie, d_counters, d_gf, N);
    nl += 2;
  }
  CK(pool, csort::sort_indices(d_pos, d_tmp, N, LessMerge{d_dru_at, d_tie}, st, &nl));
  qa.pos_sorted = d_pos; qa.idx = d_idx; qa.n_kept = d_counters; qa.R = R;
  qa.cpus = t.cpus; qa.mem = t.mem; qa.gpus = t.gpus;
  qa.filter_offensive = params->filter_offensive;
  qa.off_mem = params->offensive_max_mem_mb; qa.off_cpus = params->offensive_max_cpus;
  qa.out_order = d_out_order; qa.out_ranked = d_out_ranked; qa.out_n = d_counters + 1;
  const int qnb = (N + QF_TB - 1) / QF_TB;
  qf_gather_kernel<<<qnb, QF_TB, 0, st>>>(qa);
  nl++;
  if (pool_quota && pool_quota->enabled) {
    if (!d_pool_usage) {
      pool_usage_kernel<<<1, 32, 0, st>>>(t.cpus, t.mem, t.gpus, R, d_quota_usage, d_gf);
      nl++;
    }
    qf_quota_kernel<<<1, QF_CH, 0, st>>>(qa, *pool_quota, d_pool_usage ? d_pool_usage : d_quota_usage, d_gf);
    nl++;
  }
  if (group_quota && group_usage && group_quota->enabled) {
    CK(pool, cudaMemcpyAsync(d_quota_usage + 4, group_usage, sizeof(double) * 4, cudaMemcpyHostToDevice, st));
    qf_quota_kernel<<<1, QF_CH, 0, st>>>(qa, *group_quota, d_quota_usage + 4, d_gf);
    nl++;
  }
  // at most J survivors: the caller's out_ranked_idx holds J, so no order can make the download overrun it
  compact(QueueSurvivors{qa}, N, qa.n_kept, qa.blk_cnt, qa.out_n, J, st, &nl);
  // the queue's compaction is done with blk_cnt: the offensive one reuses it (nothing is offensive when the filter
  // is off, and the count stays 0)
  if (offensive && params->filter_offensive)
    compact(QueueOffensive{qa, offensive->pslot, offensive->jid, d_off}, N, qa.n_kept, qa.blk_cnt, d_counters + 2, J,
            st, &nl);
  if (out_dru) {
    scatter_dru_kernel<<<nb, TB, 0, st>>>(d_idx, d_dru_at, N, d_dru_task);
    nl++;
  }
  CK(pool, cudaGetLastError());
  if (queue) *queue = RankQueue{d_out_ranked, qa.out_n};
  CK(pool, cudaEventRecord(pool->ev[10], st));
  int32_t h_counters[3] = {0, 0, 0};   // [2]: offensive jobs
  CK(pool, download(h_counters, d_counters, offensive ? 3 : 2, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  const int32_t n_kept = h_counters[0], n_out = h_counters[1];
  if (n_out > 0 && out_ranked_idx) CK(pool, download(out_ranked_idx, d_out_ranked, n_out, st, &d2h));
  if (offensive) {
    *offensive->out_n = h_counters[2];
    if (h_counters[2] > 0) CK(pool, download(offensive->out, d_off, h_counters[2], st, &d2h));
  }
  if (out_order && n_kept > 0) CK(pool, download(out_order, d_out_order, n_kept, st, &d2h));
  if (out_dru) CK(pool, download(out_dru, d_dru_task, N, st, &d2h));
  CK(pool, cudaEventRecord(pool->ev[11], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_RANK, pool->ev[8], pool->ev[9], pool->ev[10], pool->ev[11], h2d, d2h, nl);
  *out_n = n_out;
  if (out_order_n) *out_order_n = n_kept;
  return COOK_OK;
}
