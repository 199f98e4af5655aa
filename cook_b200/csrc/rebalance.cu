// rebalance.cu — rebalancer preemption-victim search on the GPU (SURVEY §8a B1-B6).
//
// Replaces init-state (rebalancer.clj:222-266), compute-pending-default-job-dru
// (:182-208), compute-preemption-decision (:320-407), next-state (:270-309) and
// the rebalance loop (:434-467).  Decisions are inherently sequential (H6); the
// work INSIDE a decision is data-parallel over the running tasks and hosts, and
// the state is kept incrementally between decisions:
//
//   once:
//     S1 comparator sort of the tasks by (user name, -priority, start, task id,
//        job id)                                  -> per-user order (tools.clj:614-641)
//     S2 warp-per-user left fold                  -> cumulative sums + DRU (dru.clj:50-66)
//     S3 tasks grouped by host (a task never changes host)
//   per pending job, inside ONE persistent cooperative kernel (no host round trip):
//     P1 32-ary search for the nearest task (+ the quota fold when a quota can bind)
//                                                 -> job-below-quota, pending dru
//     P2 constraints per host (:358-377)
//     P3 warp per host: [spare ; eligible victims by desc dru] prefix sums by
//        repeated warp selection of the next victim, best sufficient prefix (:380-403)
//     P4 argmax over hosts (max dru, ties -> greatest hostname = `max-key` last wins)
//     P5 next-state -- victims die in place (a dead task adds 0.0 to every
//        fold), the job's task is inserted into its user's order, and only the
//        users that changed are re-folded, from the first position that changed
//        (dru.clj:128-144 next-task->scored-task).
//
// GPU DRU mode is rejected: the reference itself throws there (see oracle).
#include <cooperative_groups.h>

#include <algorithm>

#include "constraints.cuh"
#include "fold.cuh"
#include "sort.cuh"

namespace {

struct RTasks {  // capacity R + max_preemption; synthetic tasks appended
  int32_t* user; int32_t* prio; int64_t* start; int64_t* tid; int64_t* jid;
  double* cpus; double* mem; double* gpus; int32_t* host; uint8_t* alive; double* dru;
  int32_t* pos;        // position inside the user's sorted list (dead tasks keep their slot)
  double* cm; double* cc;  // cumulative mem / cpus of the user up to and including this slot
};

struct LessHost {
  RTasks t;
  __device__ bool operator()(int32_t a, int32_t b) const {
    int ha = t.host[a], hb = t.host[b];
    if (ha != hb) return ha < hb;
    return a < b;
  }
};

// Users to re-fold after a decision, written by the kernel's next-state step.
struct Refold {
  int32_t n;
  int32_t q_ins;       // where the new task went into the user order
  int32_t pu;          // its user
  int32_t user[64];    // victims of one decision sit on one host; more than 63 distinct
  int32_t from[64];    //   users fall back to `all` (from = segment start)
  int32_t all;
  // for the element-wise re-fold (exact-grid amounts): the victims of the decision (user, slot in the
  // OLD order, amounts) and the running sums just before the new task
  int32_t n_vict;
  int32_t vu[64], vs[64];
  double vm[64], vc[64];
  double base_m, base_c;
};

// dru.clj:50-66: one warp per user, the running sums in the reference's left-fold order (fold.cuh).
__global__ void __launch_bounds__(128) user_dru_kernel(const int32_t* ord, RTasks t, const double* div_mem,
                                                       const double* div_cpus, const int32_t* seg_start,
                                                       const int32_t* seg_end, int n_users, const GridFlag* gf,
                                                       int n_scan) {
  if (n_scan > 0 && grid_exact(gf, n_scan)) return;   // the order-wide scan below does it
  const int u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (u >= n_users) return;
  const int s = seg_start[u], e = seg_end[u];
  if (e <= s) return;
  __shared__ double stage[4][2][32];
  const double md = div_mem[u], cd = div_cpus[u];
  double acc[2] = {0.0, 0.0};   // mem, cpus
  const bool exact = grid_exact(gf, e - s);
  for (int base = s; base < e; base += 32) {
    int p = base + lane;
    int i = p < e ? ord[p] : -1;
    const bool live = i >= 0 && t.alive[i];
    double x[2] = {live ? t.mem[i] : 0.0, live ? t.cpus[i] : 0.0};
    warp_fold_prefix(x, acc, min(32, e - base), exact, stage[threadIdx.x >> 5]);
    if (i >= 0) {
      t.cm[i] = x[0]; t.cc[i] = x[1];
      double a = x[0] / md, b = x[1] / cd;
      t.dru[i] = a > b ? a : b;
      t.pos[i] = p - s;
    }
  }
}

// The same fold for exact-grid amounts: the order-wide scan (fold.cuh) of the live amounts.
struct LoadAlive {
  const int32_t* ord; RTasks t;
  __device__ void operator()(int p, double (&x)[2]) const {
    const int i = ord[p];
    if (t.alive[i]) { x[0] = t.mem[i]; x[1] = t.cpus[i]; }
  }
};

__global__ void order_dru_finish(const int32_t* ord, RTasks t, int n, const GridFlag* gf, OrderScan<double, 2> os,
                                 const int32_t* seg_start, const double* div_mem, const double* div_cpus) {
  if (!grid_exact(gf, n)) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int i = ord[p], u = t.user[i], s = seg_start[u];
  const double cm = os.segment_sum(0, p, s), cc = os.segment_sum(1, p, s);
  t.cm[i] = cm; t.cc[i] = cc;
  const double a = cm / div_mem[u], b = cc / div_cpus[u];
  t.dru[i] = a > b ? a : b;
  t.pos[i] = p - s;
}

struct HostCols {
  int H;
  const int32_t* hostname_id; const int32_t* name_rank;
  uint8_t* has_spare; double* spare_cpus; double* spare_mem; double* spare_gpus;
  const uint8_t* is_k8s; const int32_t* location;
  const int32_t* gpu_off; const int32_t* gpu_model; const double* gpu_count;
  const int32_t* disk_off; const int32_t* disk_type; const double* disk_space;
  const int64_t* host_start; int n_attr_cols; const int32_t* attr;
};

struct PendCols {
  const int32_t* user; const double* cpus; const double* mem; const double* gpus;
  const int64_t* jid; const int32_t* prio;
  const int32_t* novel_off; const int32_t* novel_host; const int32_t* gpu_model;
  const double* disk_request; const int32_t* disk_type;
  const int32_t* attr_off; const int32_t* attr_col; const int32_t* attr_val;
  const int64_t* est_end_ms; const int32_t* ckpt_location;
  const int32_t* group_off; const int32_t* group_idx;
};

struct GroupCols {
  int n; const int32_t* kind; const int32_t* attr_col; const int32_t* minimum;
  const int32_t* cot_off; const int32_t* cot_host; const int32_t* cot_attr;
};

struct PendScalars {  // per pending job, device resident
  int below_quota;
  double pending_dru;
};

__device__ __forceinline__ double csr_get(const int32_t* off, const int32_t* key, const double* val, int o, int k) {
  if (!off) return 0.0;
  for (int i = off[o]; i < off[o + 1]; i++)
    if (key[i] == k) return val[i];
  return 0.0;
}

// host has at least one live task? (preemptable-host->slave-id, :371-377)
__global__ void host_has_task_kernel(RTasks t, int n, uint8_t* has_task) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && t.alive[i]) has_task[t.host[i]] = 1;
}

struct HostBest {  // best sufficient prefix of one host
  double dru, mem, cpus, gpus;
  int32_t n_victims;  // -1: no candidate
};

// Priority-map order inside a host (:252-256, :349): (-dru, user name); equal
// (dru, user): later same-user position first (ours), then the lower index.
struct VKey {
  double dru; int32_t urank, pos, idx;   // idx < 0: none
};
__device__ __forceinline__ bool vkey_before(const VKey& a, const VKey& b) {
  if (b.idx < 0) return a.idx >= 0;
  if (a.idx < 0) return false;
  if (a.dru != b.dru) return a.dru > b.dru;
  if (a.urank != b.urank) return a.urank < b.urank;
  if (a.pos != b.pos) return a.pos > b.pos;
  return a.idx < b.idx;
}
__device__ __forceinline__ VKey vkey_shfl_xor(const VKey& k, int o) {
  VKey r;
  r.dru = __shfl_xor_sync(0xffffffffu, k.dru, o);
  r.urank = __shfl_xor_sync(0xffffffffu, k.urank, o);
  r.pos = __shfl_xor_sync(0xffffffffu, k.pos, o);
  r.idx = __shfl_xor_sync(0xffffffffu, k.idx, o);
  return r;
}

// One packed record per running task IN HOST ORDER (position q of hord): everything the host phase
// needs about a possible victim in three 128-bit loads, coalesced over the tasks of a host, instead
// of five dependent gathers through the task index.  dru / pos are refreshed by the re-fold, a
// victim's idx becomes -1.
struct __align__(16) TaskHot {
  double dru, mem, cpus, gpus;
  int32_t urank, pos, idx, user;   // idx < 0: dead
};

struct SelArgs {
  const TaskHot* hot;
  const int32_t* hord; const int32_t* hs; const int32_t* he;
  RTasks t; int R; int n_tasks;             // synthetic tasks are R .. n_tasks-1
  HostCols hc; PendCols pc; const int32_t* user_rank;
  const PendScalars* ps; double min_diff, safe;
  const int32_t* syn_cnt;   // per host: synthetic tasks (jobs placed by earlier decisions) living there
  const int32_t* syn_head;  // per host: newest synthetic task (-1: none); chained through syn_next[task]
  const int32_t* syn_next;
};

// P3 for one host, one warp: [spare ; victims by desc dru] prefix sums in the
// reference's left-fold order.  The next victim is chosen by a warp-wide argmax
// over the eligible tasks that come after the previous one; the first sufficient
// prefix has the highest dru of the host, longer prefixes with the SAME dru win
// the max-key tie (last wins).  With `emit` the first n_emit victims are written
// in ascending dru order (:397 conj onto a list).
__device__ HostBest host_select(const SelArgs& a, int p, int h, int lane, int32_t* emit, int n_emit) {
  HostBest b;
  b.dru = 0.0; b.mem = b.cpus = b.gpus = 0.0; b.n_victims = -1;
  const double pm = a.pc.mem[p], pcpu = a.pc.cpus[p], pg = a.pc.gpus ? a.pc.gpus[p] : 0.0;
  const int pu = a.pc.user[p];
  const bool below = a.ps->below_quota != 0;
  const double pend = a.ps->pending_dru;
  // the synthetic tasks are scanned only on the (few) hosts that hold one
  const int s0 = a.hs[h], seg = a.he[h] - s0, n_syn = a.syn_cnt[h], n_items = seg + (n_syn ? a.n_tasks - a.R : 0);
  if (seg + n_syn <= 64) {
    // FAST PATH (almost every host): at most two tasks per lane, loaded once from the packed records and
    // kept in registers over the sum pass and all selection rounds
    double idru[2], imem[2], icpu[2], igpu[2];
    int iur[2], ipos[2], iidx[2];
    bool iok[2];
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int k = lane + 32 * j;
      iok[j] = false; idru[j] = imem[j] = icpu[j] = igpu[j] = 0.0; iur[j] = ipos[j] = 0; iidx[j] = -1;
      if (k < seg + n_syn) {
        int q = s0 + k;
        if (k >= seg) {   // the (k - seg)-th synthetic task of the host: its record sits at its own index
          q = a.syn_head[h];
          for (int w = k - seg; w > 0; w--) q = a.syn_next[q];
        }
        const TaskHot r = a.hot[q];
        idru[j] = r.dru; imem[j] = r.mem; icpu[j] = r.cpus; igpu[j] = r.gpus; iur[j] = r.urank; ipos[j] = r.pos; iidx[j] = r.idx;
        iok[j] = r.idx >= 0 && (below || r.user == pu) && !(r.dru < a.safe) && ((r.dru - pend) > a.min_diff);
      }
    }
    double sm = 0.0, sc = 0.0, sg = 0.0;
    int nv = 0;
    bool have = false;
    double cur = 0.0;
    auto consider = [&](double dru) {
      if (sm >= pm && sc >= pcpu && (pg > 0.0 ? sg >= pg : true)) {
        if (!have || dru >= cur) { have = true; cur = dru; b.dru = dru; b.mem = sm; b.cpus = sc; b.gpus = sg; b.n_victims = nv; }
      }
    };
    if (a.hc.has_spare[h]) {
      sg = sg + a.hc.spare_gpus[h]; sm = sm + a.hc.spare_mem[h]; sc = sc + a.hc.spare_cpus[h];
      consider(1.7976931348623157e308);
    }
    if (!emit) {
      double tm = (iok[0] ? imem[0] : 0.0) + (iok[1] ? imem[1] : 0.0), tc = (iok[0] ? icpu[0] : 0.0) + (iok[1] ? icpu[1] : 0.0),
             tg = (iok[0] ? igpu[0] : 0.0) + (iok[1] ? igpu[1] : 0.0);
      for (int o = 16; o > 0; o >>= 1) {
        tm += __shfl_xor_sync(0xffffffffu, tm, o); tc += __shfl_xor_sync(0xffffffffu, tc, o);
        tg += __shfl_xor_sync(0xffffffffu, tg, o);
      }
      const double slack = 1.0 + 1e-6;
      if (!have && ((sm + tm) * slack < pm || (sc + tc) * slack < pcpu || (pg > 0.0 && (sg + tg) * slack < pg))) return b;
    }
    while (true) {
      if (emit && nv >= n_emit) break;
      VKey best;
      best.idx = -1; best.dru = 0.0; best.urank = 0; best.pos = 0;
      int bj = -1;
#pragma unroll
      for (int j = 0; j < 2; j++) {
        if (!iok[j]) continue;
        VKey c;
        c.dru = idru[j]; c.urank = iur[j]; c.pos = ipos[j]; c.idx = iidx[j];
        if (vkey_before(c, best)) { best = c; bj = j; }
      }
      const int mine = best.idx;
      for (int o = 16; o > 0; o >>= 1) {
        VKey other = vkey_shfl_xor(best, o);
        if (vkey_before(other, best)) best = other;
      }
      if (best.idx < 0) break;
      if (have && best.dru < cur) break;   // later prefixes only have smaller dru
      // the owner of the winner supplies its amounts and retires the item
      const bool won = mine == best.idx && bj >= 0;
      const int wl = __ffs(__ballot_sync(0xffffffffu, won)) - 1;
      double wm = 0.0, wc = 0.0, wg = 0.0;
      if (won) { wm = bj ? imem[1] : imem[0]; wc = bj ? icpu[1] : icpu[0]; wg = bj ? igpu[1] : igpu[0]; if (bj) iok[1] = false; else iok[0] = false; }
      wm = __shfl_sync(0xffffffffu, wm, wl); wc = __shfl_sync(0xffffffffu, wc, wl); wg = __shfl_sync(0xffffffffu, wg, wl);
      sg = sg + wg; sm = sm + wm; sc = sc + wc;
      if (emit && lane == 0) emit[n_emit - 1 - nv] = best.idx;
      nv++;
      consider(best.dru);
    }
    return b;
  }
  auto item = [&](int k) -> int {
    int i = k < seg ? a.hord[s0 + k] : a.R + (k - seg);
    if (k >= seg && a.t.host[i] != h) return -1;
    if (!a.t.alive[i]) return -1;
    double d = a.t.dru[i];
    if (!(below || a.t.user[i] == pu)) return -1;
    if (d < a.safe) return -1;
    if (!((d - pend) > a.min_diff)) return -1;
    return i;
  };
  double sm = 0.0, sc = 0.0, sg = 0.0;
  int nv = 0;
  bool have = false;
  double cur = 0.0;
  auto consider = [&](double dru) {
    if (sm >= pm && sc >= pcpu && (pg > 0.0 ? sg >= pg : true)) {
      if (!have || dru >= cur) { have = true; cur = dru; b.dru = dru; b.mem = sm; b.cpus = sc; b.gpus = sg; b.n_victims = nv; }
    }
  };
  if (a.hc.has_spare[h]) {
    sg = sg + a.hc.spare_gpus[h]; sm = sm + a.hc.spare_mem[h]; sc = sc + a.hc.spare_cpus[h];
    consider(1.7976931348623157e308);
  }
  if (!emit) {  // cannot reach the request with everything eligible (any summation order, wide margin)?
    double tm = 0.0, tc = 0.0, tg = 0.0;
    for (int k = lane; k < n_items; k += 32) {
      int i = item(k);
      if (i >= 0) { tm += a.t.mem[i]; tc += a.t.cpus[i]; tg += a.t.gpus[i]; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      tm += __shfl_xor_sync(0xffffffffu, tm, o); tc += __shfl_xor_sync(0xffffffffu, tc, o);
      tg += __shfl_xor_sync(0xffffffffu, tg, o);
    }
    const double slack = 1.0 + 1e-6;
    if (!have && ((sm + tm) * slack < pm || (sc + tc) * slack < pcpu || (pg > 0.0 && (sg + tg) * slack < pg))) return b;
  }
  VKey last;
  last.idx = -1; last.dru = 0.0; last.urank = 0; last.pos = 0;
  bool first = true;
  while (true) {
    if (emit && nv >= n_emit) break;
    VKey best;
    best.idx = -1; best.dru = 0.0; best.urank = 0; best.pos = 0;
    for (int k = lane; k < n_items; k += 32) {
      int i = item(k);
      if (i < 0) continue;
      VKey c;
      c.dru = a.t.dru[i]; c.urank = a.user_rank[a.t.user[i]]; c.pos = a.t.pos[i]; c.idx = i;
      if (!first && !vkey_before(last, c)) continue;   // already taken
      if (vkey_before(c, best)) best = c;
    }
    for (int o = 16; o > 0; o >>= 1) {
      VKey other = vkey_shfl_xor(best, o);
      if (vkey_before(other, best)) best = other;
    }
    if (best.idx < 0) break;
    if (have && best.dru < cur) break;   // later prefixes only have smaller dru
    const int i = best.idx;
    sg = sg + a.t.gpus[i]; sm = sm + a.t.mem[i]; sc = sc + a.t.cpus[i];
    if (emit && lane == 0) emit[n_emit - 1 - nv] = i;
    nv++;
    consider(best.dru);
    last = best;
    first = false;
  }
  return b;
}

__global__ void hot_build_kernel(const int32_t* hord, RTasks t, const int32_t* user_rank, int n, TaskHot* hot, int32_t* hq) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int i = hord[q];
  TaskHot r;
  r.dru = t.dru[i]; r.mem = t.mem[i]; r.cpus = t.cpus[i]; r.gpus = t.gpus[i];
  r.urank = user_rank[t.user[i]]; r.pos = t.pos[i]; r.idx = t.alive[i] ? i : -1; r.user = t.user[i];
  hot[q] = r;
  hq[i] = q;
}

// ------------------------------------------------------------------ the persistent loop
// The walk over the pending jobs (rebalancer.clj:442-458) as ONE cooperative launch: the host
// never synchronises inside the cycle.  Per pending job:
//   A  every CTA: pending scalars (binary search for the nearest task; the quota fold only when
//      the user has a finite quota), then host constraints + best sufficient prefix for the CTA's
//      hosts (warp per host) and a CTA-level argmax                      -> grid.sync
//   B  CTA 0: argmax over the CTAs, victims of the winner, next-state bookkeeping, insertion
//      point of the job's synthetic task in the user order               -> grid.sync
//   C  (only after a decision) every CTA: user order with the new task (double buffered), user
//      segments, re-fold of the users that changed                      -> grid.sync
namespace cg = cooperative_groups;

struct CtaBest { double dru; int32_t rank, host; };

// Barriers of the walk (co-residency comes from the cooperative launch).  Two counters that only grow and
// one flag: after the host phase the CTAs ARRIVE and only CTA 0 waits for all of them; the others wait
// for the flag CTA 0 raises after next-state; only the re-fold ends in a full barrier.  Pollers back off
// (nanosleep) so that the lone next-state warp is not competing with every other CTA spinning on L2.
struct WalkBar { unsigned arrive_a; unsigned flag_b; unsigned arrive_c; unsigned pad; };
__device__ __forceinline__ unsigned bar_ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void bar_arrive(unsigned* p) {   // whole CTA
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory"); }
}
__device__ __forceinline__ void bar_wait(const unsigned* p, unsigned target) {   // whole CTA
  if (threadIdx.x == 0) {
    while (bar_ld_acquire(p) < target) __nanosleep(20);
    __threadfence();
  }
  __syncthreads();
}
__device__ __forceinline__ void bar_raise(unsigned* p, unsigned v) {   // whole CTA
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
}

struct RebArgs {
  RTasks t; int R;
  int32_t* ord[2]; int32_t* us[2]; int32_t* ue[2];
  const int32_t* hord; const int32_t* hs; const int32_t* he;
  HostCols hc; PendCols pc; GroupCols gc;
  int P, U, MP;
  const int32_t* user_rank;
  const double *div_mem, *div_cpus, *q_count, *q_cpus, *q_mem, *q_gpus;
  uint8_t* has_task; int32_t* preempted_hosts;
  double min_diff, safe; int host_lifetime_mins;
  HostBest* best;        // [H]
  CtaBest* cta_best;     // [grid]
  cook_decision* dec; int32_t* victims;
  int32_t* cnt;          // [0] n_tasks [1] n_dec [2] n_vict [3] n_preempted [4] changed
  Refold* rf;
  PendScalars* ps_all;   // [P] scalars of every job the walk reached (below_quota = -1: not reached)
  int n_forced; const cook_decision* forced; const int32_t* forced_victims; int forced_only;
  const GridFlag* gf;   // exact-grid flag of the task amounts (common.cuh)
  int32_t* syn_cnt;     // [H]
  TaskHot* hot;         // [CAP] packed victim records: real tasks in host order, a synthetic task at its own index
  int32_t* hq;          // [CAP] task -> its record
  int32_t* syn_head;    // [H]
  int32_t* syn_next;    // [CAP]
  int32_t* preempted_hn; // hostname ids of preempted_hosts[]
  WalkBar* bar;
};

// task <= synthetic pending task [-prio, Long/MAX, nil(-1), job id] (tools.clj:614-641) ?
__device__ __forceinline__ bool task_le_pending(const RTasks& t, int i, int pprio, long long pj) {
  const int tp = -t.prio[i];
  if (tp != pprio) return tp < pprio;
  if (t.start[i] != 0x7fffffffffffffffLL) return true;
  if (t.tid[i] != -1) return false;  // nil < any id
  return t.jid[i] <= pj;
}

// P1 for one warp: job-below-quota (:210-220) and pending dru (:182-208) of pending job p.
__device__ void pending_scalars(const RebArgs& a, const int32_t* ord, const int32_t* us, const int32_t* ue, int p,
                                PendScalars* out, double (*stage)[32]) {
  const int lane = threadIdx.x & 31;
  const RTasks& t = a.t;
  const PendCols& pc = a.pc;
  const int u = pc.user[p];
  const int s = us[u], e = ue[u];
  const double pm = pc.mem[p], pcpu = pc.cpus[p], pg = pc.gpus ? pc.gpus[p] : 0.0;
  const int pprio = -pc.prio[p];
  const long long pj = pc.jid[p];
  // nearest: the last LIVE task of the user that sorts <= the synthetic task.  The predicate is
  // monotone along the user's order => 32-ary search for the first task that is greater
  int lo = s, hi = e;
  while (lo < hi) {
    const int step = (hi - lo + 31) / 32;
    const int q = lo + lane * step;
    const bool gt = q < hi ? !task_le_pending(t, ord[q], pprio, pj) : true;
    const unsigned m = __ballot_sync(0xffffffffu, gt);
    const int L = m ? __ffs(m) - 1 : 32;
    const int nlo = L > 0 ? lo + (L - 1) * step + 1 : lo;
    const int nhi = L < 32 ? min(hi, lo + L * step) : hi;
    lo = min(nlo, nhi); hi = nhi;
  }
  double nearest = 0.0;   // walk back over tasks preempted earlier in this cycle
  for (int base = lo; base > s; base -= 32) {
    const int q = base - 1 - lane;
    const bool live = q >= s && t.alive[ord[q]];
    const unsigned m = __ballot_sync(0xffffffffu, live);
    if (m) {
      const int l = __ffs(m) - 1;
      nearest = __shfl_sync(0xffffffffu, live ? t.dru[ord[q]] : 0.0, l);
      break;
    }
  }
  // job-below-quota: a left fold over (p, tasks in order); skipped when no quota can bind
  const double qn = a.q_count[u], qc = a.q_cpus[u], qm = a.q_mem[u], qg = a.q_gpus[u];
  const double dmax = 1.7976931348623157e308;
  int below = 1;
  if (!(qn >= dmax && qc >= dmax && qm >= dmax && qg >= dmax)) {
    double acc[4] = {1.0, pcpu, pm, pg};  // (conj running-jobs p): p first
    const bool exact = grid_exact(a.gf, e - s + 1) && grid_value_ok(pcpu) && grid_value_ok(pm) && grid_value_ok(pg);
    warp_fold_sum<4, 1>(acc, e - s, exact, [&](int k, double (&x)[4]) {
      const int i = ord[s + k];
      if (t.alive[i]) { x[0] = 1.0; x[1] = t.cpus[i]; x[2] = t.mem[i]; x[3] = t.gpus[i]; }   // preempted earlier in this cycle: adds 0.0
      return true;
    }, stage);
    below = (acc[0] <= qn && acc[1] <= qc && acc[2] <= qm && acc[3] <= qg) ? 1 : 0;
  }
  if (lane == 0) {
    out->below_quota = below;
    const double x = nearest + pm / a.div_mem[u], y = nearest + pcpu / a.div_cpus[u];
    out->pending_dru = x > y ? x : y;
  }
}

// The group constraints (constraints.clj:680-697) look at the host only through its attribute value
// (or its hostname); the value histogram over [hosts preempted so far ; the cotasks] is the same for
// every host of the walk step.  One warp per CTA builds it once per pending job (distinct values and
// their frequencies, two table entries per lane), the hosts then need one table lookup each instead
// of the O(n^2) frequency walk.  More than GP_MAXG groups on the job or more than GP_MAXV distinct
// values: `slow`, and host_ok takes the scalar walk.
constexpr int GP_MAXG = 4, GP_MAXV = 64;
struct GroupPre {
  int slow, ng;
  int kind[GP_MAXG], col[GP_MAXG], n[GP_MAXG], distinct[GP_MAXG], mn[GP_MAXG], mx[GP_MAXG], c0[GP_MAXG], c1[GP_MAXG], minimum[GP_MAXG];
  int val[GP_MAXG][GP_MAXV], freq[GP_MAXG][GP_MAXV];
};

__device__ void group_prepare(const RebArgs& a, int p, int np, GroupPre* G) {
  const int lane = threadIdx.x & 31;
  const PendCols& pc = a.pc;
  const HostCols& hc = a.hc;
  const GroupCols& gc = a.gc;
  const int k0 = (pc.group_off && gc.n > 0) ? pc.group_off[p] : 0, k1 = (pc.group_off && gc.n > 0) ? pc.group_off[p + 1] : 0;
  const int ng = k1 - k0;
  int slow = ng > GP_MAXG ? 1 : 0;
  for (int g = 0; g < ng && !slow; g++) {
    const int gi = pc.group_idx[k0 + g];
    const int kind = gc.kind[gi];
    const int col = gc.attr_col ? gc.attr_col[gi] : -1;
    const int c0 = gc.cot_off[gi], c1 = gc.cot_off[gi + 1];
    const int n = np + (c1 - c0);
    int v0 = 0, f0 = 0, v1 = 0, f1 = 0, nv = 0;   // this lane's table entries `lane` and `lane + 32`
    if (kind != COOK_GROUP_UNIQUE) {
      const bool colok = col >= 0 && col < hc.n_attr_cols;
      for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        int v = 0;
        if (i < n) v = i < np ? (colok ? hc.attr[(size_t)col * hc.H + a.preempted_hosts[i]] : 0) : gc.cot_attr[c0 + i - np];
        const int cnt = min(32, n - base);
        for (int l = 0; l < cnt; l++) {
          const int vl = __shfl_sync(0xffffffffu, v, l);
          const bool e0 = lane < nv && v0 == vl, e1 = lane + 32 < nv && v1 == vl;
          if (e0) f0++;
          if (e1) f1++;
          if (!__any_sync(0xffffffffu, e0 || e1)) {
            if (nv >= GP_MAXV) { slow = 1; break; }
            if (lane == (nv & 31)) { if (nv < 32) { v0 = vl; f0 = 1; } else { v1 = vl; f1 = 1; } }
            nv++;
          }
        }
        if (slow) break;
      }
    }
    int mn = 0x7fffffff, mx = 0;
    if (lane < nv) { mn = min(mn, f0); mx = max(mx, f0); }
    if (lane + 32 < nv) { mn = min(mn, f1); mx = max(mx, f1); }
    for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    G->val[g][lane] = v0; G->freq[g][lane] = lane < nv ? f0 : 0;
    G->val[g][lane + 32] = v1; G->freq[g][lane + 32] = lane + 32 < nv ? f1 : 0;
    if (lane == 0) {
      G->kind[g] = kind; G->col[g] = col; G->n[g] = n; G->distinct[g] = nv; G->mn[g] = mn; G->mx[g] = mx;
      G->c0[g] = c0; G->c1[g] = c1; G->minimum[g] = gc.minimum[gi];
    }
  }
  if (lane == 0) { G->slow = slow; G->ng = ng; }
}

// the group constraints of pending job p on host h through the prepared tables (whole warp)
__device__ bool host_groups_ok(const RebArgs& a, const GroupPre& G, int h, int np, bool have) {
  const int lane = threadIdx.x & 31;
  const HostCols& hc = a.hc;
  for (int g = 0; g < G.ng; g++) {
    const int kind = G.kind[g];
    if (kind == COOK_GROUP_UNIQUE) {
      if (!have) return false;
      const int hn = hc.hostname_id[h];
      bool hit = false;
      for (int q = lane; q < np; q += 32) hit |= a.preempted_hn[q] == hn;
      for (int c = G.c0[g] + lane; c < G.c1[g]; c += 32) hit |= a.gc.cot_host[c] == hn;
      if (__any_sync(0xffffffffu, hit)) return false;
    } else {
      if (G.n[g] == 0) continue;
      const int col = G.col[g];
      const int target = (have && col >= 0 && col < hc.n_attr_cols) ? hc.attr[(size_t)col * hc.H + h] : 0;
      const int nv = G.distinct[g];
      int e = 0;
      if (lane < nv && G.val[g][lane] == target) e = G.freq[g][lane];
      if (lane + 32 < nv && G.val[g][lane + 32] == target) e = G.freq[g][lane + 32];
      const unsigned m = __ballot_sync(0xffffffffu, e > 0);
      const int tf = m ? __shfl_sync(0xffffffffu, e, __ffs(m) - 1) : 0;
      if (kind == COOK_GROUP_ATTR_EQUALS) { if (tf == 0) return false; }
      else if (tf != 0 && !balanced_ok(tf, G.mn[g], G.mx[g], nv, G.minimum[g])) return false;
    }
  }
  return true;
}

// P2 for one host (every lane computes the same): constraints.clj:504-515, :680-697
__device__ bool host_ok(const RebArgs& a, int p, int h, int np, const GroupPre& G) {
  const PendCols& pc = a.pc;
  const HostCols& hc = a.hc;
  const GroupCols& gc = a.gc;
  const bool have = a.has_task[h] != 0;
  bool pass = true;
  if (have && pc.novel_off)
    for (int k = pc.novel_off[p]; k < pc.novel_off[p + 1]; k++)
      if (pc.novel_host[k] == hc.hostname_id[h]) pass = false;
  const bool k8s = have && hc.is_k8s && hc.is_k8s[h];
  const double g = pc.gpus ? pc.gpus[p] : 0.0;
  if (k8s) {
    if (g > 0.0) {
      double hv = csr_get(hc.gpu_off, hc.gpu_model, hc.gpu_count, h, pc.gpu_model ? pc.gpu_model[p] : -1);
      if (!(hv == g)) pass = false;
    } else {
      int nm = hc.gpu_off ? hc.gpu_off[h + 1] - hc.gpu_off[h] : 0;
      if (nm != 0) pass = false;
    }
  } else if (!(g == 0.0)) {
    pass = false;
  }
  if (pc.disk_request && pc.disk_request[p] >= 0.0 && k8s) {
    double space = csr_get(hc.disk_off, hc.disk_type, hc.disk_space, h, pc.disk_type ? pc.disk_type[p] : -1);
    if (!(space >= pc.disk_request[p])) pass = false;
  }
  if (pc.attr_off)
    for (int k = pc.attr_off[p]; k < pc.attr_off[p + 1]; k++) {
      int col = pc.attr_col[k], val = pc.attr_val[k];
      if (!have || col < 0 || col >= hc.n_attr_cols) { pass = false; continue; }
      int hv = hc.attr[(size_t)col * hc.H + h];
      if (val <= 0 || hv != val) pass = false;
    }
  if (pc.est_end_ms && pc.est_end_ms[p] >= 0 && have && hc.host_start && hc.host_start[h] >= 0) {
    long long death = 1000LL * hc.host_start[h] + 60000LL * a.host_lifetime_mins;
    if (!(pc.est_end_ms[p] < death)) pass = false;
  }
  if (pc.ckpt_location && pc.ckpt_location[p] >= 0) {
    int loc = (have && hc.location) ? hc.location[h] : -1;
    if (loc != pc.ckpt_location[p]) pass = false;
  }
  if (pass && !G.slow) return host_groups_ok(a, G, h, np, have);
  if (pass && pc.group_off && gc.n > 0) {   // over [hosts preempted so far ; cotasks]
    for (int k = pc.group_off[p]; k < pc.group_off[p + 1]; k++) {
      const int gi = pc.group_idx[k];
      const int kind = gc.kind[gi];
      const int c0 = gc.cot_off[gi], nc = gc.cot_off[gi + 1] - c0;
      int f;
      if (kind == COOK_GROUP_UNIQUE) {
        if (!have) return false;
        f = group_fail(kind, np + nc, hc.hostname_id[h], 0,
                       [&](int i) { return i < np ? hc.hostname_id[a.preempted_hosts[i]] : gc.cot_host[c0 + i - np]; });
      } else {
        const int col = gc.attr_col ? gc.attr_col[gi] : -1;
        auto hattr = [&](int hh) { return (col >= 0 && col < hc.n_attr_cols) ? hc.attr[(size_t)col * hc.H + hh] : 0; };
        f = group_fail(kind, np + nc, have ? hattr(h) : 0, gc.minimum[gi],
                       [&](int i) { return i < np ? hattr(a.preempted_hosts[i]) : gc.cot_attr[c0 + i - np]; });
      }
      if (f >= 0) return false;
    }
  }
  return pass;
}

constexpr int REB_TB = 512;   // 16 warps: a warp per host in the host phase, one CTA per SM at the barriers
__global__ void __launch_bounds__(REB_TB) rebalance_kernel(RebArgs a) {
  unsigned n_a = 0, n_c = 0;   // barrier generations
  const unsigned G = gridDim.x;
  __shared__ PendScalars s_ps;
  __shared__ GroupPre s_gp;
  __shared__ int s_ru[64], s_rfrom[64];
  __shared__ double s_dru[REB_TB / 32];
  __shared__ int s_rank[REB_TB / 32], s_host[REB_TB / 32];
  __shared__ double s_stage[REB_TB / 32][4][32];   // each warp's staging area of the serial folds
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nw = blockDim.x >> 5;
  const int gw = blockIdx.x * nw + warp, n_gw = gridDim.x * nw;
  const int gt = blockIdx.x * blockDim.x + tid, n_gt = gridDim.x * blockDim.x;
  const HostCols& hc = a.hc;
  const PendCols& pc = a.pc;
  RTasks t = a.t;
  int cur = 0, n_tasks = a.R, n_dec = 0;
  long long tA = 0, tB = 0, tC = 0, tS = 0, tA0 = 0, tb[5] = {0, 0, 0, 0, 0}, t0 = clock64();   // CTA 0 / thread 0: cycles per phase (COOK_PROF)
  const bool forced_only = a.n_forced > 0 && a.forced_only != 0;
  const int n_walk = forced_only ? a.n_forced : a.P;
  for (int w = 0; w < n_walk && n_dec < a.MP; w++) {
    const int p = forced_only ? a.forced[w].pending_idx : w;
    int fi = -1;
    for (int q = 0; q < a.n_forced; q++) if (a.forced[q].pending_idx == p) fi = q;
    const int32_t* ord = a.ord[cur];
    const int32_t* us = a.us[cur];
    const int32_t* ue = a.ue[cur];
    // ---- A: scalars of the job, then this CTA's hosts
    if (warp == 0) {
      pending_scalars(a, ord, us, ue, p, &s_ps, s_stage[warp]);
    }
    if (warp == nw - 1) group_prepare(a, p, a.cnt[3], &s_gp);
    __syncthreads();
    tA0 += clock64() - t0;
    if (blockIdx.x == 0 && tid == 0) a.ps_all[p] = s_ps;
    SelArgs sa;
    sa.hord = a.hord; sa.hs = a.hs; sa.he = a.he; sa.t = t; sa.R = a.R; sa.n_tasks = n_tasks;
    sa.hc = hc; sa.pc = pc; sa.user_rank = a.user_rank; sa.ps = &s_ps;
    sa.min_diff = a.min_diff; sa.safe = a.safe; sa.syn_cnt = a.syn_cnt; sa.hot = a.hot; sa.syn_head = a.syn_head; sa.syn_next = a.syn_next;
    double bd = -1.0;
    int br = -1, bh = -1;
    if (fi < 0) {
      const int np = a.cnt[3];
      for (int h = gw; h < hc.H; h += n_gw) {
        HostBest b;
        b.dru = 0.0; b.mem = b.cpus = b.gpus = 0.0; b.n_victims = -1;
        if (host_ok(a, p, h, np, s_gp)) b = host_select(sa, p, h, lane, nullptr, 0);
        if (lane == 0) a.best[h] = b;
        if (b.n_victims >= 0) {
          const int r = hc.name_rank[h];
          if (b.dru > bd || (b.dru == bd && r > br)) { bd = b.dru; br = r; bh = h; }
        }
      }
    }
    if (lane == 0) { s_dru[warp] = bd; s_rank[warp] = br; s_host[warp] = bh; }
    __syncthreads();
    if (tid == 0) {
      for (int q = 1; q < nw; q++)
        if (s_dru[q] > bd || (s_dru[q] == bd && s_rank[q] > br)) { bd = s_dru[q]; br = s_rank[q]; bh = s_host[q]; }
      CtaBest cb;
      cb.dru = bd; cb.rank = br; cb.host = bh;
      a.cta_best[blockIdx.x] = cb;
    }
    { const long long t1 = clock64(); tA += t1 - t0; t0 = t1; }
    n_a++;
    bar_arrive(&a.bar->arrive_a);
    if (blockIdx.x == 0) bar_wait(&a.bar->arrive_a, n_a * G);
    { const long long t1 = clock64(); tS += t1 - t0; t0 = t1; }
    // ---- B: argmax over the CTAs (max dru; ties -> greatest hostname), next-state
    if (blockIdx.x == 0 && warp == 0) {
      double d = -1.0;
      int r = -1, h = -1;
      for (int q = lane; q < (int)gridDim.x; q += 32) {
        const CtaBest cb = a.cta_best[q];
        if (cb.host >= 0 && (cb.dru > d || (cb.dru == d && cb.rank > r))) { d = cb.dru; r = cb.rank; h = cb.host; }
      }
      for (int o = 16; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, d, o);
        const int orr = __shfl_xor_sync(0xffffffffu, r, o), oh = __shfl_xor_sync(0xffffffffu, h, o);
        if (oh >= 0 && (od > d || (od == d && orr > r))) { d = od; r = orr; h = oh; }
      }
      tb[4] += clock64() - t0;
      HostBest b;
      b.dru = 0.0; b.mem = b.cpus = b.gpus = 0.0; b.n_victims = -1;
      const int vb = a.cnt[2];
      if (fi >= 0) {   // the decision is given (the reference's tests hand next-state its input)
        const cook_decision f = a.forced[fi];
        h = f.host; b.dru = f.dru; b.mem = f.mem; b.cpus = f.cpus; b.gpus = f.gpus; b.n_victims = f.victim_count;
        for (int q = lane; q < f.victim_count; q += 32)
          a.victims[vb + f.victim_count - 1 - q] = a.forced_victims[f.victim_begin + q];   // ascending dru
        __syncwarp();
      } else if (h >= 0) {
        b = a.best[h];
        // the victims again (same selection), stored in ascending dru order
        if (b.n_victims > 0) host_select(sa, p, h, lane, a.victims + vb, b.n_victims);
        __syncwarp();
      }
      long long tq = clock64();
      tb[0] += tq - t0;
      if (h < 0) {
        if (lane == 0) a.cnt[4] = 0;
      } else {
        const int n = n_tasks, ni = n;
        const int pu = pc.user[p];
        Refold& rf = *a.rf;
        // the victims, one per lane: dead, off their host's records, host noted as preempted; then the
        // list of users to re-fold (merged through registers, table in shared memory)
        const int nv = b.n_victims > 0 ? b.n_victims : 0;
        const int np0 = a.cnt[3];
        int rn = 0, rall = nv > 64 ? 1 : 0;
        bool pu_listed = false;
        for (int base = 0; base < nv; base += 32) {
          const int kk = base + lane;   // selection order
          int u = -1, from = 0;
          if (kk < nv) {
            const int i = a.victims[vb + nv - 1 - kk];
            t.alive[i] = 0;
            a.hot[a.hq[i]].idx = -1;
            const int hh = t.host[i];
            u = t.user[i]; from = us[u] + t.pos[i];
            a.preempted_hn[np0 + kk] = hc.hostname_id[hh];
            a.preempted_hosts[np0 + kk] = hh;
            if (kk < 64) { rf.vu[kk] = u; rf.vs[kk] = from; rf.vm[kk] = t.mem[i]; rf.vc[kk] = t.cpus[i]; }
          }
          const int cntv = min(32, nv - base);
          for (int l = 0; l < cntv; l++) {
            const int ul = __shfl_sync(0xffffffffu, u, l), fl = __shfl_sync(0xffffffffu, from, l);
            const bool e0 = lane < rn && s_ru[lane] == ul, e1 = lane + 32 < rn && s_ru[lane + 32] == ul;
            if (e0) s_rfrom[lane] = min(s_rfrom[lane], fl);
            if (e1) s_rfrom[lane + 32] = min(s_rfrom[lane + 32], fl);
            if (!__any_sync(0xffffffffu, e0 || e1)) {
              if (rn < 63) { if (lane == 0) { s_ru[rn] = ul; s_rfrom[rn] = fl; } rn++; }
              else rall = 1;
            }
            if (ul == pu) pu_listed = true;
            __syncwarp();
          }
        }
        if (!pu_listed) { if (lane == 0) { s_ru[rn] = pu; s_rfrom[rn] = 0x7fffffff; } rn++; }
        __syncwarp();
        { const long long t1 = clock64(); tb[1] += t1 - tq; tq = t1; }
        rf.user[lane] = s_ru[lane]; rf.user[lane + 32] = s_ru[lane + 32];
        rf.from[lane] = s_rfrom[lane]; rf.from[lane + 32] = s_rfrom[lane + 32];
        if (lane == 0) {
          const int di = a.cnt[1];
          cook_decision dd;
          dd.pending_idx = p; dd.host = h; dd.dru = b.dru; dd.mem = b.mem; dd.cpus = b.cpus; dd.gpus = b.gpus;
          dd.victim_begin = vb; dd.victim_count = b.n_victims;
          rf.n = rn; rf.all = rall; rf.pu = pu; rf.n_vict = min(nv, 64);
          a.cnt[3] = np0 + nv;
          a.cnt[2] = vb + b.n_victims;
          a.dec[di] = dd;
          a.cnt[1] = di + 1;
          // synthetic running task of the pending job on host h (create-task-ent :hostname)
          a.cnt[0] = n + 1;
          t.user[ni] = pu; t.prio[ni] = pc.prio[p]; t.start[ni] = 0x7fffffffffffffffLL;
          t.tid[ni] = -1; t.jid[ni] = pc.jid[p];
          t.cpus[ni] = pc.cpus[p]; t.mem[ni] = pc.mem[p]; t.gpus[ni] = pc.gpus ? pc.gpus[p] : 0.0;
          t.host[ni] = h; t.alive[ni] = 1; t.dru[ni] = 0.0; t.pos[ni] = 0; t.cm[ni] = 0.0; t.cc[ni] = 0.0;
          a.has_task[h] = 1;
          a.syn_cnt[h] += 1;
          {
            TaskHot r;
            r.dru = 0.0; r.mem = pc.mem[p]; r.cpus = pc.cpus[p]; r.gpus = pc.gpus ? pc.gpus[p] : 0.0;
            r.urank = a.user_rank[pu]; r.pos = 0; r.idx = ni; r.user = pu;
            a.hot[ni] = r; a.hq[ni] = ni;
            a.syn_next[ni] = a.syn_head[h]; a.syn_head[h] = ni;
          }
          hc.has_spare[h] = 1;
          hc.spare_mem[h] = b.mem - pc.mem[p];
          hc.spare_gpus[h] = b.gpus - (pc.gpus ? pc.gpus[p] : 0.0);
          hc.spare_cpus[h] = b.cpus - pc.cpus[p];
        }
        __syncwarp();
        // where the new task goes in the user order: after every task that is not greater
        // (32-ary search: the predicate "new task < ord[q]" is monotone in q)
        { const long long t1 = clock64(); tb[2] += t1 - tq; tq = t1; }
        const LessUserTask less{t.user, t.prio, t.start, t.tid, t.jid, a.user_rank};
        const int ps = us[pu], pe = ue[pu];
        int lo = pe > ps ? ps : 0, hi = pe > ps ? pe : n;   // a user with tasks: inside its own segment
        while (lo < hi) {
          const int step = (hi - lo + 31) / 32;
          const int q = lo + lane * step;
          const bool pred = q < hi ? less(ni, ord[q]) : true;
          const unsigned m = __ballot_sync(0xffffffffu, pred);
          const int L = m ? __ffs(m) - 1 : 32;
          const int nlo = L > 0 ? lo + (L - 1) * step + 1 : lo;
          const int nhi = L < 32 ? min(hi, lo + L * step) : hi;
          lo = min(nlo, nhi); hi = nhi;
        }
        if (lane == 0) {
          rf.q_ins = lo; a.cnt[4] = 1;
          const bool prev = pe > ps && lo > ps;
          rf.base_m = prev ? t.cm[ord[lo - 1]] : 0.0; rf.base_c = prev ? t.cc[ord[lo - 1]] : 0.0;
        }
        { const long long t1 = clock64(); tb[3] += t1 - tq; tq = t1; }
      }
      __threadfence();
    }
    { const long long t1 = clock64(); tB += t1 - t0; t0 = t1; }
    if (blockIdx.x == 0) bar_raise(&a.bar->flag_b, n_a);
    else bar_wait(&a.bar->flag_b, n_a);
    { const long long t1 = clock64(); tS += t1 - t0; t0 = t1; }
    n_dec = a.cnt[1];
    if (a.cnt[4] != 0) {
      // ---- C: next-state.  New order / segments go to the other buffer; the changed users are
      // re-folded reading the new order through the old one (no sync in between).
      const int n = n_tasks, ni = n_tasks;
      const Refold& rf = *a.rf;
      const int q = rf.q_ins, pu = rf.pu;
      int32_t* nord = a.ord[cur ^ 1];
      int32_t* nus = a.us[cur ^ 1];
      int32_t* nue = a.ue[cur ^ 1];
      auto new_at = [&](int j) { return j < q ? ord[j] : (j == q ? ni : ord[j - 1]); };
      auto user_at = [&](int j) { return t.user[new_at(j)]; };
      for (int j = gt; j <= n; j += n_gt) {
        nord[j] = new_at(j);
        mark_segment(j, n + 1, user_at, nus, nue);
      }
      const bool all = rf.all != 0;
      const int n_fold = all ? a.U : rf.n;
      // a listed user with exact-grid amounts: every running sum moves by a constant (the victims at or
      // before the slot leave, the new task joins), so the whole grid updates the slots independently.
      // Anything else (`all`, off-grid amounts) is folded by one warp per user in the reference's order.
      const double pmem = pc.mem[p], pcpus = pc.cpus[p];
      for (int wv = 0; wv < (all ? 0 : n_fold); wv++) {
        const int u = rf.user[wv];
        int s = us[u], e = ue[u];
        if (e <= s) { if (u != pu) continue; s = q; e = q + 1; }
        else if (u == pu) e = e + 1;
        else if (s >= q) { s++; e++; }
        if (!grid_exact(a.gf, e - s)) continue;
        int f = rf.from[wv];
        if (f == 0x7fffffff) f = q;
        else if (f >= q) f++;
        if (u == pu) f = min(f, q);
        f = min(max(f, s), e);
        const double md = a.div_mem[u], cd = a.div_cpus[u];
        const int nvict = rf.n_vict;
        for (int pp = f + gt; pp < e; pp += n_gt) {
          const int i = new_at(pp);
          const bool is_new = u == pu && pp == q;
          double bm = is_new ? rf.base_m : t.cm[i], bc = is_new ? rf.base_c : t.cc[i];
          double dm = 0.0, dc = 0.0;
          for (int k = 0; k < nvict; k++) {
            if (rf.vu[k] != u) continue;
            const int sv = rf.vs[k] >= q ? rf.vs[k] + 1 : rf.vs[k];
            if (sv <= pp) { dm = dm + rf.vm[k]; dc = dc + rf.vc[k]; }
          }
          bm = bm - dm; bc = bc - dc;
          if (u == pu && pp >= q) { bm = bm + pmem; bc = bc + pcpus; }
          t.cm[i] = bm; t.cc[i] = bc;
          const double x = bm / md, y = bc / cd;
          const double dr = x > y ? x : y;
          t.dru[i] = dr;
          t.pos[i] = pp - s;
          { TaskHot& hr = a.hot[a.hq[i]]; hr.dru = dr; hr.pos = pp - s; }
        }
      }
      for (int wv = gw; wv < n_fold; wv += n_gw) {
        const int u = all ? wv : rf.user[wv];
        int s = us[u], e = ue[u];
        if (e <= s) { if (u != pu) continue; s = q; e = q + 1; }
        else if (u == pu) e = e + 1;
        else if (s >= q) { s++; e++; }
        int f = s;
        if (!all) {
          f = rf.from[wv];
          if (f == 0x7fffffff) f = q;           // only the insertion touches this user
          else if (f >= q) f++;                 // slots at and after the insertion moved by one
          if (u == pu) f = min(f, q);
          f = min(max(f, s), e);
        }
        const double md = a.div_mem[u], cd = a.div_cpus[u];
        double acc[2] = {0.0, 0.0};   // mem, cpus
        if (f > s) { const int j = new_at(f - 1); acc[0] = t.cm[j]; acc[1] = t.cc[j]; }
        const bool exact = grid_exact(a.gf, e - s);
        if (exact && !all) continue;   // done element-wise above
        for (int base = f; base < e; base += 32) {
          const int pp = base + lane;
          const int i = pp < e ? new_at(pp) : -1;
          const bool live = i >= 0 && t.alive[i];
          double v[2] = {live ? t.mem[i] : 0.0, live ? t.cpus[i] : 0.0};
          warp_fold_prefix(v, acc, min(32, e - base), exact, s_stage[warp]);
          if (i >= 0) {
            const double mym = v[0], myc = v[1];
            t.cm[i] = mym; t.cc[i] = myc;
            const double x = mym / md, y = myc / cd;
            const double dr = x > y ? x : y;
            t.dru[i] = dr;
            t.pos[i] = pp - s;
            { TaskHot& hr = a.hot[a.hq[i]]; hr.dru = dr; hr.pos = pp - s; }
          }
        }
      }
      { const long long t1 = clock64(); tC += t1 - t0; t0 = t1; }
      n_c++;
      bar_arrive(&a.bar->arrive_c);
      bar_wait(&a.bar->arrive_c, n_c * G);
      { const long long t1 = clock64(); tS += t1 - t0; t0 = t1; }
      cur ^= 1;
      n_tasks = n_tasks + 1;
    }
  }
  if (blockIdx.x == 0 && tid == 0) { a.cnt[8] = (int)(tA >> 10); a.cnt[9] = (int)(tB >> 10); a.cnt[10] = (int)(tC >> 10); a.cnt[11] = (int)(tS >> 10); a.cnt[12] = (int)(tA0 >> 10); for (int k = 0; k < 5; k++) a.cnt[13 + k] = (int)(tb[k] >> 10); }
}

}  // namespace

#define RUP(dst, src, n) CK(pool, upload(ar, st, (src), (size_t)(n), &(dst)))

static int32_t rebalance_run(cook_pool* pool, const cook_running_soa* running,
                             const cook_jobs_soa* pending, const int64_t* pending_job_id,
                             const int32_t* pending_priority, const cook_host_table* hosts,
                             const cook_groups* groups, const cook_user_table* users,
                             const cook_rebalance_params* prm, cook_decision* out_decisions,
                             int32_t* out_victims, int32_t* out_n, const cook_reb_trace* tr) {
  if (!pool) return COOK_E_BADARG;
  if (!running || !pending || !pending_job_id || !pending_priority || !hosts || !users || !prm ||
      !out_decisions || !out_victims || !out_n)
    return set_err(pool, COOK_E_BADARG, "cook_rebalance: null argument");
  if (pool->dru_mode != 0)
    return set_err(pool, COOK_E_UNSUPPORTED_CONSTRAINT,
                   "cook_rebalance: GPU DRU mode has no reference behaviour (rebalancer.clj:339-349 throws)");
  const int R = running->t.n, P = pending->n, H = hosts->n, U = users->n_users;
  const int MP = prm->max_preemption;
  *out_n = 0;
  if (P <= 0 || MP <= 0 || H <= 0) return COOK_OK;
  if (!idx_in_range(running->t.user, R, 0, U) || !idx_in_range(pending->user, P, 0, U))
    return set_err(pool, COOK_E_BADARG, "cook_rebalance: user index out of range");
  if (!idx_in_range(running->host, R, 0, H)) return set_err(pool, COOK_E_BADARG, "cook_rebalance: running.host out of range");
  if (groups && pending->group_off && !idx_in_range(pending->group_idx, pending->group_off[P], 0, groups->n_groups))
    return set_err(pool, COOK_E_BADARG, "cook_rebalance: group index out of range");
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  Arena& ar = pool->arena;
  const int CAP = R + MP + 1;
  const int G = groups ? groups->n_groups : 0;
  Sizer sz;
  for (int k = 0; k < 6; k++) sz.add<int64_t>(CAP);  // generous: covers int32/int64/double columns
  for (int k = 0; k < 10; k++) sz.add<double>(CAP);
  for (int k = 0; k < 8; k++) sz.add<int32_t>(CAP);
  sz.add<Refold>(2);
  for (int k = 0; k < 12; k++) sz.add<double>(std::max(U, H) + 1);
  for (int k = 0; k < 16; k++) sz.add<int32_t>(std::max(U, H) + 2);
  size_t csr_h = (hosts->gpu_off ? hosts->gpu_off[H] : 0) + (hosts->disk_off ? hosts->disk_off[H] : 0);
  sz.add<double>(csr_h + 64); sz.add<int32_t>(csr_h + 64);
  sz.add<int32_t>((size_t)hosts->n_attr_cols * H + 1);
  sz.add<int64_t>(H + 1);
  for (int k = 0; k < 8; k++) sz.add<double>(P + 1);
  for (int k = 0; k < 12; k++) sz.add<int32_t>(P + 2);
  size_t csr_p = (pending->novel_off ? pending->novel_off[P] : 0) + 2 * (size_t)(pending->attr_off ? pending->attr_off[P] : 0) +
                 (pending->group_off ? pending->group_off[P] : 0);
  sz.add<int32_t>(csr_p + 64); sz.add<int64_t>(P + 1);
  if (G) { sz.add<int32_t>(6 * (size_t)(G + 2)); sz.add<int32_t>(2 * (size_t)(groups->cot_off ? groups->cot_off[G] : 0) + 64); }
  sz.add<HostBest>(H + 1); sz.add<cook_decision>(MP + 1); sz.add<int32_t>(CAP + MP);
  sz.add<PendScalars>(P + 4); sz.add<int32_t>(64);
  sz.add<int32_t>(CAP); sz.add<int32_t>(CAP + MP); sz.add<int32_t>(CAP + MP);   // second order buffer, preempted hosts (+ their hostname ids)
  for (int k = 0; k < 2; k++) sz.add<int32_t>(U + 1);            // second segment buffers
  sz.add<CtaBest>(4 * pool->sm_count + 8); sz.add<GridFlag>(1); sz.add<int32_t>(H + 1);
  sz.add<TaskHot>(CAP); sz.add<int32_t>(CAP); sz.add<int32_t>(H + 1); sz.add<int32_t>(CAP); sz.add<WalkBar>(1);
  sz.add<double>(CAP); sz.add<double>(CAP); sz.add<double>(CAP / OS_TILE + 2); sz.add<double>(CAP / OS_TILE + 2);
  if (tr && tr->n_forced > 0) { sz.add<cook_decision>(tr->n_forced + 1); sz.add<int32_t>(CAP + MP); }
  CK(pool, ar.reserve(sz.off + (1 << 16)));
  ar.reset();

  CK(pool, cudaEventRecord(pool->ev[12], st));
  RTasks t;
  t.user = ar.take<int32_t>(CAP); t.prio = ar.take<int32_t>(CAP); t.start = ar.take<int64_t>(CAP);
  t.tid = ar.take<int64_t>(CAP); t.jid = ar.take<int64_t>(CAP); t.cpus = ar.take<double>(CAP);
  t.mem = ar.take<double>(CAP); t.gpus = ar.take<double>(CAP); t.host = ar.take<int32_t>(CAP);
  t.alive = ar.take<uint8_t>(CAP); t.dru = ar.take<double>(CAP); t.pos = ar.take<int32_t>(CAP);
  t.cm = ar.take<double>(CAP); t.cc = ar.take<double>(CAP);
  if (!t.cc) return set_err(pool, COOK_E_OOM, "cook_rebalance: arena exhausted");
  const cook_tasks_soa& rt = running->t;
#define CPY(dst, src, T) if (R) CK(pool, cudaMemcpyAsync(dst, src, sizeof(T) * R, cudaMemcpyHostToDevice, st))
  CPY(t.user, rt.user, int32_t); CPY(t.prio, rt.priority, int32_t); CPY(t.start, rt.start_time, int64_t);
  CPY(t.tid, rt.task_id, int64_t); CPY(t.jid, rt.job_id, int64_t); CPY(t.cpus, rt.cpus, double);
  CPY(t.mem, rt.mem, double); CPY(t.host, running->host, int32_t);
  if (rt.gpus) { CPY(t.gpus, rt.gpus, double); } else CK(pool, cudaMemsetAsync(t.gpus, 0, sizeof(double) * CAP, st));
#undef CPY
  CK(pool, cudaMemsetAsync(t.alive, 0, CAP, st));
  if (R) CK(pool, cudaMemsetAsync(t.alive, 1, R, st));
  CK(pool, cudaMemsetAsync(t.dru, 0, sizeof(double) * CAP, st));

  int32_t* d_urank; double *d_divm, *d_divc, *d_qn, *d_qc, *d_qm, *d_qg;
  RUP(d_urank, users->name_rank, U); RUP(d_divm, users->div_mem, U); RUP(d_divc, users->div_cpus, U);
  RUP(d_qn, users->quota_count, U); RUP(d_qc, users->quota_cpus, U); RUP(d_qm, users->quota_mem, U);
  RUP(d_qg, users->quota_gpus, U);

  HostCols hc;
  memset(&hc, 0, sizeof(hc));
  hc.H = H;
  { int32_t* p; RUP(p, hosts->hostname_id, H); hc.hostname_id = p; RUP(p, hosts->name_rank, H); hc.name_rank = p; }
  hc.has_spare = ar.take<uint8_t>(H + 1); hc.spare_cpus = ar.take<double>(H + 1);
  hc.spare_mem = ar.take<double>(H + 1); hc.spare_gpus = ar.take<double>(H + 1);
  CK(pool, cudaMemsetAsync(hc.has_spare, 0, H + 1, st));
  CK(pool, cudaMemsetAsync(hc.spare_cpus, 0, sizeof(double) * (H + 1), st));
  CK(pool, cudaMemsetAsync(hc.spare_mem, 0, sizeof(double) * (H + 1), st));
  CK(pool, cudaMemsetAsync(hc.spare_gpus, 0, sizeof(double) * (H + 1), st));
  if (hosts->has_spare) CK(pool, cudaMemcpyAsync(hc.has_spare, hosts->has_spare, H, cudaMemcpyHostToDevice, st));
  if (hosts->spare_cpus) CK(pool, cudaMemcpyAsync(hc.spare_cpus, hosts->spare_cpus, sizeof(double) * H, cudaMemcpyHostToDevice, st));
  if (hosts->spare_mem) CK(pool, cudaMemcpyAsync(hc.spare_mem, hosts->spare_mem, sizeof(double) * H, cudaMemcpyHostToDevice, st));
  if (hosts->spare_gpus) CK(pool, cudaMemcpyAsync(hc.spare_gpus, hosts->spare_gpus, sizeof(double) * H, cudaMemcpyHostToDevice, st));
  { uint8_t* p; RUP(p, hosts->is_k8s, H); hc.is_k8s = p; }
  { int32_t* p; RUP(p, hosts->location, H); hc.location = p; }
  if (hosts->gpu_off) { int32_t* p; RUP(p, hosts->gpu_off, H + 1); hc.gpu_off = p;
    int n = std::max(1, hosts->gpu_off[H]); RUP(p, hosts->gpu_model, n); hc.gpu_model = p;
    double* q; RUP(q, hosts->gpu_count, n); hc.gpu_count = q; }
  if (hosts->disk_off) { int32_t* p; RUP(p, hosts->disk_off, H + 1); hc.disk_off = p;
    int n = std::max(1, hosts->disk_off[H]); RUP(p, hosts->disk_type, n); hc.disk_type = p;
    double* q; RUP(q, hosts->disk_space, n); hc.disk_space = q; }
  { int64_t* p; RUP(p, hosts->host_start_time, H); hc.host_start = p; }
  hc.n_attr_cols = hosts->attr ? hosts->n_attr_cols : 0;
  if (hc.n_attr_cols > 0) { int32_t* p; RUP(p, hosts->attr, (size_t)hc.n_attr_cols * H); hc.attr = p; }

  PendCols pc;
  memset(&pc, 0, sizeof(pc));
  { int32_t* p; RUP(p, pending->user, P); pc.user = p; RUP(p, pending_priority, P); pc.prio = p; }
  { double* p; RUP(p, pending->cpus, P); pc.cpus = p; RUP(p, pending->mem, P); pc.mem = p; RUP(p, pending->gpus, P); pc.gpus = p; }
  { int64_t* p; RUP(p, pending_job_id, P); pc.jid = p; RUP(p, pending->est_end_ms, P); pc.est_end_ms = p; }
  if (pending->novel_off) { int32_t* p; RUP(p, pending->novel_off, P + 1); pc.novel_off = p;
    RUP(p, pending->novel_host, std::max(1, pending->novel_off[P])); pc.novel_host = p; }
  { int32_t* p; RUP(p, pending->gpu_model, P); pc.gpu_model = p; RUP(p, pending->disk_type, P); pc.disk_type = p;
    RUP(p, pending->ckpt_location, P); pc.ckpt_location = p; }
  { double* p; RUP(p, pending->disk_request, P); pc.disk_request = p; }
  if (pending->attr_off) { int32_t* p; RUP(p, pending->attr_off, P + 1); pc.attr_off = p;
    int n = std::max(1, pending->attr_off[P]); RUP(p, pending->attr_col, n); pc.attr_col = p;
    RUP(p, pending->attr_val, n); pc.attr_val = p; }
  GroupCols gc;
  memset(&gc, 0, sizeof(gc));
  if (G && pending->group_off) {
    int32_t* p; RUP(p, pending->group_off, P + 1); pc.group_off = p;
    RUP(p, pending->group_idx, std::max(1, pending->group_off[P])); pc.group_idx = p;
    gc.n = G;
    RUP(p, groups->kind, G); gc.kind = p; RUP(p, groups->attr_col, G); gc.attr_col = p;
    RUP(p, groups->minimum, G); gc.minimum = p; RUP(p, groups->cot_off, G + 1); gc.cot_off = p;
    int n = std::max(1, groups->cot_off ? groups->cot_off[G] : 0);
    RUP(p, groups->cot_hostname_id, n); gc.cot_host = p; RUP(p, groups->cot_attr_val, n); gc.cot_attr = p;
    if (!gc.cot_off || !gc.kind) return set_err(pool, COOK_E_BADARG, "cook_rebalance: incomplete cook_groups");
  }

  int32_t* d_ord = ar.take<int32_t>(CAP); int32_t* d_ord2 = ar.take<int32_t>(CAP);
  int32_t* d_hord = ar.take<int32_t>(CAP);
  int32_t* d_tmp = ar.take<int32_t>(CAP);
  int32_t* d_us = ar.take<int32_t>(U + 1); int32_t* d_ue = ar.take<int32_t>(U + 1);
  int32_t* d_us2 = ar.take<int32_t>(U + 1); int32_t* d_ue2 = ar.take<int32_t>(U + 1);
  int32_t* d_hs = ar.take<int32_t>(H + 1); int32_t* d_he = ar.take<int32_t>(H + 1);
  uint8_t* d_has_task = ar.take<uint8_t>(H + 1);
  HostBest* d_best = ar.take<HostBest>(H + 1);
  CtaBest* d_cta = ar.take<CtaBest>(4 * pool->sm_count + 8);
  cook_decision* d_dec = ar.take<cook_decision>(MP + 1);
  int32_t* d_vict = ar.take<int32_t>(CAP + MP);
  int32_t* d_pre = ar.take<int32_t>(CAP + MP);
  int32_t* d_prehn = ar.take<int32_t>(CAP + MP);
  PendScalars* d_ps = ar.take<PendScalars>(P + 4);
  Refold* d_rf = ar.take<Refold>(1);
  int32_t* d_cnt = ar.take<int32_t>(64);  // [0] n_tasks [1] n_dec [2] n_vict [3] n_preempted [4] changed
  cook_decision* d_forced = nullptr;
  int32_t* d_fvict = nullptr;
  const int NF = tr ? tr->n_forced : 0;
  if (NF > 0) {
    int nfv = 0;
    for (int q = 0; q < NF; q++) {
      const cook_decision& f = tr->forced[q];
      if (f.pending_idx < 0 || f.pending_idx >= P || f.host < 0 || f.host >= H || f.victim_count < 0 || f.victim_begin < 0)
        return set_err(pool, COOK_E_BADARG, "cook_rebalance_trace: bad forced decision");
      nfv = std::max(nfv, f.victim_begin + f.victim_count);
    }
    if (nfv > CAP + MP) return set_err(pool, COOK_E_BADARG, "cook_rebalance_trace: too many forced victims");
    d_forced = ar.take<cook_decision>(NF + 1);
    d_fvict = ar.take<int32_t>(CAP + MP);
    if (d_forced) CK(pool, cudaMemcpyAsync(d_forced, tr->forced, sizeof(cook_decision) * NF, cudaMemcpyHostToDevice, st));
    if (d_fvict && nfv > 0) CK(pool, cudaMemcpyAsync(d_fvict, tr->forced_victims, sizeof(int32_t) * nfv, cudaMemcpyHostToDevice, st));
  }
  if (ar.failed) return set_err(pool, COOK_E_OOM, "cook_rebalance: arena exhausted");
  GridFlag* d_gf = ar.take<GridFlag>(1);
  int32_t* d_syn = ar.take<int32_t>(H + 1);
  TaskHot* d_hot = ar.take<TaskHot>(CAP);
  int32_t* d_hq = ar.take<int32_t>(CAP);
  int32_t* d_synh = ar.take<int32_t>(H + 1);
  int32_t* d_synn = ar.take<int32_t>(CAP);
  WalkBar* d_bar = ar.take<WalkBar>(1);
  double* d_pm = ar.take<double>(CAP); double* d_pc = ar.take<double>(CAP);
  double* d_btm = ar.take<double>(CAP / OS_TILE + 2); double* d_btc = ar.take<double>(CAP / OS_TILE + 2);
  if (ar.failed) return set_err(pool, COOK_E_OOM, "cook_rebalance: arena exhausted");
  CK(pool, cudaMemsetAsync(d_gf, 0, sizeof(GridFlag), st));
  CK(pool, cudaMemsetAsync(d_syn, 0, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(d_synh, 0xff, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(d_bar, 0, sizeof(WalkBar), st));
  if (R > 0) grid_check_kernel<<<(R + 255) / 256, 256, 0, st>>>(t.cpus, t.mem, t.gpus, R, d_gf);
  grid_check_kernel<<<(P + 255) / 256, 256, 0, st>>>(pc.cpus, pc.mem, pc.gpus, P, d_gf);
  int32_t h_cnt[16] = {R, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  CK(pool, cudaMemcpyAsync(d_cnt, h_cnt, sizeof(h_cnt), cudaMemcpyHostToDevice, st));
  CK(pool, cudaMemsetAsync(d_ps, 0xff, sizeof(PendScalars) * (P + 4), st));   // below_quota -1, dru NaN: not reached

  CK(pool, cudaEventRecord(pool->ev[13], st));
  const int TB = 256;
  // ---- init-state: user order + DRU of every user, tasks grouped by host
  CK(pool, cudaMemsetAsync(d_us, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(d_ue, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(d_us2, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(d_ue2, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(d_hs, 0, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(d_he, 0, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(d_has_task, 0, H + 1, st));
  int launches = 0;
  if (R > 0) {
    CK(pool, csort::sort_indices(d_ord, d_tmp, R, LessUserTask{t.user, t.prio, t.start, t.tid, t.jid, d_urank}, st));
    seg_bounds_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(SortedKey{d_ord, nullptr, t.user}, R, d_us, d_ue, nullptr);
    {
      const OrderScan<double, 2> os{{d_pm, d_pc}, {d_btm, d_btc}};
      order_scan(os, LoadAlive{d_ord, t}, R, d_gf, st);
      order_dru_finish<<<(R + TB - 1) / TB, TB, 0, st>>>(d_ord, t, R, d_gf, os, d_us, d_divm, d_divc);
      launches += 3;
    }
    user_dru_kernel<<<(U + 3) / 4, 128, 0, st>>>(d_ord, t, d_divm, d_divc, d_us, d_ue, U, d_gf, R);
    CK(pool, csort::sort_indices(d_hord, d_tmp, R, LessHost{t}, st));
    seg_bounds_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(SortedKey{d_hord, nullptr, t.host}, R, d_hs, d_he, nullptr);
    host_has_task_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(t, R, d_has_task);
    hot_build_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(d_hord, t, d_urank, R, d_hot, d_hq);
    launches += 7;
    for (long long w = csort::TILE; w < R; w <<= 1) launches += 2;
  }
  // ---- the walk over the pending jobs: one cooperative launch, no host round trip inside
  RebArgs ra;
  ra.t = t; ra.R = R;
  ra.ord[0] = d_ord; ra.ord[1] = d_ord2; ra.us[0] = d_us; ra.us[1] = d_us2; ra.ue[0] = d_ue; ra.ue[1] = d_ue2;
  ra.hord = d_hord; ra.hs = d_hs; ra.he = d_he;
  ra.hc = hc; ra.pc = pc; ra.gc = gc; ra.P = P; ra.U = U; ra.MP = MP;
  ra.user_rank = d_urank; ra.div_mem = d_divm; ra.div_cpus = d_divc;
  ra.q_count = d_qn; ra.q_cpus = d_qc; ra.q_mem = d_qm; ra.q_gpus = d_qg;
  ra.has_task = d_has_task; ra.preempted_hosts = d_pre; ra.preempted_hn = d_prehn;
  ra.min_diff = prm->min_dru_diff; ra.safe = prm->safe_dru_threshold; ra.host_lifetime_mins = prm->host_lifetime_mins;
  ra.best = d_best; ra.cta_best = d_cta; ra.dec = d_dec; ra.victims = d_vict; ra.cnt = d_cnt; ra.rf = d_rf;
  ra.ps_all = d_ps; ra.gf = d_gf; ra.syn_cnt = d_syn; ra.hot = d_hot; ra.hq = d_hq; ra.syn_head = d_synh; ra.syn_next = d_synn; ra.bar = d_bar;
  ra.n_forced = NF; ra.forced = d_forced; ra.forced_victims = d_fvict; ra.forced_only = tr ? tr->forced_only : 0;
  {
    int occ = 0;
    CK(pool, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rebalance_kernel, REB_TB, 0));
    if (occ < 1) return set_err(pool, COOK_E_CUDA, "cook_rebalance: kernel does not fit on an SM");
    // a warp per host in the host phase: as many co-resident CTAs as help (<= 3 per SM)
    int per_sm = 1;   // measured: more CTAs shorten the host phase but lengthen the barriers by as much
    if (const char* e = getenv("COOK_REB_CTAS_PER_SM")) per_sm = std::max(1, std::min(occ, atoi(e)));
    int grid = std::min(per_sm * pool->sm_count, std::max(1, (H + REB_TB / 32 - 1) / (REB_TB / 32)));
    void* kargs[] = {&ra};
    CK(pool, cudaEventRecord(pool->ev[19], st));
    CK(pool, cudaLaunchCooperativeKernel((void*)rebalance_kernel, dim3(grid), dim3(REB_TB), kargs, 0, st));
    launches++;
  }
  CK(pool, cudaEventRecord(pool->ev[14], st));
  CK(pool, cudaMemcpyAsync(h_cnt, d_cnt, sizeof(int32_t) * 5, cudaMemcpyDeviceToHost, st));
  CK(pool, cudaStreamSynchronize(st));
  if (getenv("COOK_PROF")) {
    int32_t hp[10];
    CK(pool, cudaMemcpy(hp, d_cnt + 8, sizeof(hp), cudaMemcpyDeviceToHost));
    float pre = 0.f, walk = 0.f;
    if (R > 0 && P > 0) { cudaEventElapsedTime(&pre, pool->ev[13], pool->ev[19]); cudaEventElapsedTime(&walk, pool->ev[19], pool->ev[14]); }
    fprintf(stderr, "[cook_prof] rebalance kcycles (CTA 0): hosts %d (scalars+groups %d)  next-state %d  refold %d  grid-sync %d | setup %.3f ms walk %.3f ms\n",
            hp[0], hp[4], hp[1], hp[2], hp[3], pre, walk);
    fprintf(stderr, "[cook_prof]   next-state split: argmax+victim selection %d  victims %d  bookkeeping %d  insertion search %d (argmax alone %d)\n", hp[5], hp[6], hp[7], hp[8], hp[9]);
  }
  const int n_dec = h_cnt[1], n_tasks = h_cnt[0];
  if (n_dec > 0) {
    CK(pool, cudaMemcpyAsync(out_decisions, d_dec, sizeof(cook_decision) * n_dec, cudaMemcpyDeviceToHost, st));
    if (h_cnt[2] > 0)
      CK(pool, cudaMemcpyAsync(out_victims, d_vict, sizeof(int32_t) * h_cnt[2], cudaMemcpyDeviceToHost, st));
  }
  if (tr) {   // the state the reference's own tests read (K18 pending dru, K21 next-state, job-below-quota)
    std::vector<PendScalars> hps(P);
    std::vector<double> hdru(n_tasks);
    std::vector<uint8_t> halive(n_tasks);
    std::vector<int32_t> hpos(n_tasks), huser(n_tasks);
    CK(pool, cudaMemcpyAsync(hps.data(), d_ps, sizeof(PendScalars) * P, cudaMemcpyDeviceToHost, st));
    if (n_tasks > 0) {
      CK(pool, cudaMemcpyAsync(hdru.data(), t.dru, sizeof(double) * n_tasks, cudaMemcpyDeviceToHost, st));
      CK(pool, cudaMemcpyAsync(halive.data(), t.alive, n_tasks, cudaMemcpyDeviceToHost, st));
      CK(pool, cudaMemcpyAsync(hpos.data(), t.pos, sizeof(int32_t) * n_tasks, cudaMemcpyDeviceToHost, st));
      CK(pool, cudaMemcpyAsync(huser.data(), t.user, sizeof(int32_t) * n_tasks, cudaMemcpyDeviceToHost, st));
    }
    if (tr->has_spare) CK(pool, cudaMemcpyAsync(tr->has_spare, hc.has_spare, H, cudaMemcpyDeviceToHost, st));
    if (tr->spare_mem) CK(pool, cudaMemcpyAsync(tr->spare_mem, hc.spare_mem, sizeof(double) * H, cudaMemcpyDeviceToHost, st));
    if (tr->spare_cpus) CK(pool, cudaMemcpyAsync(tr->spare_cpus, hc.spare_cpus, sizeof(double) * H, cudaMemcpyDeviceToHost, st));
    if (tr->spare_gpus) CK(pool, cudaMemcpyAsync(tr->spare_gpus, hc.spare_gpus, sizeof(double) * H, cudaMemcpyDeviceToHost, st));
    CK(pool, cudaStreamSynchronize(st));
    for (int p = 0; p < P; p++) {
      if (hps[p].below_quota < 0) continue;   // the walk did not reach this job
      if (tr->pending_dru) tr->pending_dru[p] = hps[p].pending_dru;
      if (tr->below_quota) tr->below_quota[p] = hps[p].below_quota ? 1 : 0;
    }
    std::vector<int32_t> order;
    for (int i = 0; i < n_tasks; i++) {
      if (tr->task_dru) tr->task_dru[i] = hdru[i];
      if (tr->task_alive) tr->task_alive[i] = halive[i];
      if (halive[i]) order.push_back(i);
    }
    // priority-map order (:252-256): (-dru, user name); equal (dru, user): later position first (ours)
    std::sort(order.begin(), order.end(), [&](int x, int y) {
      if (hdru[x] != hdru[y]) return hdru[x] > hdru[y];
      if (huser[x] != huser[y]) return users->name_rank[huser[x]] < users->name_rank[huser[y]];
      return hpos[x] > hpos[y];
    });
    if (tr->order) for (size_t i = 0; i < order.size(); i++) tr->order[i] = order[i];
    if (tr->n_order) *tr->n_order = (int32_t)order.size();
  }
  CK(pool, cudaEventRecord(pool->ev[15], st));
  CK(pool, cudaStreamSynchronize(st));
  {
    cook_phase_stats& ps = pool->phase[COOK_PHASE_REBALANCE];
    ps.ms_h2d = ev_ms(pool->ev[12], pool->ev[13]);
    ps.ms_device = ev_ms(pool->ev[13], pool->ev[14]);
    ps.ms_d2h = ev_ms(pool->ev[14], pool->ev[15]);
    ps.h2d_bytes = (int64_t)R * 60 + (int64_t)P * 48 + (int64_t)H * 48 + (int64_t)U * 60;
    ps.d2h_bytes = (int64_t)n_dec * (int64_t)sizeof(cook_decision) + (int64_t)h_cnt[2] * 4 + 20;
    ps.n_launches = launches;
  }
  *out_n = n_dec;
  return COOK_OK;
}

extern "C" int32_t cook_rebalance(cook_pool* pool, const cook_running_soa* running,
                                  const cook_jobs_soa* pending, const int64_t* pending_job_id,
                                  const int32_t* pending_priority, const cook_host_table* hosts,
                                  const cook_groups* groups, const cook_user_table* users,
                                  const cook_rebalance_params* prm, cook_decision* out_decisions,
                                  int32_t* out_victims, int32_t* out_n) {
  return rebalance_run(pool, running, pending, pending_job_id, pending_priority, hosts, groups, users, prm,
                       out_decisions, out_victims, out_n, nullptr);
}

extern "C" int32_t cook_rebalance_trace(cook_pool* pool, const cook_running_soa* running,
                                        const cook_jobs_soa* pending, const int64_t* pending_job_id,
                                        const int32_t* pending_priority, const cook_host_table* hosts,
                                        const cook_groups* groups, const cook_user_table* users,
                                        const cook_rebalance_params* prm, cook_decision* out_decisions,
                                        int32_t* out_victims, int32_t* out_n, const cook_reb_trace* tr) {
  if (!tr) return set_err(pool, COOK_E_BADARG, "cook_rebalance_trace: null trace");
  return rebalance_run(pool, running, pending, pending_job_id, pending_priority, hosts, groups, users, prm,
                       out_decisions, out_victims, out_n, tr);
}
