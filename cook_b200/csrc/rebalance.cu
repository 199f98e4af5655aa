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
#include <type_traits>

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

// caller-written rows: each victim as its task id (a synthetic one as -1 - the decision that placed it: the
// walk appends decision e's task at index R + e), each decision's job id
__global__ void victim_ids_kernel(const int32_t* cnt, const int32_t* victims, const int64_t* tid, int R,
                                  const cook_decision* dec, const int64_t* jid, int64_t* out_tid, int64_t* out_jid) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < cnt[2]) {
    const int i = victims[k];
    out_tid[k] = i < R ? tid[i] : -1 - (int64_t)(i - R);
  }
  if (k < cnt[1]) out_jid[k] = jid[dec[k].pending_idx];
}

}  // namespace

// One rebalance's device buffers (carved by rebalance_build from the pool's arena) and what its run needs.
struct RebPlan {
  int R = 0, P = 0, H = 0, U = 0, MP = 0, CAP = 0, NF = 0;
  bool zero_gpus = false;   // no gpus column uploaded: the task gpus are zeros
  bool ids = false;         // caller-written rows: report task ids and job ids
  const cook_reb_trace* tr = nullptr;
  const cook_user_table* users = nullptr;
  cook_rebalance_params prm = {};
  RTasks t = {};
  HostCols hc = {};
  PendCols pc = {};
  GroupCols gc = {};
  int32_t *d_urank, *d_ord, *d_ord2, *d_hord, *d_tmp, *d_us, *d_ue, *d_us2, *d_ue2, *d_hs, *d_he, *d_vict, *d_pre, *d_prehn;
  int32_t *d_cnt, *d_fvict = nullptr, *d_syn, *d_hq, *d_synh, *d_synn;
  double *d_divm, *d_divc, *d_qn, *d_qc, *d_qm, *d_qg, *d_pm, *d_pc, *d_btm, *d_btc;
  uint8_t* d_has_task;
  HostBest* d_best;
  CtaBest* d_cta;
  cook_decision *d_dec, *d_forced = nullptr;
  PendScalars* d_ps;
  Refold* d_rf;
  GridFlag* d_gf;
  TaskHot* d_hot;
  WalkBar* d_bar;
  int64_t *d_vtid = nullptr, *d_djid = nullptr;
  int64_t h2d = 0;
};

void RebPlanFree::operator()(RebPlan* p) const { delete p; }

// The build: the call's buffers, carved from one description of its rows.  Host tables (sh.running) are
// uploaded in the same pass; otherwise the running and pending columns are carved for the caller to write.
// The host table, the users' rebalance columns and the groups are uploaded either way.
static int32_t build(cook_pool* pool, const RebShape& sh, const cook_host_table* hosts, const cook_groups* groups,
                     const cook_user_table* users, const cook_rebalance_params* prm, const cook_reb_trace* tr,
                     RebPlan& q) {
  static const cook_running_soa no_running = {};
  static const cook_jobs_soa no_pending = {};
  const bool up = sh.running != nullptr;
  const cook_tasks_soa& rt = (up ? sh.running : &no_running)->t;
  const cook_running_soa& running = up ? *sh.running : no_running;
  const cook_jobs_soa& pending = up ? *sh.pending : no_pending;
  const int R = sh.R, P = sh.P, H = hosts->n, U = users->n_users, MP = prm->max_preemption;
  const int G = groups ? groups->n_groups : 0;
  const int CAP = R + MP + 1;
  const int NF = tr ? tr->n_forced : 0;
  int nfv = 0;   // forced victims (checked by the caller)
  for (int k = 0; k < NF; k++) nfv = std::max(nfv, tr->forced[k].victim_begin + tr->forced[k].victim_count);
  q.R = R; q.P = P; q.H = H; q.U = U; q.MP = MP; q.CAP = CAP; q.NF = NF;
  q.zero_gpus = up && !rt.gpus; q.ids = !up; q.tr = tr; q.users = users; q.prm = *prm;
  RTasks& t = q.t;
  HostCols& hc = q.hc;
  PendCols& pc = q.pc;
  GroupCols& gc = q.gc;
  hc.H = H;
  hc.n_attr_cols = hosts->attr ? hosts->n_attr_cols : 0;
  const bool novel = up ? pending.novel_off != nullptr : sh.n_novel > 0;
  const bool attr = up ? pending.attr_off != nullptr : sh.n_attr > 0;
  const bool grouped = G && (up ? pending.group_off != nullptr : sh.n_group > 0);
  CK(pool, cudaSetDevice(pool->device));
  const cudaError_t carved = carve(pool->arena, pool->stream, pool->ev[12], &q.h2d, [&](Carve& c) {
    // a running column: the host's R rows in CAP, or CAP for the caller; a pending column likewise
    const auto run_col = [&](auto* host) {
      using T = std::remove_const_t<std::remove_pointer_t<decltype(host)>>;
      return up ? c.part(host, (size_t)R, (size_t)CAP) : c.take<T>(CAP);
    };
    const auto pend_col = [&](auto* host, size_t n) {
      using T = std::remove_const_t<std::remove_pointer_t<decltype(host)>>;
      return up ? c.up(host, n) : c.take<T>(n);
    };
    t.user = run_col(rt.user); t.prio = run_col(rt.priority); t.start = run_col(rt.start_time);
    t.tid = run_col(rt.task_id); t.jid = run_col(rt.job_id); t.cpus = run_col(rt.cpus);
    t.mem = run_col(rt.mem); t.gpus = rt.gpus ? run_col(rt.gpus) : c.take<double>(CAP);
    t.host = run_col(running.host);
    t.alive = c.take<uint8_t>(CAP); t.dru = c.take<double>(CAP); t.pos = c.take<int32_t>(CAP);
    t.cm = c.take<double>(CAP); t.cc = c.take<double>(CAP);

    q.d_urank = c.up(users->name_rank, U); q.d_divm = c.up(users->div_mem, U); q.d_divc = c.up(users->div_cpus, U);
    q.d_qn = c.up(users->quota_count, U); q.d_qc = c.up(users->quota_cpus, U); q.d_qm = c.up(users->quota_mem, U);
    q.d_qg = c.up(users->quota_gpus, U);

    hc.hostname_id = c.up(hosts->hostname_id, H); hc.name_rank = c.up(hosts->name_rank, H);
    hc.has_spare = c.part(hosts->has_spare, H, H + 1, true); hc.spare_cpus = c.part(hosts->spare_cpus, H, H + 1, true);
    hc.spare_mem = c.part(hosts->spare_mem, H, H + 1, true); hc.spare_gpus = c.part(hosts->spare_gpus, H, H + 1, true);
    hc.is_k8s = c.up(hosts->is_k8s, H);
    hc.location = c.up(hosts->location, H);
    if (hosts->gpu_off) {
      const int n = std::max(1, hosts->gpu_off[H]);
      hc.gpu_off = c.up(hosts->gpu_off, H + 1); hc.gpu_model = c.up(hosts->gpu_model, n); hc.gpu_count = c.up(hosts->gpu_count, n);
    }
    if (hosts->disk_off) {
      const int n = std::max(1, hosts->disk_off[H]);
      hc.disk_off = c.up(hosts->disk_off, H + 1); hc.disk_type = c.up(hosts->disk_type, n); hc.disk_space = c.up(hosts->disk_space, n);
    }
    hc.host_start = c.up(hosts->host_start_time, H);
    if (hc.n_attr_cols > 0) hc.attr = c.up(hosts->attr, (size_t)hc.n_attr_cols * H);

    pc.user = pend_col(pending.user, P); pc.prio = pend_col(sh.priority, P);
    pc.cpus = pend_col(pending.cpus, P); pc.mem = pend_col(pending.mem, P); pc.gpus = pend_col(pending.gpus, P);
    pc.jid = pend_col(sh.job_id, P); pc.est_end_ms = pend_col(pending.est_end_ms, P);
    if (novel) {
      pc.novel_off = pend_col(pending.novel_off, P + 1);
      pc.novel_host = pend_col(pending.novel_host, std::max<int64_t>(1, up ? pending.novel_off[P] : sh.n_novel));
    }
    pc.gpu_model = pend_col(pending.gpu_model, P); pc.disk_type = pend_col(pending.disk_type, P);
    pc.ckpt_location = pend_col(pending.ckpt_location, P);
    pc.disk_request = pend_col(pending.disk_request, P);
    if (attr) {
      const int64_t n = std::max<int64_t>(1, up ? pending.attr_off[P] : sh.n_attr);
      pc.attr_off = pend_col(pending.attr_off, P + 1); pc.attr_col = pend_col(pending.attr_col, n); pc.attr_val = pend_col(pending.attr_val, n);
    }
    if (grouped) {
      pc.group_off = pend_col(pending.group_off, P + 1);
      pc.group_idx = pend_col(pending.group_idx, std::max<int64_t>(1, up ? pending.group_off[P] : sh.n_group));
      gc.n = G;
      gc.kind = c.up(groups->kind, G); gc.attr_col = c.up(groups->attr_col, G);
      gc.minimum = c.up(groups->minimum, G);
      if (sh.dev.cot) {   // derived by the caller on the device
        const size_t n = std::max<int64_t>(1, sh.dev.n_cot);
        gc.cot_off = c.take<int32_t>(G + 1); gc.cot_host = c.take<int32_t>(n); gc.cot_attr = c.take<int32_t>(n);
      } else {
        gc.cot_off = c.up(groups->cot_off, G + 1);
        const int n = std::max(1, groups->cot_off[G]);
        gc.cot_host = c.up(groups->cot_hostname_id, n); gc.cot_attr = c.up(groups->cot_attr_val, n);
      }
    }

    q.d_ord = c.take<int32_t>(CAP); q.d_ord2 = c.take<int32_t>(CAP);
    q.d_hord = c.take<int32_t>(CAP);
    q.d_tmp = c.take<int32_t>(CAP);
    q.d_us = c.take<int32_t>(U + 1); q.d_ue = c.take<int32_t>(U + 1);
    q.d_us2 = c.take<int32_t>(U + 1); q.d_ue2 = c.take<int32_t>(U + 1);
    q.d_hs = c.take<int32_t>(H + 1); q.d_he = c.take<int32_t>(H + 1);
    q.d_has_task = c.take<uint8_t>(H + 1);
    q.d_best = c.take<HostBest>(H + 1);
    q.d_cta = c.take<CtaBest>(4 * pool->sm_count + 8);
    q.d_dec = c.take<cook_decision>(MP + 1);
    q.d_vict = c.take<int32_t>(CAP + MP);
    q.d_pre = c.take<int32_t>(CAP + MP);
    q.d_prehn = c.take<int32_t>(CAP + MP);
    q.d_ps = c.take<PendScalars>(P + 4);
    q.d_rf = c.take<Refold>(1);
    q.d_cnt = c.take<int32_t>(64);  // [0] n_tasks [1] n_dec [2] n_vict [3] n_preempted [4] changed
    if (NF > 0) {
      q.d_forced = c.part(tr->forced, NF, NF + 1);
      q.d_fvict = c.part(tr->forced_victims, nfv, CAP + MP);
    }
    q.d_gf = c.take<GridFlag>(1);
    q.d_syn = c.take<int32_t>(H + 1);
    q.d_hot = c.take<TaskHot>(CAP);
    q.d_hq = c.take<int32_t>(CAP);
    q.d_synh = c.take<int32_t>(H + 1);
    q.d_synn = c.take<int32_t>(CAP);
    q.d_bar = c.take<WalkBar>(1);
    q.d_pm = c.take<double>(CAP); q.d_pc = c.take<double>(CAP);
    q.d_btm = c.take<double>(CAP / OS_TILE + 2); q.d_btc = c.take<double>(CAP / OS_TILE + 2);
    if (q.ids) { q.d_vtid = c.take<int64_t>(CAP + MP); q.d_djid = c.take<int64_t>(MP + 1); }
  });
  CK(pool, carved);
  return COOK_OK;
}

// The run: the grid checks, init-state (sorts, initial fold, host grouping), the walk, the download.
static int32_t run(cook_pool* pool, RebPlan& q, cook_decision* out_decisions, int32_t* out_victims,
                   int64_t* out_victim_tid, int64_t* out_decision_jid, int32_t* out_n) {
  cudaStream_t st = pool->stream;
  const int R = q.R, P = q.P, H = q.H, U = q.U, MP = q.MP, CAP = q.CAP, NF = q.NF;
  const cook_reb_trace* tr = q.tr;
  const cook_rebalance_params* prm = &q.prm;
  const cook_user_table* users = q.users;
  RTasks& t = q.t;
  HostCols& hc = q.hc;
  int64_t d2h = 0;
  if (q.zero_gpus) CK(pool, cudaMemsetAsync(t.gpus, 0, sizeof(double) * CAP, st));
  CK(pool, cudaMemsetAsync(t.alive, 0, CAP, st));
  if (R) CK(pool, cudaMemsetAsync(t.alive, 1, R, st));
  CK(pool, cudaMemsetAsync(t.dru, 0, sizeof(double) * CAP, st));
  CK(pool, cudaMemsetAsync(q.d_gf, 0, sizeof(GridFlag), st));
  CK(pool, cudaMemsetAsync(q.d_syn, 0, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(q.d_synh, 0xff, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(q.d_bar, 0, sizeof(WalkBar), st));
  int launches = 0;
  if (R > 0) {
    grid_check_kernel<<<(R + 255) / 256, 256, 0, st>>>(t.cpus, t.mem, t.gpus, R, q.d_gf);
    launches++;
  }
  grid_check_kernel<<<(P + 255) / 256, 256, 0, st>>>(q.pc.cpus, q.pc.mem, q.pc.gpus, P, q.d_gf);
  launches++;
  int32_t h_cnt[16] = {R, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  CK(pool, cudaMemcpyAsync(q.d_cnt, h_cnt, sizeof(h_cnt), cudaMemcpyHostToDevice, st));
  CK(pool, cudaMemsetAsync(q.d_ps, 0xff, sizeof(PendScalars) * (P + 4), st));   // below_quota -1, dru NaN: not reached

  CK(pool, cudaEventRecord(pool->ev[13], st));
  const int TB = 256;
  // ---- init-state: user order + DRU of every user, tasks grouped by host
  CK(pool, cudaMemsetAsync(q.d_us, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(q.d_ue, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(q.d_us2, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(q.d_ue2, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(q.d_hs, 0, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(q.d_he, 0, sizeof(int32_t) * (H + 1), st));
  CK(pool, cudaMemsetAsync(q.d_has_task, 0, H + 1, st));
  if (R > 0) {
    CK(pool, csort::sort_indices(q.d_ord, q.d_tmp, R, LessUserTask{t.user, t.prio, t.start, t.tid, t.jid, q.d_urank}, st, &launches));
    seg_bounds_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(SortedKey{q.d_ord, nullptr, t.user}, R, q.d_us, q.d_ue, nullptr);
    launches++;
    {
      const OrderScan<double, 2> os{{q.d_pm, q.d_pc}, {q.d_btm, q.d_btc}};
      order_scan(os, LoadAlive{q.d_ord, t}, R, q.d_gf, st, &launches);
      order_dru_finish<<<(R + TB - 1) / TB, TB, 0, st>>>(q.d_ord, t, R, q.d_gf, os, q.d_us, q.d_divm, q.d_divc);
      launches++;
    }
    user_dru_kernel<<<(U + 3) / 4, 128, 0, st>>>(q.d_ord, t, q.d_divm, q.d_divc, q.d_us, q.d_ue, U, q.d_gf, R);
    launches++;
    CK(pool, csort::sort_indices(q.d_hord, q.d_tmp, R, LessHost{t}, st, &launches));
    seg_bounds_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(SortedKey{q.d_hord, nullptr, t.host}, R, q.d_hs, q.d_he, nullptr);
    host_has_task_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(t, R, q.d_has_task);
    hot_build_kernel<<<(R + TB - 1) / TB, TB, 0, st>>>(q.d_hord, t, q.d_urank, R, q.d_hot, q.d_hq);
    launches += 3;
  }
  // ---- the walk over the pending jobs: one cooperative launch, no host round trip inside
  RebArgs ra;
  ra.t = t; ra.R = R;
  ra.ord[0] = q.d_ord; ra.ord[1] = q.d_ord2; ra.us[0] = q.d_us; ra.us[1] = q.d_us2; ra.ue[0] = q.d_ue; ra.ue[1] = q.d_ue2;
  ra.hord = q.d_hord; ra.hs = q.d_hs; ra.he = q.d_he;
  ra.hc = hc; ra.pc = q.pc; ra.gc = q.gc; ra.P = P; ra.U = U; ra.MP = MP;
  ra.user_rank = q.d_urank; ra.div_mem = q.d_divm; ra.div_cpus = q.d_divc;
  ra.q_count = q.d_qn; ra.q_cpus = q.d_qc; ra.q_mem = q.d_qm; ra.q_gpus = q.d_qg;
  ra.has_task = q.d_has_task; ra.preempted_hosts = q.d_pre; ra.preempted_hn = q.d_prehn;
  ra.min_diff = prm->min_dru_diff; ra.safe = prm->safe_dru_threshold; ra.host_lifetime_mins = prm->host_lifetime_mins;
  ra.best = q.d_best; ra.cta_best = q.d_cta; ra.dec = q.d_dec; ra.victims = q.d_vict; ra.cnt = q.d_cnt; ra.rf = q.d_rf;
  ra.ps_all = q.d_ps; ra.gf = q.d_gf; ra.syn_cnt = q.d_syn; ra.hot = q.d_hot; ra.hq = q.d_hq; ra.syn_head = q.d_synh;
  ra.syn_next = q.d_synn; ra.bar = q.d_bar;
  ra.n_forced = NF; ra.forced = q.d_forced; ra.forced_victims = q.d_fvict; ra.forced_only = tr ? tr->forced_only : 0;
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
  if (q.ids) {
    victim_ids_kernel<<<(CAP + MP + 255) / 256, 256, 0, st>>>(q.d_cnt, q.d_vict, t.tid, R, q.d_dec, q.pc.jid, q.d_vtid,
                                                             q.d_djid);
    launches++;
    CK(pool, cudaGetLastError());
  }
  CK(pool, cudaEventRecord(pool->ev[14], st));
  CK(pool, download(h_cnt, q.d_cnt, 5, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  if (getenv("COOK_PROF")) {
    int32_t hp[10];
    CK(pool, cudaMemcpy(hp, q.d_cnt + 8, sizeof(hp), cudaMemcpyDeviceToHost));
    float pre = 0.f, walk = 0.f;
    if (R > 0 && P > 0) { cudaEventElapsedTime(&pre, pool->ev[13], pool->ev[19]); cudaEventElapsedTime(&walk, pool->ev[19], pool->ev[14]); }
    fprintf(stderr, "[cook_prof] rebalance kcycles (CTA 0): hosts %d (scalars+groups %d)  next-state %d  refold %d  grid-sync %d | setup %.3f ms walk %.3f ms\n",
            hp[0], hp[4], hp[1], hp[2], hp[3], pre, walk);
    fprintf(stderr, "[cook_prof]   next-state split: argmax+victim selection %d  victims %d  bookkeeping %d  insertion search %d (argmax alone %d)\n", hp[5], hp[6], hp[7], hp[8], hp[9]);
  }
  const int n_dec = h_cnt[1], n_tasks = h_cnt[0];
  if (n_dec > 0) {
    CK(pool, download(out_decisions, q.d_dec, n_dec, st, &d2h));
    if (q.ids) {
      CK(pool, download(out_decision_jid, q.d_djid, n_dec, st, &d2h));
      if (h_cnt[2] > 0) CK(pool, download(out_victim_tid, q.d_vtid, h_cnt[2], st, &d2h));
    } else if (h_cnt[2] > 0) {
      CK(pool, download(out_victims, q.d_vict, h_cnt[2], st, &d2h));
    }
  }
  if (tr) {   // the state the reference's own tests read (K18 pending dru, K21 next-state, job-below-quota)
    std::vector<PendScalars> hps(P);
    std::vector<double> hdru(n_tasks);
    std::vector<uint8_t> halive(n_tasks);
    std::vector<int32_t> hpos(n_tasks), huser(n_tasks);
    CK(pool, download(hps.data(), q.d_ps, P, st, &d2h));
    if (n_tasks > 0) {
      CK(pool, download(hdru.data(), t.dru, n_tasks, st, &d2h));
      CK(pool, download(halive.data(), t.alive, n_tasks, st, &d2h));
      CK(pool, download(hpos.data(), t.pos, n_tasks, st, &d2h));
      CK(pool, download(huser.data(), t.user, n_tasks, st, &d2h));
    }
    if (tr->has_spare) CK(pool, download(tr->has_spare, hc.has_spare, H, st, &d2h));
    if (tr->spare_mem) CK(pool, download(tr->spare_mem, hc.spare_mem, H, st, &d2h));
    if (tr->spare_cpus) CK(pool, download(tr->spare_cpus, hc.spare_cpus, H, st, &d2h));
    if (tr->spare_gpus) CK(pool, download(tr->spare_gpus, hc.spare_gpus, H, st, &d2h));
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
  record_phase(pool, COOK_PHASE_REBALANCE, pool->ev[12], pool->ev[13], pool->ev[14], pool->ev[15], q.h2d, d2h, launches);
  *out_n = n_dec;
  return COOK_OK;
}

int32_t rebalance_build(cook_pool* pool, const RebShape& sh, const cook_host_table* hosts, const cook_groups* groups,
                        const cook_user_table* users, const cook_rebalance_params* prm, RebPlanPtr* plan,
                        RebRows* rows) {
  plan->reset(new RebPlan());
  RebPlan& q = **plan;
  const int32_t rc = build(pool, sh, hosts, groups, users, prm, nullptr, q);
  if (rc != COOK_OK) return rc;
  const PendCols& pc = q.pc;
  rows->t = TaskCols{q.t.user, q.t.prio, q.t.start, q.t.tid, q.t.jid, q.t.cpus, q.t.mem, q.t.gpus};
  rows->host = q.t.host;
  rows->jb = JobDev{};
  JobDev& jb = rows->jb;
  jb.user = pc.user; jb.cpus = pc.cpus; jb.mem = pc.mem; jb.gpus = pc.gpus;
  jb.novel_off = pc.novel_off; jb.novel_host = pc.novel_host; jb.gpu_model = pc.gpu_model;
  jb.disk_request = pc.disk_request; jb.disk_type = pc.disk_type;
  jb.attr_off = pc.attr_off; jb.attr_col = pc.attr_col; jb.attr_val = pc.attr_val;
  jb.est_end_ms = pc.est_end_ms; jb.ckpt_location = pc.ckpt_location;
  jb.group_off = pc.group_off; jb.group_idx = pc.group_idx;
  rows->jid = pc.jid; rows->prio = pc.prio;
  rows->hostname_id = q.hc.hostname_id;
  rows->attr = q.hc.attr;
  rows->gcol = q.gc.attr_col;
  const bool cot = sh.dev.cot && q.gc.cot_off;
  rows->cot_off = cot ? writable(q.gc.cot_off) : nullptr;
  rows->cot_host = cot ? writable(q.gc.cot_host) : nullptr;
  rows->cot_attr = cot ? writable(q.gc.cot_attr) : nullptr;
  return COOK_OK;
}

int32_t rebalance_run(cook_pool* pool, RebPlan& plan, cook_decision* out_decisions, int64_t* out_victim_tid,
                      int64_t* out_decision_jid, int32_t* out_n) {
  return run(pool, plan, out_decisions, nullptr, out_victim_tid, out_decision_jid, out_n);
}

// cook_rebalance(_trace) on host tables: the checks, then build and run
static int32_t rebalance_host(cook_pool* pool, const cook_running_soa* running,
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
  const int G = groups ? groups->n_groups : 0;
  if (G && pending->group_off && (!groups->cot_off || !groups->kind))
    return set_err(pool, COOK_E_BADARG, "cook_rebalance: incomplete cook_groups");
  const int CAP = R + MP + 1;
  const int NF = tr ? tr->n_forced : 0;
  int nfv = 0;   // forced victims
  for (int q = 0; q < NF; q++) {
    const cook_decision& f = tr->forced[q];
    if (f.pending_idx < 0 || f.pending_idx >= P || f.host < 0 || f.host >= H || f.victim_count < 0 || f.victim_begin < 0)
      return set_err(pool, COOK_E_BADARG, "cook_rebalance_trace: bad forced decision");
    nfv = std::max(nfv, f.victim_begin + f.victim_count);
  }
  if (nfv > CAP + MP) return set_err(pool, COOK_E_BADARG, "cook_rebalance_trace: too many forced victims");
  RebShape sh;
  sh.R = R; sh.P = P;
  sh.running = running; sh.pending = pending; sh.job_id = pending_job_id; sh.priority = pending_priority;
  RebPlan q;
  const int32_t rc = build(pool, sh, hosts, groups, users, prm, tr, q);
  if (rc != COOK_OK) return rc;
  return run(pool, q, out_decisions, out_victims, nullptr, nullptr, out_n);
}

extern "C" int32_t cook_rebalance(cook_pool* pool, const cook_running_soa* running,
                                  const cook_jobs_soa* pending, const int64_t* pending_job_id,
                                  const int32_t* pending_priority, const cook_host_table* hosts,
                                  const cook_groups* groups, const cook_user_table* users,
                                  const cook_rebalance_params* prm, cook_decision* out_decisions,
                                  int32_t* out_victims, int32_t* out_n) {
  return rebalance_host(pool, running, pending, pending_job_id, pending_priority, hosts, groups, users, prm,
                        out_decisions, out_victims, out_n, nullptr);
}

extern "C" int32_t cook_rebalance_trace(cook_pool* pool, const cook_running_soa* running,
                                        const cook_jobs_soa* pending, const int64_t* pending_job_id,
                                        const int32_t* pending_priority, const cook_host_table* hosts,
                                        const cook_groups* groups, const cook_user_table* users,
                                        const cook_rebalance_params* prm, cook_decision* out_decisions,
                                        int32_t* out_victims, int32_t* out_n, const cook_reb_trace* tr) {
  if (!tr) return set_err(pool, COOK_E_BADARG, "cook_rebalance_trace: null trace");
  return rebalance_host(pool, running, pending, pending_job_id, pending_priority, hosts, groups, users, prm,
                        out_decisions, out_victims, out_n, tr);
}
