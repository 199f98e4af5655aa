// match.cu — considerable-job filter (M0) and the exact greedy best-fit matcher
// (M3/M4) on the GPU.  Replaces pending-jobs->considerable-jobs
// (scheduler/scheduler.clj:729-762, tools.clj:903-973) and Fenzo's
// TaskScheduler.scheduleOnce as Cook calls it (scheduler.clj:665-671) with
// good-enough-fitness >= 1.0 (every VM evaluated for every task).
//
// Exactness on a parallel machine (SURVEY H1).  Fenzo places requests one at a
// time; each placement mutates one VM and may change every later argmax.  One
// persistent cooperative launch keeps that order and splits the work:
//
//   evaluators (all CTAs but #0): one CTA per job scores ALL offers against a
//     SNAPSHOT of the dynamic VM state and emits, per chunk of offers (VM v is in
//     chunk v mod 32), the sorted top-TOPK (fitness, v) pairs: the job's ROW.
//   resolver (CTA 0): walks the jobs in rank order.  Every placement is appended to
//     a commit LOG in shared memory; VMs in the log since the row's snapshot are
//     re-evaluated exactly, every other VM is unchanged, so the row's clean
//     candidates are still exact.  Warp roles (driver / spec / commit) pipeline
//     that work; only "evaluate the job on the VM the previous job just changed,
//     compare, append" is serial (see the resolver section below and DESIGN.md 4).
//
//   The two sides are software-pipelined: while the resolver places block t the
//   evaluators score block t+1 against the state published after block t-1
//   (double-buffered snapshot, two monotone counters, no grid barrier).
//
// Tie-break: equal fitness => lowest hostname (offers are index-sorted by
// name_rank on upload, so "lowest v").  All f64 ops are IEEE in the reference's
// order (-fmad=false; divisions via correctly rounded reciprocals, see div_y):
// identical to oracle/cook_oracle.cpp eval_pair bit for bit.
#include <cooperative_groups.h>

#include <algorithm>
#include <mutex>
#include <numeric>

#include "constraints.cuh"
#include "fold.cuh"
#include "sort.cuh"

namespace {

constexpr int RES_THREADS = 512;   // threads per CTA of the match kernel
constexpr int TOPK = 8;            // candidates kept per (job, chunk)
constexpr int ROW_V_OFF = TOPK * 32 * 8;             // byte offset of the v part of a row
constexpr int ROW_BYTES = TOPK * 32 * (8 + 4);       // 3072 B per job

// Per-VM state is AoS, 32 B per record, so one record is two 128-bit loads and a
// clean candidate's state can be staged with 16-byte async copies.
struct __align__(32) VmStatic { double lc, lm, rc, rm; };
// Dynamic record: cpus/mem assigned this cycle + the (static) correctly rounded
// reciprocals of the fitness denominators, yc = RN(1/(lc+rc)), ym = RN(1/(lm+rm)):
// x/den is then q0 = x*y, q = fma(fma(-den, q0, x), y, q0) == RN(x/den) (Markstein's
// correction; checked against IEEE division in tests/test_fastdiv.py); y == 0 marks
// denominators outside the safe range (true division is used for those).
struct __align__(32) VmDyn { double ac, am, yc, ym; };
struct __align__(8) VmCnt { int an, pu; };  // tasks assigned this cycle, ports used (constraint kernel)

// Offer-side inputs of the hard constraints, one 48 B record per VM (rank space).
struct __align__(16) VmCons {
  int hostname_id, location, max_tasks, num_tasks;          // -1 = absent (location, max_tasks)
  int run_count, flags, gpu_lo, ports_total;                // flags: bit0 k8s, bit1 reserved, bits 8.. #gpu models
  long long host_start;                                     // -1 = absent
  int disk_lo, disk_n;
};
enum { VC_K8S = 1, VC_RESERVED = 2 };

struct VmState {  // everything one fit evaluation needs about a VM
  double ac, am, lc, lm, rc, rm, yc, ym;
  int an, pu;
  // constraint kernel, resolver only: the static inputs of the count-dependent checks
  int room;   // max-tasks-per-host minus tasks already on the host (INT_MAX = no limit)
  int occ;    // tasks running on the host before this cycle (a gpu job needs occ + an == 0)
  int ptot;   // ports offered
};

struct OfferDev {
  int O;
  // hot columns, gathered into rank-sorted index space v
  const VmStatic* vs;   // {lease cpus, lease mem, running cpus, running mem} per VM
  const int32_t* perm;  // v -> original offer index
  // constraint columns, ORIGINAL index space (may be null)
  const int32_t* hostname_id;
  const int32_t* run_count;
  const int32_t* ports_total;  // computed on device; null when no ports
  const int32_t* port_off; const int32_t* port_begin; const int32_t* port_end;
  const uint8_t* is_k8s;
  const int32_t* location;
  const int32_t* gpu_off; const int32_t* gpu_model; const double* gpu_count;
  const int32_t* disk_off; const int32_t* disk_type; const double* disk_space;
  const int32_t* max_tasks; const int32_t* num_tasks;
  const int64_t* host_start;
  int n_attr_cols; const int32_t* attr;
  const uint8_t* reserved;
  // rank space (index v), built on the device per cycle: everything the constraints need
  // about a VM in three 128-bit loads + the attribute table gathered by v
  const struct VmCons* vc;
  const int32_t* attr_v;   // [n_attr_cols][O]
};

struct GroupDev {
  int n_groups;
  const int32_t* kind; const int32_t* attr_col; const int32_t* minimum;
  const int32_t* cot_off; const int32_t* cot_host; const int32_t* cot_attr;
  const int32_t* gp_off;  // capacity offsets of per-group placed lists
  int32_t* gp_n;          // dynamic count per group
  int32_t* gp_vm;         // placed VM (v space)
};

struct DynBuf {  // dynamic per-VM state, index space v, double buffered
  VmDyn* d[2];
  VmCnt* n[2];
};

struct MatchArgs {
  JobDev jb;
  OfferDev of;
  GroupDev gr;
  DynBuf dyn;
  int n_cons;
  const int32_t* cons;     // k -> job index
  const double* kc;        // gathered cpus per k
  const double* km;        // gathered mem per k
  const uint8_t* kflags;   // bit0: has groups
  int B;                   // jobs per block at the start (blocks 0 and 1)
  int bmin, bmax, btarget; // adaptive blocks: bounds and target placements per block
  int32_t* bk0;            // [max blocks + 4] first job of block b (bk0[b+1] = end); resolver writes ahead
  int host_lifetime_mins;
  unsigned char* rows;     // [2][B][ROW_BYTES]: f[TOPK][32] f64 then v[TOPK][32] i32
  const double* kg;        // gathered gpus per k (constraint kernel)
  const double* smin_c;    // suffix minima of kc / km: the smallest request among jobs k..n_cons-1
  const double* smin_m;
  const int32_t* kports;   // gathered port counts per k
  int32_t* feas;           // [2][bmax] block + 1 once any VM is feasible for the row at the snapshot
  int vs_in_smem;          // evaluators keep the static VM table in shared memory
  int sparse_ok;           // evaluators may score rows over the compacted live-VM lists (COOK_NO_SPARSE=1 disables)
  // constraint kernel: one bit per (row, VM) = "the VM passed every check at the row's snapshot"
  // (two blocks of rows, like `rows`); all checks only tighten within a cycle, so the resolver
  // re-evaluates a changed VM as bit && resources && the three count-dependent checks
  unsigned* sbits;
  int sb_words;            // words per row = ceil(O / 32); 0 in the plain kernel
  unsigned* rows_ready;    // [nblk] rows scored per block
  unsigned* published;     // # blocks resolved and published
  int32_t* assign;         // [n_cons] v (rank space) or -1
  int32_t* ports_start;    // [n_cons] ports_used of the VM before assignment
  uint8_t* fail;           // [n_cons]
  unsigned long long* stats;  // [0]=fast [1]=chunk rescans [2]=group jobs [3]=matched [4]=fallbacks [5]=truncated specs [6]=skipped
  int* latest_global;         // newest-log-entry table when it does not fit in shared memory
  int lookahead;              // queue entries in flight (<= RING)
  int poll_ns;                // back-off of the resolver's shared-memory polling loops
  int max_spec_warp;          // spec warps of a spec CTA are warps 2 .. max_spec_warp - 1
  int spec_kmin;              // candidate rounds stop once this many candidates are out
  // ---- spec CTAs (blocks 1 .. n_spec): the resolver's log, replicated through global memory
  int n_spec;                 // thread blocks that only compute candidate sets
  struct LogEnt* glog;        // [LOGN] copy of the commit log (publisher warp -> follower warps)
  int4* glogx;                // [LOGN] constraint kernel: {room, occ, ptot, -}
  unsigned long long* gchain; // the chain word as published (entries below its log size are in glog)
  int32_t* lo_g;              // [max blocks] lo_g[b] = log size at the start of block b
  struct SpecOut* gres;       // [GRING] candidate sets on their way to the resolver (fetched with cp.async.bulk)
  unsigned* gres_seq;         // [GRING] g + 1 once the result of queue entry g is complete
  int32_t* dead_blk;          // b + 1 once no VM can take even the smallest request from block b on
  int32_t* dead_k0;           // first job of that block (-1 while unknown): finalize marks the rest
};

// ------------------------------------------------------------------ helpers
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// ---- mbarrier + bulk async copy (TMA engine, no tensor map): the resolver receives the
// spec CTAs' candidate sets with cp.async.bulk completing on an mbarrier its commit warps sleep on
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// potentially blocking: the warp sleeps in hardware until the phase completes or ~hint_ns pass
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity, unsigned hint_ns) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(hint_ns) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

struct JobRegs {  // per-job values the hot loop keeps in registers
  double c, m, g;
  int j, ports;
};

template <bool CONSTR>
__device__ __forceinline__ JobRegs load_job(const MatchArgs& a, int k) {
  JobRegs r;
  r.c = a.kc[k]; r.m = a.km[k];
  r.j = a.cons[k];
  r.g = 0.0; r.ports = 0;
  if (CONSTR) {
    r.g = a.kg[k];
    r.ports = a.kports[k];
  }
  return r;
}

// Static + count-dependent hard constraints of one (job, VM) pair in Cook's evaluation order (see
// oracle eval_pair; constraints.clj): -1, or the index of the first failing check (0 checkpoint
// locality, 1 estimated completion, 2 user-defined attribute equals, 3 disk, 4 gpu host, 5 novel host,
// 6 max tasks per host, 7 reservation).  Group constraints are first_failing_group's.
// `an` = tasks assigned to the VM this cycle.
__device__ int first_failing_constraint(const MatchArgs& a, const JobRegs& r, int v, int an) {
  const JobDev& jb = a.jb;
  const OfferDev& of = a.of;
  const int j = r.j;
  // the VM's record: three independent 128-bit loads, issued before any check
  const int4* vcp = reinterpret_cast<const int4*>(of.vc + v);
  const int4 c0 = __ldg(vcp), c1 = __ldg(vcp + 1), c2 = __ldg(vcp + 2);
  const int hostname = c0.x, location = c0.y, max_tasks = c0.z, num_tasks = c0.w;
  const int run_count = c1.x, flags = c1.y, gpu_lo = c1.z;
  const long long host_start = ((long long)(unsigned)c2.y << 32) | (unsigned)c2.x;
  const int disk_lo = c2.z, disk_n = c2.w;
  const int gpu_n = flags >> 8;
  if (jb.ckpt_location && jb.ckpt_location[j] >= 0) {
    if (location != jb.ckpt_location[j]) return 0;
  }
  if (jb.est_end_ms && jb.est_end_ms[j] >= 0 && host_start >= 0) {
    long long death = 1000LL * host_start + 60000LL * a.host_lifetime_mins;
    if (!(jb.est_end_ms[j] < death)) return 1;
  }
  if (jb.attr_off) {
    for (int k = jb.attr_off[j]; k < jb.attr_off[j + 1]; k++) {
      int col = jb.attr_col[k], val = jb.attr_val[k];
      if (col < 0 || col >= of.n_attr_cols) return 2;
      int hv = of.attr_v[(size_t)col * of.O + v];
      if (val <= 0 || hv != val) return 2;
    }
  }
  const bool k8s = flags & VC_K8S;
  if (jb.disk_request && jb.disk_request[j] >= 0.0 && k8s) {
    const int want = jb.disk_type ? jb.disk_type[j] : -1;
    double space = 0.0;
    for (int i = 0; i < disk_n; i++)
      if (of.disk_type[disk_lo + i] == want) { space = of.disk_space[disk_lo + i]; break; }
    if (!(space >= jb.disk_request[j])) return 3;
  }
  if (k8s) {
    if (r.g > 0.0) {
      const int want = jb.gpu_model ? jb.gpu_model[j] : -1;
      double have = 0.0;
      for (int i = 0; i < gpu_n; i++)
        if (of.gpu_model[gpu_lo + i] == want) { have = of.gpu_count[gpu_lo + i]; break; }
      int on_vm = run_count + an;
      if (!(have == r.g && on_vm == 0)) return 4;
    } else {
      if (gpu_n != 0) return 4;
    }
  } else if (!(r.g == 0.0)) {
    return 4;
  }
  if (jb.novel_off) {
    for (int k = jb.novel_off[j]; k < jb.novel_off[j + 1]; k++)
      if (jb.novel_host[k] == hostname) return 5;
  }
  if (max_tasks >= 0) {
    int total = num_tasks + an;
    if (!(total < max_tasks)) return 6;
  }
  if (flags & VC_RESERVED) {
    int mine = jb.reserved_host ? jb.reserved_host[j] : -1;
    if (mine != hostname) return 7;
  }
  return -1;
}

__device__ __forceinline__ int vm_attr(const OfferDev& of, int col, int v) {
  return (col >= 0 && col < of.n_attr_cols) ? of.attr_v[(size_t)col * of.O + v] : 0;
}

// Group constraints of job j on VM v (constraints.clj:586-678): -1, or the index of the first failing
// one.  A group's known members are its running cotasks, then the first n_placed(g) entries of the
// group's placed list.  The resolver appends to that list in queue order, so the members placed by the
// jobs before turn k are a prefix of it.
template <class Placed>
__device__ __forceinline__ int first_failing_group(const MatchArgs& a, int j, int v, Placed n_placed) {
  const JobDev& jb = a.jb;
  const GroupDev& gr = a.gr;
  const OfferDev& of = a.of;
  for (int k = jb.group_off[j]; k < jb.group_off[j + 1]; k++) {
    const int g = jb.group_idx[k];
    const int kind = gr.kind[g];
    const int c0 = gr.cot_off[g], nc = gr.cot_off[g + 1] - c0;
    const int p0 = gr.gp_off[g], n = nc + n_placed(g);
    auto placed = [&](int i) { return __ldcg(gr.gp_vm + p0 + i - nc); };
    int f;
    if (kind == COOK_GROUP_UNIQUE) {   // cotasks by hostname, this cycle's members by VM
      const int h = of.vc[v].hostname_id;
      f = group_fail(kind, n, h, 0, [&](int i) { return i < nc ? gr.cot_host[c0 + i] : (placed(i) == v ? h : ~h); });
    } else {
      const int col = gr.attr_col[g];
      f = group_fail(kind, n, vm_attr(of, col, v), gr.minimum[g],
                     [&](int i) { return i < nc ? gr.cot_attr[c0 + i] : vm_attr(of, col, placed(i)); });
    }
    if (f >= 0) return f;
  }
  return -1;
}

// against the live group state: every member placed so far
__device__ bool group_pass(const MatchArgs& a, const JobRegs& r, int v) {
  return first_failing_group(a, r.j, v, [&](int g) { return __ldcg(a.gr.gp_n + g); }) < 0;
}

// x / den with y = RN(1 / den) (or 0 => plain division): three dependent f64 ops
// instead of the ~10 of div.rn.f64, same correctly rounded result.
__device__ __forceinline__ double div_y(double x, double den, double y) {
  if (y == 0.0) return x / den;
  const double q0 = x * y;
  return fma(fma(-den, q0, x), y, q0);
}
// (y = 0 selects the IEEE division in div_y.)  The Markstein correction is proven for a faithful q0 and a
// denominator whose significand is not all ones; such denominators take the plain division as well.
__device__ __forceinline__ double safe_rcp(double den) {
  const unsigned long long frac = (unsigned long long)__double_as_longlong(den) & 0x000fffffffffffffULL;
  return (den > 1e-100 && den < 1e100 && frac != 0x000fffffffffffffULL) ? 1.0 / den : 0.0;
}

// FENZO 3a + 4 (see oracle): resource fit then cpuMemBinPacker fitness.
// The usual case (both reciprocals usable) takes no branch between the two divisions, so their
// dependent chains interleave: on the commit chain that is one 7-op f64 path instead of two 5-op ones
// each fenced by a branch to the IEEE division.  Same operations, same results.
__device__ __forceinline__ double fit_fitness(double jc, double jm, const VmState& st) {
  const bool no = (st.ac + jc > st.lc) | (st.am + jm > st.lm);
  double cpu_fit, mem_fit;
  if (st.yc != 0.0 && st.ym != 0.0) {
    const double xc = (jc + st.ac) + st.rc, xm = (jm + st.am) + st.rm;
    const double qc = xc * st.yc, qm = xm * st.ym;
    cpu_fit = fma(fma(-(st.lc + st.rc), qc, xc), st.yc, qc);
    mem_fit = fma(fma(-(st.lm + st.rm), qm, xm), st.ym, qm);
  } else {
    cpu_fit = div_y((jc + st.ac) + st.rc, st.lc + st.rc, st.yc);
    mem_fit = div_y((jm + st.am) + st.rm, st.lm + st.rm, st.ym);
  }
  return no ? 0.0 : (cpu_fit + mem_fit) * 0.5;
}

// Full evaluation of (job, VM v) against an explicit VM state.
template <bool CONSTR>
__device__ __forceinline__ double eval_vm(const MatchArgs& a, const JobRegs& r, int v, const VmState& st,
                                          bool with_groups) {
  if (CONSTR) {
    if (st.ac + r.c > st.lc) return 0.0;
    if (st.am + r.m > st.lm) return 0.0;
    if (r.ports > 0) {
      const int tot = a.of.vc[v].ports_total;
      if (r.ports > tot - st.pu) return 0.0;
    }
    if (first_failing_constraint(a, r, v, st.an) >= 0) return 0.0;
    if (with_groups && !group_pass(a, r, v)) return 0.0;
  }
  return fit_fitness(r.c, r.m, st);
}

// state of VM v at the snapshot of block blk (global memory / L2)
template <bool CONSTR>
__device__ __forceinline__ VmState load_snap(const MatchArgs& a, int blk, int v) {
  const double2* st2 = reinterpret_cast<const double2*>(a.of.vs + v);
  const double2* dy2 = reinterpret_cast<const double2*>(a.dyn.d[blk & 1] + v);
  const double2 s0 = __ldg(st2), s1 = __ldg(st2 + 1);
  const double2 d0 = __ldcg(dy2), d1 = __ldcg(dy2 + 1);
  VmState st;
  st.ac = d0.x; st.am = d0.y; st.yc = d1.x; st.ym = d1.y;
  st.lc = s0.x; st.lm = s0.y; st.rc = s1.x; st.rm = s1.y;
  st.an = 0; st.pu = 0;
  st.room = 0x7fffffff; st.occ = 0; st.ptot = 0;
  if (CONSTR) {
    const int2 c = __ldcg(reinterpret_cast<const int2*>(a.dyn.n[blk & 1] + v));
    st.an = c.x; st.pu = c.y;
    const int4* vcp = reinterpret_cast<const int4*>(a.of.vc + v);
    const int4 c0 = __ldg(vcp), c1 = __ldg(vcp + 1);   // {.., max_tasks, num_tasks}, {run_count, .., ports_total}
    st.room = c0.z >= 0 ? c0.z - c0.w : 0x7fffffff;
    st.occ = c1.x; st.ptot = c1.w;
  }
  return st;
}

// Resolver-side evaluation of (job, VM v) against an explicit state.  Constraint kernel:
// `sbit` is the evaluators' verdict for the pair at the row's snapshot (every static check
// passed and the VM fitted then); resources and the count-dependent checks -- ports, a gpu
// job's empty host, max-tasks-per-host -- only tighten during a cycle, so the verdict at
// the new state is sbit && those checks, with no constraint input read from global memory.
template <bool CONSTR>
__device__ __forceinline__ double eval_res(const MatchArgs& a, const JobRegs& r, int v, const VmState& st,
                                           bool with_groups, bool sbit) {
  if (CONSTR) {
    if (!sbit) return 0.0;
    if (st.ac + r.c > st.lc) return 0.0;
    if (st.am + r.m > st.lm) return 0.0;
    if (r.ports > 0 && r.ports > st.ptot - st.pu) return 0.0;
    if (r.g > 0.0 && st.occ + st.an != 0) return 0.0;
    if (!(st.an < st.room)) return 0.0;
    if (with_groups && !group_pass(a, r, v)) return 0.0;
  }
  return fit_fitness(r.c, r.m, st);
}
__device__ __forceinline__ bool sb_global(const unsigned* row, int v) { return (__ldcg(row + (v >> 5)) >> (v & 31)) & 1u; }
__device__ __forceinline__ bool sb_shared(const unsigned* row, int v) { return (row[v >> 5] >> (v & 31)) & 1u; }

// ------------------------------------------------------------- evaluators
// One CTA scores one job against ALL offers of a snapshot.  The offers are cut
// into tiles of 32 consecutive VMs; tile t belongs to CHUNK t mod 32 and a warp
// owns whole chunks (warp w: chunks w, w + NW, ...), so the per-chunk top-TOPK
// lists of a row need no cross-warp merge and no CTA barrier: lane i of the
// owning warp scores VM 32*t + i of every tile of the chunk, keeps its own
// sorted top-TOPK, and TOPK warp-argmax rounds emit the chunk's list.
//   row[k]: f[TOPK][32 chunks] f64 then v[TOPK][32 chunks] i32, sorted per chunk
//   feas[k] = generation stamp (block + 1) once any VM is feasible for the job
// The static VM table {lease cpus/mem, running cpus/mem} lives in shared memory
// (SoA, loaded once per CTA) when it fits; the dynamic state is read from L2 with
// all loads of a batch in flight.
constexpr int NW = 16;  // evaluator warps per CTA (warps beyond NW only exist for the resolver CTA's roles)
static_assert(32 % NW == 0 && NW * 32 <= RES_THREADS, "a warp owns 32 / NW chunks");
constexpr int CPW = 32 / NW;  // chunks per warp

__device__ __forceinline__ bool better(double f, int v, double g, int w) {
  return f > g || (f == g && v < w);
}

__device__ __forceinline__ double warp_max_f64(double f) {  // f >= 0
  unsigned hi = (unsigned)__double2hiint(f);
  unsigned mh = __reduce_max_sync(0xffffffffu, hi);
  unsigned lo = hi == mh ? (unsigned)__double2loint(f) : 0u;
  unsigned ml = __reduce_max_sync(0xffffffffu, lo);
  return __hiloint2double((int)mh, (int)ml);
}

// argmax over lanes of (f desc, key asc); key < 0xffffffff.  Returns the winning
// fitness (0 => nobody), wk = its key, wl = its lane.
__device__ __forceinline__ double warp_argmax(double f, unsigned key, unsigned& wk, int& wl) {
  const double wf = warp_max_f64(f);
  const unsigned k2 = (f == wf && wf > 0.0) ? key : 0xffffffffu;
  wk = __reduce_min_sync(0xffffffffu, k2);
  wl = __ffs(__ballot_sync(0xffffffffu, k2 == wk)) - 1;
  return wf;
}


struct EvalStatic {  // static VM table in shared memory (SoA), or null => global
  const double* lc; const double* lm; const double* rc; const double* rm;
};

// per-CTA exchange buffer: every warp's per-lane partial lists of one row.  The sizes of EvalShared, SparseLive
// and ResolverShared set the offer counts where match_run moves the static VM table and latest[] to global
// memory; tests/match_edge_cases.py builds cases on either side of those counts from the sizes it records
// (SMEM_STATIC_O, LATEST_O): change them together.
struct EvalShared {
  double f[NW][TOPK][32];
  int32_t v[NW][TOPK][32];
  int any[NW];
};

// Once most VMs are full, a row only has to look at the LIVE ones.  Per block every evaluator CTA
// compacts the live VMs of each chunk (chunk = v mod 32 = lane) into a short list in shared
// memory; when every list fits (SL_MAX entries) the rows of the block are scored over the lists
// instead of over all tiles (rows of a saturated cluster: a handful of evaluations per thread).
constexpr int SL_MAX = 64;        // live VMs per chunk in sparse mode
constexpr int SBW_MAX = 1024;     // verdict-bit words staged in shared memory (sparse mode, constraint kernel)
struct SparseLive {
  unsigned short t[32][SL_MAX];   // tile index of the i-th live VM of chunk c: v = 32 * t + c
  int cnt[32];
  int maxc;                       // max over chunks; sparse mode iff maxc <= SL_MAX
  unsigned sb[SBW_MAX];           // one row's verdict bits being assembled
};

template <bool CONSTR, bool PROF>
__device__ void evaluate_row(const MatchArgs& a, const JobRegs& r, const bool grp, int blk, int ib,
                             const EvalStatic& es, EvalShared& E, const unsigned long long live,
                             unsigned long long* ep, SparseLive& SP, const bool sparse) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long e0 = PROF ? clock64() : 0;
  const double2* st2 = reinterpret_cast<const double2*>(a.of.vs);
  const double2* dy2 = reinterpret_cast<const double2*>(a.dyn.d[blk & 1]);  // S_{b-2} = buffer b&1
  unsigned char* row = a.rows + ((size_t)(blk & 1) * a.bmax + ib) * ROW_BYTES;
  double* rf = reinterpret_cast<double*>(row);
  int32_t* rv = reinterpret_cast<int32_t*>(row + ROW_V_OFF);
  unsigned* sbrow = CONSTR ? a.sbits + ((size_t)(blk & 1) * a.bmax + ib) * a.sb_words : nullptr;
  // (1) every warp scans its tiles (32 consecutive VMs, coalesced): VM v belongs to chunk
  // v mod 32 = lane, so equal-fitness runs of consecutive VMs spread over all chunks
  double f[TOPK];
  int vv[TOPK];
#pragma unroll
  for (int i = 0; i < TOPK; i++) { f[i] = 0.0; vv[i] = 0x7fffffff; }
  if (sparse) {
    if (CONSTR) {   // the row's verdict bits are assembled in shared memory (live VMs only; the rest is 0)
      for (int wd = threadIdx.x; wd < a.sb_words; wd += NW * 32) SP.sb[wd] = 0u;
      __syncthreads();
    }
    const int nl = SP.cnt[lane];
    for (int i0 = warp; i0 < SP.maxc; i0 += 2 * NW) {   // warp-uniform trip count, two VMs in flight
      VmState st[2];
      int vq[2];
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int i = i0 + u * NW;
        vq[u] = i < nl ? 32 * (int)SP.t[lane][i] + lane : -1;
        st[u].ac = st[u].am = st[u].yc = st[u].ym = st[u].lc = st[u].lm = st[u].rc = st[u].rm = 0.0;
        st[u].an = st[u].pu = 0;
        if (vq[u] >= 0) {
          const int v = vq[u];
          const double2 d0 = __ldcg(dy2 + 2 * v), d1 = __ldcg(dy2 + 2 * v + 1);
          st[u].ac = d0.x; st[u].am = d0.y; st[u].yc = d1.x; st[u].ym = d1.y;
          if (CONSTR) {
            const int2 cn = __ldcg(reinterpret_cast<const int2*>(a.dyn.n[blk & 1] + v));
            st[u].an = cn.x; st[u].pu = cn.y;
          }
          if (es.lc) { st[u].lc = es.lc[v]; st[u].lm = es.lm[v]; st[u].rc = es.rc[v]; st[u].rm = es.rm[v]; }
          else {
            const double2 s0 = __ldg(st2 + 2 * v), s1 = __ldg(st2 + 2 * v + 1);
            st[u].lc = s0.x; st[u].lm = s0.y; st[u].rc = s1.x; st[u].rm = s1.y;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int v = vq[u];
        double x = 0.0;
        if (v >= 0) x = eval_vm<CONSTR>(a, r, v, st[u], false);
        if (CONSTR && x > 0.0) atomicOr(&SP.sb[v >> 5], 1u << (v & 31));
        // the lists are unordered: ties are resolved on v explicitly
        if (x > 0.0 && better(x, v, f[TOPK - 1], vv[TOPK - 1])) {
          f[TOPK - 1] = x; vv[TOPK - 1] = v;
#pragma unroll
          for (int i = TOPK - 1; i > 0; i--) {
            if (better(f[i], vv[i], f[i - 1], vv[i - 1])) {
              double tf = f[i]; f[i] = f[i - 1]; f[i - 1] = tf;
              int tv = vv[i]; vv[i] = vv[i - 1]; vv[i - 1] = tv;
            }
          }
        }
      }
    }
  } else {
    const int O = a.of.O;
    constexpr int U = 4;  // VMs in flight per lane
    int ui = 0;  // index of the lane's VM (bit of `live`)
    for (int base = 32 * warp; base < O; base += U * 32 * NW, ui += U) {  // warp-uniform trip count
      const int v0 = base + lane;
      // VMs that cannot take even the smallest remaining job are dead for the rest of the
      // cycle: a lane (and often the whole warp) skips their loads
      const unsigned lb = ui < 64 ? (unsigned)((live >> ui) & ((1u << U) - 1u)) : ((1u << U) - 1u);
      if (!__any_sync(0xffffffffu, lb != 0u)) {
        if (CONSTR && lane < U && base + lane * 32 * NW < O) __stcg(sbrow + (base >> 5) + lane * NW, 0u);
        continue;
      }
      VmState st[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const int v = v0 + u * 32 * NW;
        st[u].ac = st[u].am = st[u].yc = st[u].ym = st[u].lc = st[u].lm = st[u].rc = st[u].rm = 0.0;
        st[u].an = st[u].pu = 0;
        if (v < O && ((lb >> u) & 1u)) {
          const double2 d0 = __ldcg(dy2 + 2 * v), d1 = __ldcg(dy2 + 2 * v + 1);
          st[u].ac = d0.x; st[u].am = d0.y; st[u].yc = d1.x; st[u].ym = d1.y;
          if (CONSTR) {
            const int2 cn = __ldcg(reinterpret_cast<const int2*>(a.dyn.n[blk & 1] + v));
            st[u].an = cn.x; st[u].pu = cn.y;
          }
          if (es.lc) { st[u].lc = es.lc[v]; st[u].lm = es.lm[v]; st[u].rc = es.rc[v]; st[u].rm = es.rm[v]; }
          else {
            const double2 s0 = __ldg(st2 + 2 * v), s1 = __ldg(st2 + 2 * v + 1);
            st[u].lc = s0.x; st[u].lm = s0.y; st[u].rc = s1.x; st[u].rm = s1.y;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const int v = v0 + u * 32 * NW;
        if (base + u * 32 * NW >= O) break;   // warp-uniform: the tile does not exist
        double x = 0.0;
        if (v < O && ((lb >> u) & 1u)) x = eval_vm<CONSTR>(a, r, v, st[u], false);
        if (CONSTR) {
          const unsigned m = __ballot_sync(0xffffffffu, x > 0.0);
          if (lane == 0) __stcg(sbrow + (base >> 5) + u * NW, m);
        }
        if (x > f[TOPK - 1]) {  // v ascends within a lane: strict > keeps the lower v on ties
          f[TOPK - 1] = x; vv[TOPK - 1] = v;
#pragma unroll
          for (int i = TOPK - 1; i > 0; i--) {
            if (f[i] > f[i - 1]) {
              double tf = f[i]; f[i] = f[i - 1]; f[i - 1] = tf;
              int tv = vv[i]; vv[i] = vv[i - 1]; vv[i - 1] = tv;
            }
          }
        }
      }
    }
  }
  const bool wany = __any_sync(0xffffffffu, f[0] > 0.0);
  if (wany) {
#pragma unroll
    for (int i = 0; i < TOPK; i++) { E.f[warp][i][lane] = f[i]; E.v[warp][i][lane] = vv[i]; }
  }
  if (lane == 0) E.any[warp] = wany ? 1 : 0;
  long long e1 = PROF ? clock64() : 0;
  __syncthreads();
  if (CONSTR && sparse)
    for (int wd = threadIdx.x; wd < a.sb_words; wd += NW * 32) __stcg(sbrow + wd, SP.sb[wd]);
  // (2) warp w merges chunks w, w + NW, ...: the NW partial lists of a chunk (sorted, TOPK
  // each) are spread over the lanes, TOPK warp-argmax rounds emit the chunk's sorted list
  bool any = false;
#pragma unroll
  for (int w = 0; w < NW; w++) any |= E.any[w] != 0;
  if (any) {
    constexpr int PER = NW * TOPK / 32;  // entries per lane
    static_assert(NW * TOPK % 32 == 0 && TOPK % PER == 0, "partial lists split evenly over the lanes");
#pragma unroll 1
    for (int ci = 0; ci < CPW; ci++) {
      const int c = warp + ci * NW;
      const int sw = lane / (TOPK / PER), so = (lane % (TOPK / PER)) * PER;  // source warp, first entry
      double lf[PER];
      int lv[PER];
#pragma unroll
      for (int j = 0; j < PER; j++) {
        const bool has = E.any[sw] != 0;
        lf[j] = has ? E.f[sw][so + j][c] : 0.0;
        lv[j] = has ? E.v[sw][so + j][c] : 0x7fffffff;
      }
      double of = 0.0;
      int ov = -1;
#pragma unroll 1
      for (int i = 0; i < TOPK; i++) {
        unsigned wk;
        int wl;
        const double wf = warp_argmax(lf[0], (unsigned)lv[0], wk, wl);
        if (!(wf > 0.0)) break;
        if (lane == i) { of = wf; ov = (int)wk; }
        if (lane == wl) {
#pragma unroll
          for (int q = 0; q < PER - 1; q++) { lf[q] = lf[q + 1]; lv[q] = lv[q + 1]; }
          lf[PER - 1] = 0.0; lv[PER - 1] = 0x7fffffff;
        }
      }
      if (lane < TOPK) {
        __stcg(rf + lane * 32 + c, of);
        __stcg(rv + lane * 32 + c, ov);
      }
    }
  }
  long long e2 = PROF ? clock64() : 0;
  __syncthreads();  // row complete; E may be rewritten
  if (threadIdx.x == 0) {
    // feasibility stamp: block + 1 (stale stamps of the buffer's previous blocks are smaller).
    // Group constraints are not applied here (they depend on same-cycle placements): the row of
    // a group job lists its best VMs without them and the resolver filters against live state.
    if (any) atomicMax(a.feas + (size_t)(blk & 1) * a.bmax + ib, blk + 1);
    // the release orders the CTA's row stores (made visible to this thread by the barrier)
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(a.rows_ready + blk), "r"(1u) : "memory");
  }
  if (PROF) {
    long long e3 = clock64();
    ep[0] += (unsigned long long)(e1 - e0); ep[1] += (unsigned long long)(e2 - e1);
    ep[2] += (unsigned long long)(e3 - e2);
  }
}

// --------------------------------------------------------------- resolver
// CTA 0 resolves the jobs in rank order, exactly, as a pipeline of warp roles:
//
//   driver (warp 1)   turns the evaluators' per-block feasibility stamps into an
//                     in-order QUEUE of entries (JOB / END-of-block / EXIT); at
//                     most `lookahead` entries are in flight.
//   spec (most warps) each takes the next queue ticket and computes, against the
//                     state at some VERSION s (= commits it saw), a candidate set of
//                     the job: clean chunk candidates from the job's row merged with
//                     an exact re-evaluation of every VM committed since the row's
//                     snapshot (the commit LOG, an append-only ring), plus a bound z
//                     on everything left out.
//   commit (warps 0..3, one per SM scheduler) own the entries round-robin and form
//                     the serial chain.  Before its turn the owner re-evaluates the VMs
//                     committed since s (one lane per log entry) and reduces its lanes'
//                     items to an exact, warp-uniform top-3; entries that appear while it
//                     waits are folded in with scalar code.  At its turn exactly the newest
//                     log entry is new: every lane evaluates it redundantly, the winner is
//                     the better of it and the best listed item it did not supersede - no
//                     warp collective on the chain - and is appended to the log.
//
// Constraint kernel: the evaluators also emit one verdict bit per (job, VM) ("passed every
// check at the row's snapshot"); all checks only tighten within a cycle, so the resolver
// re-evaluates a changed VM as bit && resources && the count-dependent checks whose static
// inputs travel with the log entry (eval_res) - it reads no constraint input from global
// memory.  Group constraints stay dynamic (group_pass against the live group state).
//
// Validity of a log entry e for VM x is `latest[x] == e` (latest[] = index of
// the newest entry per VM, monotone), so nothing is ever cleared: a VM is dirty
// with respect to a block's snapshot iff latest[x] >= lo, lo = log size at the
// start of the previous block.
constexpr int MAXB = 512;             // max jobs per block
constexpr int LOGN = 2 * MAXB;        // commit-log ring (entries of two blocks)
constexpr int RING = 32;              // queue entries / spec results in flight
constexpr int GRING = 64;             // candidate sets in flight between the spec CTAs and the resolver (global)
constexpr int MAX_SPEC_CTAS = 8;
constexpr int KC = 16;                // candidates per spec result
#ifndef COOK_LK
#define COOK_LK 4
#endif
constexpr int LK = COOK_LK;           // entries a lane keeps while building a result
#ifndef COOK_NCW
#define COOK_NCW 5
#endif
// Commit warps.  Each owns every NCW-th turn and does its off-turn work (result, first look, folds) in
// the NCW - 1 turns before it; with four, the owner was still folding an older entry when its turn came
// in over half of C2's turns.  Constraint pools keep four: each of their commit warps holds the current
// job's verdict bit for every offer in shared memory, and those rows bound the pool's offer count.
constexpr int NCW_PLAIN = COOK_NCW, NCW_CONSTR = 4;
constexpr int NCW_MAX = NCW_PLAIN > NCW_CONSTR ? NCW_PLAIN : NCW_CONSTR;

enum { Q_JOB = 0, Q_END = 1, Q_EXIT = 2 };

// newest log entry per VM: in shared memory when it fits (the usual case), else global
struct Latest {
  int* s;  // shared (derived from the dynamic shared base so loads/stores stay LDS/STS)
  int* g;  // global fallback
  __device__ __forceinline__ int get(int v) const { return g ? g[v] : s[v]; }
  __device__ __forceinline__ void set(int v, int e) const { if (g) g[v] = e; else s[v] = e; }
};

// Per-turn timeline of the PROF instantiation (COOK_PROF=1 with COOK_PROF_TRACE=<file>): null unless the
// host armed it.  turn_trace[g] = TURN_WORDS stamps of queue entry g (clock64 of the resolver SM, so every
// role of CTA 0 is on one clock); blk_trace[b] = when the driver saw every row of block b scored.
// TT_HAND: 1 << 32 | the low word of the clock when the owner learned that turn g-1 had ended (0: not
// stamped); TT_POLL: how often the owner waited for a turn to end before that (low word) | 1 << 32 when
// it learned it right after folding an older entry.
constexpr int TURN_WORDS = 12;
enum { TT_FREE = 0, TT_LAND, TT_READY, TT_SEEN, TT_DONE, TT_FENCE, TT_INFO, TT_K, TT_EVAL, TT_DEC, TT_HAND, TT_POLL };
enum { TP_EXACT = 0, TP_ZTAKE = 1, TP_FALLBACK = 2, TP_GROUP = 3 };
__device__ unsigned long long* g_turn_trace;
__device__ int g_turn_cap;
__device__ unsigned long long* g_blk_trace;
__device__ int g_blk_cap;

__device__ __forceinline__ void fence_cta() { asm volatile("fence.acq_rel.cta;" ::: "memory"); }
// Readers of the resolver's shared flags: shared-memory loads of one warp complete in
// program order, so polling needs no hardware fence - only the compiler must not move
// the data loads above the (volatile) flag load.
__device__ __forceinline__ void compiler_barrier() { asm volatile("" ::: "memory"); }

struct QEntry {
  int type, blk, k, lo;
  double jc, jm, jg;
  int jports, jj, grp, row;   // row: index of the job inside its block
};

// One log entry, 80 B: a lane reads it with five 128-bit loads (conflict-free at
// this stride when 8 consecutive entries are read by 8 lanes).
struct __align__(16) LogEnt {
  int vm, an, pu, k;
  double ac, am, lc, lm, rc, rm, yc, ym;
};

struct Cand {  // one candidate VM with its state at the result's version
  double f;
  VmState st;
  int vm, e;
};

struct __align__(16) SpecOut {
  int type, s, n, complete;  // type: Q_JOB / Q_END / Q_EXIT (the commit warps wait on the result flag only)
  double zf;                 // bound: every unchanged VM outside c[] is no better than (zf, zv)
  int gver, pad;             // group-state version the result was computed against (group jobs)
  int zv, z_real;            // z_real: (zf, zv) is the exact fitness of VM zv (state in c[KC]), not just a bound
  Cand c[KC + 1];            // unsorted; c[KC] = the bound VM when z_real
};

static_assert(sizeof(SpecOut) % 16 == 0, "candidate sets travel with cp.async.bulk (16 B granules)");
static_assert(RING == 32, "the fetcher warp owns one result slot per lane");

// Shared state of the resolver CTA; the spec CTAs keep a replica of the log / queue part.
struct ResolverShared {
  LogEnt log[LOGN];
  int4 logx[LOGN];                // constraint kernel: {room, occ, ptot, -} of the entry's VM
  QEntry q[RING];
  SpecOut res[RING + 1];          // [RING] = the commit warps' fallback slot
  unsigned long long res_bar[RING];  // mbarrier per result slot: phase (g / RING) & 1 completes when the
                                     // result of entry g has landed (bulk copy) or the entry is END / EXIT
  unsigned long long hand[NCW_MAX];  // mbarrier per commit warp: phase (g / NCW) & 1 of hand[g % NCW]
                                     // completes when turn g has ended (its chain word is stored)
  volatile int q_seq[RING];       // g+1 once queue entry g is filled
  // chain word: (entries consumed by the commit warps) << 32 | (log entries written)
  volatile unsigned long long chain;
  volatile int exit_g;            // queue index of the EXIT entry (-1 while running)
  int ticket;                     // next queue entry for the spec warps
  volatile int lo_ring[4];        // lo_ring[b & 3] = log size at the start of block b
  volatile int bk_ring[8];        // bk_ring[b & 7] = first job of block b
  volatile int bk_known;          // blocks 0..bk_known have their first job recorded
  volatile int out_done, blk_c0, last_b;  // END bookkeeping shared by the commit warps
};

__device__ __forceinline__ int chain_gdone(unsigned long long w) { return (int)(w >> 32); }
__device__ __forceinline__ int chain_ncommit(unsigned long long w) { return (int)(unsigned)w; }
__device__ __forceinline__ unsigned long long chain_pack(int gdone, int ncommit) {
  return ((unsigned long long)(unsigned)gdone << 32) | (unsigned)ncommit;
}

template <bool CONSTR>
__device__ __forceinline__ VmState load_log(const ResolverShared& S, int idx, int& vm, int& k) {
  const LogEnt* e = &S.log[idx & (LOGN - 1)];
  const int4 h = *reinterpret_cast<const int4*>(e);
  const double2 a0 = *reinterpret_cast<const double2*>(&e->ac);
  const double2 a1 = *reinterpret_cast<const double2*>(&e->lc);
  const double2 a2 = *reinterpret_cast<const double2*>(&e->rc);
  const double2 a3 = *reinterpret_cast<const double2*>(&e->yc);
  VmState st;
  vm = h.x; st.an = h.y; st.pu = h.z; k = h.w;
  st.ac = a0.x; st.am = a0.y; st.lc = a1.x; st.lm = a1.y; st.rc = a2.x; st.rm = a2.y; st.yc = a3.x; st.ym = a3.y;
  st.room = 0x7fffffff; st.occ = 0; st.ptot = 0;
  if (CONSTR) {
    const int4 x = S.logx[idx & (LOGN - 1)];
    st.room = x.x; st.occ = x.y; st.ptot = x.z;
  }
  return st;
}
template <bool CONSTR>
__device__ __forceinline__ void store_log(ResolverShared& S, int idx, int vm, int k, const VmState& st) {
  LogEnt* e = &S.log[idx & (LOGN - 1)];
  *reinterpret_cast<int4*>(e) = make_int4(vm, st.an, st.pu, k);
  *reinterpret_cast<double2*>(&e->ac) = make_double2(st.ac, st.am);
  *reinterpret_cast<double2*>(&e->lc) = make_double2(st.lc, st.lm);
  *reinterpret_cast<double2*>(&e->rc) = make_double2(st.rc, st.rm);
  *reinterpret_cast<double2*>(&e->yc) = make_double2(st.yc, st.ym);
  if (CONSTR) S.logx[idx & (LOGN - 1)] = make_int4(st.room, st.occ, st.ptot, 0);
}

// A lane's working set during a spec: a sorted list of candidates plus two
// "sentinels" that bound everything the lane is responsible for but does not
// list: cb = the row's last entry (the rest of the lane's chunk is strictly
// worse), db = the best entry ever dropped from the list.
struct LaneList {
  double f[LK];
  int v[LK], e[LK];
  double cbf, dbf;
  int cbv, dbv;
  bool cb_real;  // the cb sentinel is itself a clean VM of the chunk with exactly that fitness
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < LK; i++) { f[i] = 0.0; v[i] = 0x7fffffff; e[i] = -1; }
    cbf = dbf = 0.0; cbv = dbv = 0x7fffffff; cb_real = false;
  }
  // x is better than every listed entry (row entries are pushed worst first)
  __device__ __forceinline__ void push_front(double x, int xv, int xe) {
#pragma unroll
    for (int i = LK - 1; i > 0; i--) { f[i] = f[i - 1]; v[i] = v[i - 1]; e[i] = e[i - 1]; }
    f[0] = x; v[0] = xv; e[0] = xe;
  }
  __device__ __forceinline__ void insert(double x, int xv, int xe) {
    if (!(x > 0.0)) return;
    if (!better(x, xv, f[LK - 1], v[LK - 1])) {  // not listed => dropped
      if (better(x, xv, dbf, dbv)) { dbf = x; dbv = xv; }
      return;
    }
    if (f[LK - 1] > 0.0 && better(f[LK - 1], v[LK - 1], dbf, dbv)) { dbf = f[LK - 1]; dbv = v[LK - 1]; }
    f[LK - 1] = x; v[LK - 1] = xv; e[LK - 1] = xe;
#pragma unroll
    for (int i = LK - 1; i > 0; i--) {
      if (better(f[i], v[i], f[i - 1], v[i - 1])) {
        double tf = f[i]; f[i] = f[i - 1]; f[i - 1] = tf;
        int tv = v[i]; v[i] = v[i - 1]; v[i - 1] = tv;
        int te = e[i]; e[i] = e[i - 1]; e[i - 1] = te;
      }
    }
  }
};


// Sum of the placed-member counts of the job's groups: changes iff a member of one of the job's
// groups is placed (counts only grow), so equal sums => the group state a result was computed
// against is still current.
__device__ __forceinline__ int group_version(const MatchArgs& a, int j) {
  int v = 0;
  for (int q = a.jb.group_off[j]; q < a.jb.group_off[j + 1]; q++) v += __ldcg(a.gr.gp_n + a.jb.group_idx[q]);
  return v;
}

// Candidate set of one job against the state at version s (warp-wide): up to
// `depth` VMs such that everything left out is no better than the bound z.
// Sentinel hits while fewer than `exact_n` candidates are out are resolved by an
// exact chunk re-scan; later ones truncate the set (complete = 0).
template <bool CONSTR>
__device__ __forceinline__ void spec_job(const MatchArgs& a, ResolverShared& S, const Latest latest, const QEntry& qe,
                                         const int s, const int depth, const int exact_n, SpecOut& out) {
  const int lane = threadIdx.x & 31;
  JobRegs r;
  r.c = qe.jc; r.m = qe.jm; r.g = qe.jg; r.ports = qe.jports; r.j = qe.jj;
  const int lo = qe.lo, blk = qe.blk;
  const bool wg = CONSTR && qe.grp;  // group constraints against the live group state
  const int gver = wg ? group_version(a, r.j) : 0;  // read BEFORE any group state is used
  const unsigned char* rowp = a.rows + ((size_t)(blk & 1) * a.bmax + qe.row) * ROW_BYTES;
  const unsigned* sbrow = CONSTR ? a.sbits + ((size_t)(blk & 1) * a.bmax + qe.row) * a.sb_words : nullptr;
  LaneList L;
  L.init();
  {
    const double* rf = reinterpret_cast<const double*>(rowp);
    const int32_t* rv = reinterpret_cast<const int32_t*>(rowp + ROW_V_OFF);
    double f[TOPK];
    int v[TOPK];
#pragma unroll
    for (int i = 0; i < TOPK; i++) { f[i] = __ldcg(rf + i * 32 + lane); v[i] = __ldcg(rv + i * 32 + lane); }
    if (f[TOPK - 1] > 0.0) { L.cbf = f[TOPK - 1]; L.cbv = v[TOPK - 1]; }  // full row: the rest of the chunk is worse
#pragma unroll
    for (int i = TOPK - 1; i >= 0; i--) {  // worst first: every push lands in front
      const bool live = f[i] > 0.0;
      const int vi = live ? v[i] : 0;
      if (live && latest.get(vi) < lo && (!wg || group_pass(a, r, vi))) {
        // a full list drops its worst entry; drops come in improving order, so the last one
        // dropped is the best clean VM of the chunk that is not listed: it becomes the bound
        if (L.f[LK - 1] > 0.0) { L.cbf = L.f[LK - 1]; L.cbv = L.v[LK - 1]; L.cb_real = true; }
        L.push_front(f[i], vi, -1);
      }
    }
  }
  // every VM committed since the snapshot, at its state as of version s
  for (int e = lo + lane; e < s; e += 32) {
    int vm, k;
    const VmState st = load_log<CONSTR>(S, e, vm, k);
    if (latest.get(vm) == e) L.insert(eval_res<CONSTR>(a, r, vm, st, wg, CONSTR ? sb_global(sbrow, vm) : true), vm, e);
  }
  // ---- selection.  A lane exposes its best entry not yet taken (its head) and keeps back
  // the next one and its sentinels.  Every head that beats everything any lane keeps back is
  // safe to take, all such heads at once; rounds repeat until at least `kmin` candidates
  // are out (the later rounds add few).  The set is unsorted; what is left defines z.
  int n = 0, complete = 0;
  unsigned taken = 0u;  // bit j: this lane's entry j went into the set
  auto store_cand = [&](int slot, double f, int vm, int e) {
    Cand& c = out.c[slot];
    c.f = f; c.vm = vm; c.e = e;
    if (e >= 0) { int vm2, k2; c.st = load_log<CONSTR>(S, e, vm2, k2); }
    else c.st = load_snap<CONSTR>(a, blk, vm);
  };
  const int kmin = depth == 1 ? 1 : min(a.spec_kmin, depth);
  while (n < kmin) {
    // head = first entry not taken, nx = the one after it
    double hf = 0.0, nf2 = 0.0;
    int hv = 0x7fffffff, he = -1, nv2 = 0x7fffffff, hj = LK;
#pragma unroll
    for (int j = LK - 1; j >= 0; j--)
      if (L.f[j] > 0.0 && !((taken >> j) & 1u)) { nf2 = hf; nv2 = hv; hf = L.f[j]; hv = L.v[j]; he = L.e[j]; hj = j; }
    double sf = L.cbf;
    int sv = L.cbv;
    bool s_cb = true;
    if (L.dbf > 0.0 && better(L.dbf, L.dbv, sf, sv)) { sf = L.dbf; sv = L.dbv; s_cb = false; }
    const bool head_sent = sf > 0.0 && better(sf, sv, hf, hv);  // head hidden behind a sentinel
    double rf = sf;  // what the lane keeps back when its head is taken
    int rv = sv;
    if (!head_sent && nf2 > 0.0 && better(nf2, nv2, rf, rv)) { rf = nf2; rv = nv2; }
    const double mf = warp_max_f64(rf);
    const int mv = (int)__reduce_min_sync(0xffffffffu, (rf == mf && mf > 0.0) ? (unsigned)rv : 0xffffffffu);
    const bool qual = !head_sent && hf > 0.0 && (!(mf > 0.0) || better(hf, hv, mf, mv));
    unsigned q = __ballot_sync(0xffffffffu, qual);
    if (q == 0u) {
      const unsigned anyh = __ballot_sync(0xffffffffu, hf > 0.0 || sf > 0.0);
      if (anyh == 0u) { complete = 1; break; }
      // a sentinel dominates every head: the lane that holds it
      const int wl = __ffs(__ballot_sync(0xffffffffu, rf == mf && rv == mv)) - 1;
      const bool wcb = __shfl_sync(0xffffffffu, (s_cb && rf == sf && rv == sv) ? 1 : 0, wl) != 0;
      if (!wcb || n >= exact_n) { if (lane == 0) atomicAdd(a.stats + 5, 1ull); break; }
      // exact re-scan of chunk wl: clean VMs strictly worse than its bound
      const double bf = __shfl_sync(0xffffffffu, L.cbf, wl);
      const int bv = __shfl_sync(0xffffffffu, L.cbv, wl);
      if (lane == wl) {
        if (L.cb_real) L.insert(L.cbf, L.cbv, -1);  // the bound itself is a clean candidate
        L.cbf = 0.0; L.cbv = 0x7fffffff; L.cb_real = false;
      }
      // NB: inserts shift list positions; nothing of lane wl has been taken yet in that case
      // only if its head was hidden from the start, which is when a chunk bound can dominate
      for (int v = wl + 32 * lane; v < a.of.O; v += 32 * 32) {  // chunk wl = VMs v with v mod 32 == wl
        if (latest.get(v) >= lo) continue;
        if (CONSTR && !sb_global(sbrow, v)) continue;
        const VmState st = load_snap<CONSTR>(a, blk, v);
        const double x = eval_res<CONSTR>(a, r, v, st, wg, true);
        if (x > 0.0 && better(bf, bv, x, v)) L.insert(x, v, -1);
      }
      if (lane == 0) atomicAdd(a.stats + 1, 1ull);
      continue;
    }
    int cnt = __popc(q);
    if (cnt > depth - n) {
      // more heads qualify than fit: take the single best of them (keeps depth == 1 exact)
      unsigned wk;
      int wl;
      warp_argmax(qual ? hf : 0.0, (unsigned)hv, wk, wl);
      q = 1u << wl;
      cnt = 1;
    }
    if ((q >> lane) & 1u) {
      store_cand(n + __popc(q & ((1u << lane) - 1u)), hf, hv, he);
      taken |= 1u << hj;
    }
    n += cnt;
  }
  // bound: the best entry not taken or sentinel of any lane
  double zf;
  int zv, z_real = 0;
  {
    double ef = 0.0;
    int ev = 0x7fffffff, ee = -1;
    bool head = false;  // the exposure is a real entry (not a sentinel)
#pragma unroll
    for (int j = LK - 1; j >= 0; j--)
      if (L.f[j] > 0.0 && !((taken >> j) & 1u)) { ef = L.f[j]; ev = L.v[j]; ee = L.e[j]; head = true; }
    if (L.cbf > 0.0 && better(L.cbf, L.cbv, ef, ev)) { ef = L.cbf; ev = L.cbv; head = false; }
    if (L.dbf > 0.0 && better(L.dbf, L.dbv, ef, ev)) { ef = L.dbf; ev = L.dbv; head = false; }
    zf = warp_max_f64(ef);
    zv = (int)__reduce_min_sync(0xffffffffu, (ef == zf && zf > 0.0) ? (unsigned)ev : 0xffffffffu);
    if (!(zf > 0.0)) complete = 1;
    else {
      // when the bound is a real entry it is the best VM outside the set: the commit warp
      // may take it directly if everything it knows is worse (instead of recomputing)
      const unsigned hm = __ballot_sync(0xffffffffu, ef == zf && ev == zv);
      const unsigned rm = __ballot_sync(0xffffffffu, ef == zf && ev == zv && head);
      if (hm == rm && hm != 0u) {  // no sentinel ties with it
        z_real = 1;
        if (lane == __ffs(rm) - 1) store_cand(KC, zf, zv, ee);
      }
    }
  }
  if (lane == 0) { out.type = Q_JOB; out.s = s; out.n = n; out.complete = complete; out.zf = zf; out.zv = zv; out.z_real = z_real; out.gver = gver; }
  __syncwarp();
}

// the commit warps' rare exact recomputation, kept out of their hot loop
template <bool CONSTR>
__device__ __noinline__ void spec_job_fallback(const MatchArgs& a, ResolverShared& S, const Latest latest,
                                               const QEntry& qe, const int s) {
  spec_job<CONSTR>(a, S, latest, qe, s, 1, 1, S.res[RING]);
}

// Exact placement of a group-constrained job against the live state (commit warp).
// Returns the winning VM (or -1); the winner's pre-placement state lands in `w`.
template <bool CONSTR>
__device__ __noinline__ int resolve_group_job(const MatchArgs& a, ResolverShared& S, const Latest latest,
                                              const QEntry& qe, VmState& w) {
  const int lane = threadIdx.x & 31;
  JobRegs r;
  r.c = qe.jc; r.m = qe.jm; r.g = qe.jg; r.ports = qe.jports; r.j = qe.jj;
  const unsigned* sbrow = CONSTR ? a.sbits + ((size_t)(qe.blk & 1) * a.bmax + qe.row) * a.sb_words : nullptr;
  double cf = 0.0;
  int cv = 0x7fffffff;
  for (int v = lane; v < a.of.O; v += 32) {
    const int e = latest.get(v);
    VmState st;
    if (e >= qe.lo) { int vm, k; st = load_log<CONSTR>(S, e, vm, k); }
    else st = load_snap<CONSTR>(a, qe.blk, v);
    const double f = eval_res<CONSTR>(a, r, v, st, true, CONSTR ? sb_global(sbrow, v) : true);
    if (f > cf) { cf = f; cv = v; }  // v ascends per lane: strict > keeps the lowest
  }
  unsigned wk;
  int wl;
  const double wf = warp_argmax(cf, (unsigned)cv, wk, wl);
  if (!(wf > 0.0)) return -1;
  const int wv = (int)wk;
  const int we = latest.get(wv);
  if (we >= qe.lo) { int vm, k; w = load_log<CONSTR>(S, we, vm, k); }
  else w = load_snap<CONSTR>(a, qe.blk, wv);
  return wv;
}

// ---- driver warp: feasibility stamps -> in-order queue
// The resolver CTA runs the driver; every spec CTA runs a replica (REMOTE) that derives the same
// queue from the same global inputs (stamps, block bounds, lo_g) and fills only its local ring.
template <bool CONSTR, bool REMOTE, bool PROF = false>
__device__ void driver_warp(const MatchArgs& a, ResolverShared& S) {
  const int lane = threadIdx.x & 31;
  int g = 0;
  unsigned long long skipped = 0;
  auto wait_slot = [&](int gi) {  // entry gi may be filled once entry gi - lookahead is consumed
    while (chain_gdone(S.chain) <= gi - a.lookahead) __nanosleep(a.poll_ns);
  };
  for (int b = 0;; b++) {
    int k0, k1;
    if (!REMOTE) {
      while (S.bk_known < b + 1) __nanosleep(20);  // block b's bounds are set two block ends ahead
      k0 = S.bk_ring[b & 7];
      k1 = S.bk_ring[(b + 1) & 7];
    } else {
      if (b >= 2) {  // bk0[b], bk0[b+1] and lo_g[b-1] are written before `published` reaches b - 1
        if (lane == 0) {
          while ((int)ld_relaxed_u32(a.published) < b - 1) __nanosleep(64);
          __threadfence();
        }
        __syncwarp();
      }
      k0 = __ldcg(a.bk0 + b);
      k1 = __ldcg(a.bk0 + b + 1);
    }
    if (k0 >= a.n_cons) break;
    const int nj = min(k1, a.n_cons) - k0;
    // the evaluators stop as soon as no VM can take even the smallest request left (exact: the
    // assigned amounts only grow): everything from this block on is unplaceable
    int dead = 0;
    if (lane == 0) {
      while (ld_acquire_u32(a.rows_ready + b) < (unsigned)nj) {
        const int db = (int)ld_relaxed_u32(reinterpret_cast<const unsigned*>(a.dead_blk));
        if (db != 0 && db - 1 <= b) { dead = 1; break; }
        __nanosleep(20);
      }
    }
    if (PROF && lane == 0 && b < g_blk_cap) g_blk_trace[b] = (unsigned long long)clock64();
    dead = __shfl_sync(0xffffffffu, dead, 0);
    if (dead) {
      if (!REMOTE && lane == 0) {
        skipped += (unsigned long long)(a.n_cons - k0);
        *a.dead_k0 = k0;
      }
      break;
    }
    // rows b ready => END(b-2) was processed => the start of block b-1 is recorded
    const int lo = b == 0 ? 0 : (REMOTE ? __ldcg(a.lo_g + b - 1) : S.lo_ring[(b - 1) & 3]);
    const int32_t* feas = a.feas + (size_t)(b & 1) * a.bmax;
    // all stamps of the block in one L2 round trip (a block has at most MAXB rows)
    int stamp[MAXB / 32];
#pragma unroll
    for (int t = 0; t < MAXB / 32; t++) stamp[t] = (t * 32 + lane) < nj ? __ldcg(feas + t * 32 + lane) : 0;
#pragma unroll
    for (int t = 0; t < MAXB / 32; t++) {
      const int base = t * 32;
      if (base >= nj) break;
      const int i = base + lane;
      const bool valid = i < nj;
      const bool fz = valid && stamp[t] == b + 1;
      // jobs with no feasible VM at the snapshot are unplaceable now too (resources
      // and count constraints only tighten within a cycle): skip them wholesale.
      if (!REMOTE && valid && !fz) { a.assign[k0 + i] = -1; a.fail[k0 + i] = COOK_FAIL_RESOURCES; }
      const unsigned mask = __ballot_sync(0xffffffffu, fz);
      skipped += __popc(__ballot_sync(0xffffffffu, valid && !fz));
      if (fz) {
        const int gi = g + __popc(mask & ((1u << lane) - 1u));
        const int k = k0 + i;
        QEntry q;
        q.type = Q_JOB; q.blk = b; q.k = k; q.lo = lo;
        q.jc = a.kc[k]; q.jm = a.km[k]; q.jj = a.cons[k];
        q.jg = CONSTR ? a.kg[k] : 0.0;
        q.jports = CONSTR ? a.kports[k] : 0;
        q.grp = CONSTR ? (a.kflags[k] & 1) : 0;
        q.row = i;
        wait_slot(gi);
        S.q[gi & (RING - 1)] = q;
        fence_cta();
        S.q_seq[gi & (RING - 1)] = gi + 1;
      }
      g += __popc(mask);
      __syncwarp();
    }
    if (lane == 0) {
      wait_slot(g);
      QEntry& q = S.q[g & (RING - 1)];
      q.type = Q_END; q.blk = b; q.k = -1; q.lo = lo; q.grp = 0;
      if (!REMOTE) S.res[g & (RING - 1)].type = Q_END;
      fence_cta();
      S.q_seq[g & (RING - 1)] = g + 1;
      if (!REMOTE) mbar_arrive(&S.res_bar[g & (RING - 1)]);
    }
    g++;
    __syncwarp();
  }
  if (lane == 0) {
    wait_slot(g);
    S.q[g & (RING - 1)].type = Q_EXIT;
    if (!REMOTE) S.res[g & (RING - 1)].type = Q_EXIT;
    fence_cta();
    S.q_seq[g & (RING - 1)] = g + 1;
    if (!REMOTE) mbar_arrive(&S.res_bar[g & (RING - 1)]);
    S.exit_g = g;
    if (!REMOTE) a.stats[6] = skipped;
  }
}

// ---- spec warps (spec CTA ci of n_spec): entries g = ci, ci + n_spec, ... of the queue.  The
// candidate set goes to global memory; the resolver's fetcher warp pulls it into its result ring.
template <bool CONSTR>
__device__ void spec_warp(const MatchArgs& a, ResolverShared& S, const Latest latest, const int ci) {
  const int lane = threadIdx.x & 31;
  while (true) {
    int t = 0;
    if (lane == 0) t = atomicAdd(&S.ticket, 1);
    t = __shfl_sync(0xffffffffu, t, 0);
    const int g = t * a.n_spec + ci;
    const int slot = g & (RING - 1);
    bool quit = false;
    while (S.q_seq[slot] != g + 1) {
      const int xg = S.exit_g;
      if (xg >= 0 && g > xg) { quit = true; break; }
      __nanosleep(a.poll_ns);
    }
    if (quit) return;
    compiler_barrier();
    const QEntry qe = S.q[slot];
    if (qe.type == Q_EXIT) return;
    if (qe.type != Q_JOB) continue;
    const int s = chain_ncommit(S.chain);
    compiler_barrier();
    spec_job<CONSTR>(a, S, latest, qe, s, KC, 2, a.gres[g & (GRING - 1)]);
    __threadfence();  // every lane's part of the result is out before the flag
    __syncwarp();
    if (lane == 0) st_release_u32(a.gres_seq + (g & (GRING - 1)), (unsigned)(g + 1));
  }
}

// ---- publisher warp (resolver CTA): copies new log entries to global memory and then publishes
// the chain word they belong to; off the chain, batches whatever accumulated since its last pass.
template <bool CONSTR>
__device__ void publisher_warp(const MatchArgs& a, ResolverShared& S) {
  const int lane = threadIdx.x & 31;
  int p = 0;
  unsigned long long last = 0ull;
  while (true) {
    const unsigned long long w = S.chain;
    compiler_barrier();
    if (w != last) {
      const int c = chain_ncommit(w);
      for (int base = p; base < c; base += 6) {  // 6 entries x 5 granules of 16 B per pass
        const int e = base + lane / 5, ch = lane % 5;
        if (lane < 30 && e < c) {
          const int4 v = reinterpret_cast<const int4*>(&S.log[e & (LOGN - 1)])[ch];
          __stcg(reinterpret_cast<int4*>(a.glog + (e & (LOGN - 1))) + ch, v);
        }
      }
      if (CONSTR)
        for (int e = p + lane; e < c; e += 32) __stcg(a.glogx + (e & (LOGN - 1)), S.logx[e & (LOGN - 1)]);
      __threadfence();
      __syncwarp();
      if (lane == 0) st_release_u64(a.gchain, w);
      p = c;
      last = w;
    } else {
      __nanosleep(40);
    }
    const int xg = S.exit_g;
    if (xg >= 0 && chain_gdone(last) >= xg) return;
  }
}

// ---- follower warp (spec CTA): keeps the CTA's replica of the log, latest[] and the chain word
// up to date.  The replica may lag: a candidate set computed against version s is valid for any
// s (the owner folds every entry >= s), lag only shifts work to the owner's first look.
template <bool CONSTR>
__device__ void follower_warp(const MatchArgs& a, ResolverShared& S, const Latest latest) {
  const int lane = threadIdx.x & 31;
  int p = 0;
  unsigned long long last = 0ull;
  while (true) {
    unsigned long long w = 0ull;
    if (lane == 0) w = ld_relaxed_u64(a.gchain);
    w = __shfl_sync(0xffffffffu, w, 0);
    if (w != last) {
      __threadfence();  // acquire: the entries below the published log size are visible
      const int c = chain_ncommit(w);
      for (int base = p; base < c; base += 6) {
        const int e = base + lane / 5, ch = lane % 5;
        if (lane < 30 && e < c) {
          const int4 v = __ldcg(reinterpret_cast<const int4*>(a.glog + (e & (LOGN - 1))) + ch);
          reinterpret_cast<int4*>(&S.log[e & (LOGN - 1)])[ch] = v;
        }
      }
      if (CONSTR)
        for (int e = p + lane; e < c; e += 32) S.logx[e & (LOGN - 1)] = __ldcg(a.glogx + (e & (LOGN - 1)));
      __syncwarp();
      if (lane == 0) {
        for (int e = p; e < c; e++) latest.set(S.log[e & (LOGN - 1)].vm, e);  // in order: the newest entry wins
        fence_cta();
        S.chain = w;
      }
      __syncwarp();
      p = c;
      last = w;
    } else {
      __nanosleep(40);
    }
    const int xg = S.exit_g;
    if (xg >= 0 && chain_gdone(last) >= xg) return;
  }
}

// ---- fetcher warp (resolver CTA): lane l owns result slot l.  Once the queue entry of its next
// g is known to be a job it polls the spec CTAs' flag for g and then moves the candidate set
// global -> shared with ONE bulk async copy that completes on the slot's mbarrier: the commit
// warps sleep on that barrier instead of polling.
__device__ void fetcher_warp(const MatchArgs& a, ResolverShared& S) {
  const int lane = threadIdx.x & 31;
  int g = lane;
  bool have_q = false, done = false;
  while (true) {
    if (!done && !have_q) {
      if (S.q_seq[lane] == g + 1) {
        compiler_barrier();
        const int type = S.q[lane].type;
        if (type == Q_JOB) have_q = true;
        else if (type == Q_EXIT) done = true;
        else g += RING;
      } else {
        const int xg = S.exit_g;
        if (xg >= 0 && g > xg) done = true;
      }
    }
    bool issued = false;
    if (!done && have_q) {
      const int gi = g & (GRING - 1);
      if (ld_relaxed_u32(a.gres_seq + gi) == (unsigned)(g + 1)) {
        __threadfence();             // acquire the spec warp's stores ...
        fence_proxy_async_global();  // ... and order them before the async proxy's read
        mbar_arrive_expect_tx(&S.res_bar[lane], (unsigned)sizeof(SpecOut));
        bulk_g2s(&S.res[lane], a.gres + gi, (unsigned)sizeof(SpecOut), &S.res_bar[lane]);
        have_q = false;
        g += RING;
        issued = true;
      }
    }
    if (__all_sync(0xffffffffu, done)) return;
    if (!__any_sync(0xffffffffu, issued)) __nanosleep(a.poll_ns);
  }
}

// ---- commit warps
// argmax over lanes of (f desc, v asc) with an early exit when the high words
// of the fitness already single out one lane (the common case).
__device__ __forceinline__ double warp_argmax_fast(double f, int v, int& wv, int& wl) {
  const unsigned hi = (unsigned)__double2hiint(f);
  const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
  unsigned cand = __ballot_sync(0xffffffffu, hi == mh);
  if (mh == 0u) { wv = 0x7fffffff; wl = 0; return 0.0; }  // f in (0, 1] has a non-zero high word
  if (__popc(cand) > 1) {
    const unsigned lo = hi == mh ? (unsigned)__double2loint(f) : 0u;
    const unsigned ml = __reduce_max_sync(0xffffffffu, lo);
    cand = __ballot_sync(0xffffffffu, hi == mh && lo == ml);
    if (__popc(cand) > 1) {
      const unsigned key = ((cand >> (threadIdx.x & 31)) & 1u) ? (unsigned)v : 0xffffffffu;
      const unsigned mk = __reduce_min_sync(0xffffffffu, key);
      cand = __ballot_sync(0xffffffffu, key == mk);
    }
  }
  wl = __ffs(cand) - 1;
  wv = __shfl_sync(0xffffffffu, v, wl);
  return __shfl_sync(0xffffffffu, f, wl);
}

// The hand-off of the commit turn (plain pools): the owner of turn t stores its chain word and then
// arrives (release) on hand[t % NCW], completing phase t / NCW of that barrier; wait_turn(S, t) returns
// (acquire) once it has, so every store of turn t is visible.  The owner of turn g waits only for a turn
// t in [g - NCW + 1, g - 1] (its own turn g - NCW has ended), so the parity cannot alias: the barrier's
// next phase completes at the end of turn t + NCW > g, owned by the same warp as turn t, which cannot
// end before turn g does.  For the same reason a wait may be repeated.
template <int NCW>
__device__ __forceinline__ void wait_turn(ResolverShared& S, const int t) {
  asm volatile(
      "{\n\t.reg .pred p;\n"
      "WAIT_TURN:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WAIT_TURN;\n\t}"
      :: "r"(smem_u32(&S.hand[t % NCW])), "r"((unsigned)(t / NCW) & 1u) : "memory");
}

template <bool CONSTR, bool PROF>
__device__ void commit_warp(const MatchArgs& a, ResolverShared& S, const Latest latest, const int cw,
                            unsigned* sbw) {  // sbw: this warp's copy of the current job's verdict bits
  constexpr int NCW = CONSTR ? NCW_CONSTR : NCW_PLAIN;
  const int lane = threadIdx.x & 31;
  unsigned long long n_fast = 0, n_group = 0, n_matched = 0, n_fallback = 0, n_slow_turn = 0, n_ztake = 0, n_relook = 0;
  unsigned long long prof[6] = {0, 0, 0, 0, 0, 0};
  const long long t_start = clock64();
  for (int g = cw;; g += NCW) {
    const int slot = g & (RING - 1);
    long long t0 = PROF ? clock64() : 0;
    bool quit = false;
    // the result of entry g lands in res[slot] by bulk copy (or the driver marks END / EXIT) and
    // completes phase (g / RING) & 1 of the slot's mbarrier: the warp sleeps in hardware
    while (!mbar_try_wait(&S.res_bar[slot], (unsigned)(g >> 5) & 1u, 2000u)) {
      const int xg = S.exit_g;
      if (xg >= 0 && g > xg) { quit = true; break; }
    }
    if (quit) break;
    const SpecOut* R = &S.res[slot];
    const int type = R->type;
    const long long t_land = PROF ? clock64() : 0;
    if (PROF) prof[0] += (unsigned long long)(t_land - t0);
    // lane 0: this turn's row of the timeline
    // (t_done is read right after the chain store: the row's other stamps may come back from local memory)
    auto trace_turn = [&](long long t_ready, long long t_seen, long long t_eval, long long t_dec, long long t_fence,
                          long long t_done, unsigned long long info, int key, unsigned long long hand,
                          unsigned long long poll) {
      if (PROF && lane == 0 && g < g_turn_cap) {
        unsigned long long* p = g_turn_trace + (size_t)g * TURN_WORDS;
        p[TT_FREE] = (unsigned long long)t0; p[TT_LAND] = (unsigned long long)t_land;
        p[TT_READY] = (unsigned long long)t_ready; p[TT_SEEN] = (unsigned long long)t_seen;
        p[TT_DONE] = (unsigned long long)t_done; p[TT_FENCE] = (unsigned long long)t_fence;
        p[TT_INFO] = info; p[TT_K] = (unsigned long long)(long long)key;
        p[TT_EVAL] = (unsigned long long)t_eval; p[TT_DEC] = (unsigned long long)t_dec;
        p[TT_HAND] = hand; p[TT_POLL] = poll;
      }
    };
    if (type == Q_EXIT) {
      while (chain_gdone(S.chain) != g) __nanosleep(20);
      if (lane == 0) a.stats[14] = (unsigned long long)(clock64() - t_start);
      break;
    }
    if (type == Q_END) {
      unsigned long long w;
      while (chain_gdone(w = S.chain) != g) __nanosleep(20);
      compiler_barrier();
      long long t4 = PROF ? clock64() : 0;
      // publish the newest state of every VM touched in this or the previous block
      // into the buffer the evaluators read for block blk+2; write the block's results
      const int b = S.q[slot].blk, lo = S.q[slot].lo;
      const int c = chain_ncommit(w), out_done = S.out_done;
      VmDyn* pub = a.dyn.d[b & 1];
      for (int e = lo + lane; e < c; e += 32) {
        int vm, k;
        const VmState st = load_log<CONSTR>(S, e, vm, k);
        if (latest.get(vm) == e) {
          __stcg(reinterpret_cast<double2*>(pub + vm), make_double2(st.ac, st.am));
          if (CONSTR) __stcg(reinterpret_cast<int2*>(a.dyn.n[b & 1] + vm), make_int2(st.an, st.pu));
        }
        if (e >= out_done) {  // results of this block's placements
          a.assign[k] = vm;
          a.fail[k] = COOK_FAIL_NONE;
          a.ports_start[k] = CONSTR ? st.pu - a.kports[k] : 0;
        }
      }
      __syncwarp();
      if (lane == 0) {
        S.out_done = c;
        S.lo_ring[(b + 1) & 3] = c;
        // size of block b+2 from this block's placement rate: about btarget placements per
        // block keeps the log ranges short while the cluster fills and the blocks long after
        const int nb = S.bk_ring[(b + 1) & 7] - S.bk_ring[b & 7];
        const int placed = c - S.blk_c0;
        long long want = placed > 0 ? ((long long)a.btarget * nb + placed - 1) / placed : a.bmax;
        want = min(want, (long long)min(a.bmax, 2 * S.last_b));
        const int nbn = max((int)want, a.bmin);
        S.last_b = nbn;
        S.blk_c0 = c;
        const int end2 = S.bk_ring[(b + 2) & 7] + nbn;   // = first job of block b+3
        S.bk_ring[(b + 3) & 7] = end2;
        __stcg(a.bk0 + b + 3, end2);
        __stcg(a.lo_g + b + 1, c);   // the spec CTAs' driver replicas read the block's lo from here
        fence_cta();
        S.bk_known = b + 3;
        const long long t_fence = PROF ? clock64() : 0;
        __threadfence();
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.published), "r"((unsigned)(b + 1)) : "memory");
        S.chain = chain_pack(g + 1, c);
        const long long t_done = PROF ? clock64() : 0;   // the arrive belongs to the hand-off
        if (!CONSTR) mbar_arrive(&S.hand[g % NCW]);
        if (PROF) {
          trace_turn(t_land, t4, 0, 0, t_fence, t_done, 1ull | ((unsigned long long)b << 32), c - lo, 0, 0);
        }
        if (PROF && S.bk_ring[b & 7] < a.n_cons / 4) a.stats[15] = (unsigned long long)(clock64() - t_start);  // timeline: end of the first quarter
      }
      __syncwarp();
      if (PROF) prof[4] += (unsigned long long)(clock64() - t4);
      continue;
    }
    const QEntry& qe = S.q[slot];
    JobRegs r;
    r.c = qe.jc; r.m = qe.jm; r.g = CONSTR ? qe.jg : 0.0; r.ports = CONSTR ? qe.jports : 0; r.j = qe.jj;
    const int k = qe.k;
    const bool grp = CONSTR && qe.grp;
    if (CONSTR) {  // the job's verdict bits: global -> shared, before anything is evaluated
      const unsigned* sbrow = a.sbits + ((size_t)(qe.blk & 1) * a.bmax + qe.row) * a.sb_words;
      for (int wd = lane; wd < a.sb_words; wd += 32) sbw[wd] = __ldcg(sbrow + wd);
      __syncwarp();
    }
    auto join_groups = [&](int wv) {  // lane 0: record the placement in the job's groups
      for (int q = a.jb.group_off[r.j]; q < a.jb.group_off[r.j + 1]; q++) {
        const int gi = a.jb.group_idx[q];
        const int n = __ldcg(a.gr.gp_n + gi);
        __stcg(a.gr.gp_vm + a.gr.gp_off[gi] + n, wv);
        __threadfence();  // the member is visible before the count that covers it
        __stcg(a.gr.gp_n + gi, n + 1);
      }
      __threadfence();
    };
    // ---- plain job
    const int s = R->s, n = R->n;
    const bool r_complete = R->complete != 0;
    const double r_zf = R->zf;
    const int r_zv = R->zv;
    const int el = s + lane;
    const double yf = lane < n ? R->c[lane & (KC - 1)].f : 0.0;   // this lane's listed candidate
    const int yv = lane < n ? R->c[lane & (KC - 1)].vm : 0x7fffffff;
    static_assert(KC <= 32 && (KC & (KC - 1)) == 0, "one candidate per lane");
    // Uniform (same in every lane) exact top-`d` of the valid items known so far: log
    // entries [s, c_seen) still newest for their VM + listed candidates unchanged since s.
    // src >= 0: log entry index, src < 0: ~candidate index.  `more`: valid items exist
    // outside the list.
    // depth 3: with NCW owners up to NCW - 1 entries appear between the first look and the turn; a
    // deeper list costs more on every job than the rare exact recomputation it avoids (measured)
    constexpr int TD = 3;
    double tf[TD];
    int tv[TD], ts[TD], d = 0;
#pragma unroll
    for (int i = 0; i < TD; i++) { tf[i] = 0.0; tv[i] = 0x7fffffff; ts[i] = 0; }
    bool more = false, have = false;
    int c_seen = s;
    long long t1 = PROF ? clock64() : 0;
    long long t_ready = 0, t_seen = 0;               // PROF: end of the (first) first look, turn observed
    unsigned n_fold = 0, n_rel = 0, slow = 0;        // PROF: entries folded one by one, relooks, slow turn
    // PROF: t_hand = the low word of the clock when the owner learned that turn g-1 had ended;
    // hp = HP_FOLDED (the last step was a fold) | HP_MID (it learned that right after a fold) | HP_HAND
    // (t_hand taken) + HP_WAIT per wait for a turn to end; two registers, as the PROF instantiation spills
    enum : unsigned { HP_FOLDED = 1u, HP_MID = 2u, HP_HAND = 4u, HP_WAIT = 8u };
    unsigned t_hand = 0, hp = 0;
    auto mark_hand = [&](bool mid) { t_hand = (unsigned)clock64(); hp |= HP_HAND | (mid ? HP_MID : 0u); };
    unsigned long long w;
    int c = 0;
  relook:
    while (true) {
      w = S.chain;
      compiler_barrier();
      const int gd = chain_gdone(w);
      const int c_now = chain_ncommit(w);
      const bool mine = gd == g;
      // under a predicate computed from the chain word: the stamp waits for its load
      if (PROF && mine && !(hp & HP_HAND)) mark_hand(have && ((hp & HP_FOLDED) || c_now > c_seen + 1));
      if (!have) {
        // (a) first look: one lane per log entry committed since s, TD argmax rounds
        double xf = 0.0;
        int x_vm = 0x7fffffff;
        if (el < c_now) {
          int kk;
          const VmState x = load_log<CONSTR>(S, el, x_vm, kk);
          xf = eval_res<CONSTR>(a, r, x_vm, x, grp, CONSTR ? sb_shared(sbw, x_vm) : true);
        }
        c_seen = c_now;
        bool xin = el < c_seen && xf > 0.0 && latest.get(x_vm) == el;
        bool ok = lane < n && latest.get(yv) < s;
        const int nvalid = __popc(__ballot_sync(0xffffffffu, xin)) + __popc(__ballot_sync(0xffffffffu, ok));
        more = nvalid > TD;
        d = min(nvalid, TD);
#pragma unroll
        for (int rnd = 0; rnd < TD; rnd++) {
          const bool use_y = ok && (!xin || better(yf, yv, xf, x_vm));
          const double lf = use_y ? yf : (xin ? xf : 0.0);
          const int lv = use_y ? yv : (xin ? x_vm : 0x7fffffff);
          int bv, bl;
          const double bf = warp_argmax_fast(lf, lv, bv, bl);
          const bool by = __shfl_sync(0xffffffffu, use_y ? 1 : 0, bl) != 0;
          tf[rnd] = bf; tv[rnd] = bv; ts[rnd] = by ? ~bl : s + bl;
          if (lane == bl) { if (use_y) ok = false; else xin = false; }
        }
        have = true;
        if (mine) n_slow_turn++;
        if (PROF && t_ready == 0) { t_ready = clock64(); slow = mine ? 1u : 0u; }
        continue;
      }
      if (mine && c_now <= c_seen + 1) { c = c_now; break; }
      if (c_now > c_seen) {
        // (b) one more entry, not the last before the turn: every lane evaluates it (uniform)
        // and the list is updated without a warp collective
        if (PROF) { n_fold++; hp |= HP_FOLDED; }
        int nvm, kk;
        const VmState ne = load_log<CONSTR>(S, c_seen, nvm, kk);
        const double nf = eval_res<CONSTR>(a, r, nvm, ne, grp, CONSTR ? sb_shared(sbw, nvm) : true);
        const int nsrc = c_seen;
        c_seen++;
        // the entry supersedes whatever was known about its VM
        bool hit = false;
#pragma unroll
        for (int i = 0; i < TD; i++) {
          hit = hit || (i < d && tv[i] == nvm);
          if (hit && i + 1 < TD) { tf[i] = tf[i + 1]; tv[i] = tv[i + 1]; ts[i] = ts[i + 1]; }
        }
        if (hit) d--;
        if (nf > 0.0) {
          // position: before the first listed item it beats; behind all of them only if
          // nothing is hidden (then it is the next best)
          int pos = TD;
#pragma unroll
          for (int i = TD - 1; i >= 0; i--)
            if (i < d && better(nf, nvm, tf[i], tv[i])) pos = i;
          if (pos == TD && !more && d < TD) pos = d;
          if (pos < TD) {
            if (d == TD) more = true; else d++;   // the last listed item falls out of a full list
#pragma unroll
            for (int i = TD - 1; i > 0; i--)
              if (i > pos) { tf[i] = tf[i - 1]; tv[i] = tv[i - 1]; ts[i] = ts[i - 1]; }
#pragma unroll
            for (int i = 0; i < TD; i++)
              if (i == pos) { tf[i] = nf; tv[i] = nvm; ts[i] = nsrc; }
          } else {
            more = true;
          }
        }
        continue;
      }
      // every entry below c_now is folded: sleep until turn gd ends, then fold its entry, if any
      if (PROF) hp = (hp & ~HP_FOLDED) + HP_WAIT;
      if (CONSTR) {   // constraint pools poll for it: the barrier made config #3's step 0.6 % slower
        if (gd < g - 1) __nanosleep(40);  // only the next in line polls hard
        continue;
      }
      wait_turn<NCW>(S, gd);
      if (gd < g - 1) continue;
      // turn g-1 has ended and appended at most entry c_seen; the chain word's load is still in
      // flight when the turn below issues the loads of that entry
      if (PROF) mark_hand(false);
      c = *reinterpret_cast<volatile int*>(&S.chain);   // the low word: log entries written
      break;
    }
    long long t2 = PROF ? clock64() : 0;
    if (PROF) prof[1] += (unsigned long long)(t2 - t1);
    if (PROF && t_seen == 0) t_seen = t2;   // a relook after this point belongs to the turn
    // ---- the turn: c == c_seen (nothing new) or c == c_seen + 1 (one new entry)
    // log[c_seen] is loaded before c is tested, so its loads issue together with the chain word's:
    // the entry's stores precede turn g-1's chain store (and, in plain pools, its arrive), so the entry
    // is the committed one whenever the word covers it, and is not used otherwise
    int ne_vm, kk;
    VmState ne = load_log<CONSTR>(S, c_seen, ne_vm, kk);
    double nf = 0.0;
    if (c > c_seen) {  // uniform: every lane evaluates the newest entry
      nf = eval_res<CONSTR>(a, r, ne_vm, ne, grp, CONSTR ? sb_shared(sbw, ne_vm) : true);
    } else {
      ne_vm = -1;
    }
    // best old item that the newest entry did not supersede
    const bool first = !(d > 0 && tv[0] == ne_vm);
    const bool known = first ? (d > 0 || !more) : (d > 1 || !more);  // that rank is known (possibly "none")
    if (!known) {
      // the short list ran dry (its items were superseded one after the other): look at all
      // lanes' items again at the current version; the list is exact again afterwards
      have = false;
      n_relook++;
      if (PROF) n_rel++;
      goto relook;
    }
    const double pf = first ? (d > 0 ? tf[0] : 0.0) : (d > 1 ? tf[1] : 0.0);
    const int pv = first ? (d > 0 ? tv[0] : 0x7fffffff) : (d > 1 ? tv[1] : 0x7fffffff);
    const int ps = first ? ts[0] : ts[1];
    const bool take_new = nf > 0.0 && better(nf, ne_vm, pf, pv);
    const double wf = take_new ? nf : pf;
    const int wv0 = take_new ? ne_vm : pv;
    // every unchanged VM outside the candidate set is no better than the bound z: the
    // winner is exact when its rank is known and the set is complete or it beats z
    const bool exact = known && (r_complete || (wf > 0.0 && better(wf, wv0, r_zf, r_zv)));
    // everything known is worse than the bound, the bound is a real VM and nothing touched it
    // since s: it is the best VM outside the set, hence the winner
    const bool take_z = !exact && known && R->z_real != 0 && ne_vm != r_zv && latest.get(r_zv) < s;
    // PROF: stamps taken under a predicate computed from the value, so they wait for it
    long long t_eval = 0, t_dec = 0;
    if (PROF && __double_as_longlong(nf) != 0x7ff8deadbeef0000ll) t_eval = clock64();
    if (PROF && (__double_as_longlong(wf) != 0x7ff8deadbeef0000ll || take_z)) t_dec = clock64();
    int wv = -1;
    auto append = [&](int vm, VmState st) {  // lane 0: the placement becomes log entry c
      st.ac = st.ac + r.c; st.am = st.am + r.m; st.an += 1; st.pu += r.ports;
      store_log<CONSTR>(S, c, vm, k, st);
      latest.set(vm, c);
      if (grp) join_groups(vm);
      fence_cta();
      S.chain = chain_pack(g + 1, c + 1);
    };
    bool wv_group = false;  // PROF: the group path was taken
    if (grp && group_version(a, r.j) != R->gver) {
      // a member of one of the job's groups was placed since the result was computed: the group
      // constraints it was filtered with are stale => exact full scan against the live state
      if (PROF) wv_group = true;
      const QEntry q2 = qe;
      VmState ws;
      wv = resolve_group_job<CONSTR>(a, S, latest, q2, ws);  // uniform across lanes
      n_group++;
      if (lane == 0) {
        if (wv >= 0) append(wv, ws);
        else S.chain = chain_pack(g + 1, c);
      }
    } else if (take_z) {
      n_fast++;
      n_ztake++;
      wv = r_zv;
      if (lane == 0) append(wv, R->c[KC].st);
    } else if (exact) {
      n_fast++;
      if (wf > 0.0) {
        wv = wv0;
        if (!take_new) {  // the winner's state: its log entry or its candidate record
          int vm2, kk;
          if (ps >= 0) ne = load_log<CONSTR>(S, ps, vm2, kk);
          else ne = R->c[(~ps) & (KC - 1)].st;
        }
        if (lane == 0) append(wv, ne);
      } else if (lane == 0) {
        S.chain = chain_pack(g + 1, c);  // assign / fail keep their defaults (-1, COOK_FAIL_CONSTRAINT)
      }
    } else {
      // recompute at the current version (exact): its one candidate is the answer
      const QEntry q2 = qe;
      const long long tf0 = PROF ? clock64() : 0;
      spec_job_fallback<CONSTR>(a, S, latest, q2, c);
      if (PROF) prof[5] += (unsigned long long)(clock64() - tf0);
      n_fallback++;
      const bool got = S.res[RING].n > 0;
      if (lane == 0) {
        if (got) append(S.res[RING].c[0].vm, S.res[RING].c[0].st);
        else S.chain = chain_pack(g + 1, c);
      }
      if (got) wv = 0;
    }
    // lane 0 stored the chain word on every path above
    const long long t_done = PROF ? clock64() : 0;   // the arrive belongs to the hand-off
    if (!CONSTR && lane == 0) mbar_arrive(&S.hand[g % NCW]);
    if (PROF) {
      const unsigned path = wv_group ? TP_GROUP : take_z ? TP_ZTAKE : exact ? TP_EXACT : TP_FALLBACK;
      trace_turn(t_ready, t_seen, t_eval, t_dec, 0, t_done, (unsigned long long)(path << 4 | min(n_rel, 15u) << 8 | min(n_fold, 255u) << 12 |
                                                          slow << 20 | (wv >= 0 ? 1u : 0u) << 21) |
                                         ((unsigned long long)qe.blk << 32), k,
                 (hp & HP_HAND) ? (1ull << 32 | t_hand) : 0ull, hp / HP_WAIT | (unsigned long long)((hp & HP_MID) ? 1u : 0u) << 32);
    }
    if (wv >= 0) n_matched++;
    __syncwarp();
    if (PROF) prof[2] += (unsigned long long)(clock64() - t2);
  }
  if (lane == 0) {
    atomicAdd(a.stats + 0, n_fast); atomicAdd(a.stats + 2, n_group); atomicAdd(a.stats + 3, n_matched);
    atomicAdd(a.stats + 4, n_fallback); atomicAdd(a.stats + 7, n_slow_turn); atomicAdd(a.stats + 24, n_ztake); atomicAdd(a.stats + 25, n_relook);
    for (int i = 0; i < 6; i++) atomicAdd(a.stats + 8 + i, prof[i]);
  }
}

// Pipeline.  The resolver CTA places block t while the evaluator CTAs score
// block t+1 against the state published after block t-1 (buffer (t+1)&1).
// Synchronisation across CTAs is by two monotone counters only:
//   rows_ready[b]  evaluators -> resolver (one arrival per scored row)
//   published      resolver -> evaluators (# blocks resolved and published)
template <bool CONSTR, bool PROF>
__global__ void __launch_bounds__(RES_THREADS, 1) match_kernel(MatchArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int ns = a.n_spec;
  if ((int)blockIdx.x <= ns) {
    // block 0: the resolver; blocks 1..ns: spec CTAs with a replica of the resolver's log
    constexpr int NCW = CONSTR ? NCW_CONSTR : NCW_PLAIN;
    ResolverShared& S = *reinterpret_cast<ResolverShared*>(smem_raw);
    Latest latest;
    const size_t res_base = (sizeof(ResolverShared) + 15) & ~size_t(15);
    unsigned* sbw_base = reinterpret_cast<unsigned*>(smem_raw + res_base);   // NCW rows of verdict bits
    latest.s = reinterpret_cast<int*>(smem_raw + res_base + (((size_t)NCW * a.sb_words * 4 + 15) & ~size_t(15)));
    latest.g = a.latest_global ? a.latest_global + (size_t)blockIdx.x * (size_t)(a.of.O + 1) : nullptr;
    const int warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < a.of.O; i += RES_THREADS) latest.set(i, -1);
    if (threadIdx.x < RING) S.q_seq[threadIdx.x] = 0;
    for (int i = threadIdx.x; i < LOGN; i += RES_THREADS) S.log[i].vm = 0;
    if (threadIdx.x == 0) {
      S.chain = 0ull; S.exit_g = -1; S.ticket = 0;
      S.lo_ring[0] = S.lo_ring[1] = S.lo_ring[2] = S.lo_ring[3] = 0;
      S.bk_ring[0] = 0; S.bk_ring[1] = a.B; S.bk_ring[2] = 2 * a.B; S.bk_known = 2;  // = host-initialised bk0[0..2]
      S.out_done = 0; S.blk_c0 = 0; S.last_b = a.B;
      for (int i = 0; i < RING; i++) mbar_init(&S.res_bar[i], 1u);
      for (int i = 0; i < NCW_MAX; i++) mbar_init(&S.hand[i], 1u);
      fence_proxy_async_smem();  // the barriers are visible to the async proxy (bulk copies complete on them)
    }
    __syncthreads();
    if (blockIdx.x == 0) {
      // warps 0..3 sit on different schedulers (warp id mod 4): one commit warp each, a fifth shares
      // warp 0's scheduler
      if (warp < NCW) commit_warp<CONSTR, PROF>(a, S, latest, warp, sbw_base + (size_t)warp * a.sb_words);
      else if (warp == NCW) driver_warp<CONSTR, false, PROF>(a, S);
      else if (warp == NCW + 1) publisher_warp<CONSTR>(a, S);
      else if (warp == NCW + 2) fetcher_warp(a, S);
    } else {
      if (warp == 0) follower_warp<CONSTR>(a, S, latest);
      else if (warp == 1) driver_warp<CONSTR, true>(a, S);
      else if (warp < a.max_spec_warp) spec_warp<CONSTR>(a, S, latest, (int)blockIdx.x - 1);
    }
  } else {
    EvalStatic es;
    es.lc = es.lm = es.rc = es.rm = nullptr;
    EvalShared& E = *reinterpret_cast<EvalShared*>(smem_raw);
    if (a.vs_in_smem) {  // static VM table -> shared memory, SoA (conflict-free 64-bit reads)
      double* base = reinterpret_cast<double*>(smem_raw + ((sizeof(EvalShared) + 127) & ~size_t(127)));
      const size_t O = (size_t)a.of.O;
      double* lc = base; double* lm = base + O; double* rc = base + 2 * O; double* rm = base + 3 * O;
      for (int v = threadIdx.x; v < a.of.O; v += RES_THREADS) {
        const VmStatic x = a.of.vs[v];
        lc[v] = x.lc; lm[v] = x.lm; rc[v] = x.rc; rm[v] = x.rm;
      }
      __syncthreads();
      es.lc = lc; es.lm = lm; es.rc = rc; es.rm = rm;
    }
    __shared__ int bk_s[2];
    __shared__ double smin_s[2];
    __shared__ double red_c[NW], red_m[NW];
    SparseLive& SP = *reinterpret_cast<SparseLive*>(
        smem_raw + ((sizeof(EvalShared) + 127) & ~size_t(127)) + (a.vs_in_smem ? (size_t)a.of.O * 32 : 0));
    if ((threadIdx.x >> 5) >= NW) return;  // only NW warps score rows (exited threads do not block the barriers)
    const int n_eval = gridDim.x - 1 - ns;
    const int ei = (int)blockIdx.x - 1 - ns;   // this evaluator's index
    unsigned long long work = 0, wait = 0, work_q1 = 0, rows_q1 = 0, nblk_seen = 0, n_hopeless = 0;
    unsigned long long ep[3] = {0, 0, 0};
    // largest capacities of the cluster (static): scale of the rounding margin of the row pre-test below
    double capc = 0.0, capm = 0.0;
    {
      const double2* stb = reinterpret_cast<const double2*>(a.of.vs);
      for (int v = threadIdx.x; v < a.of.O; v += NW * 32) {
        double lc, lm;
        if (es.lc) { lc = es.lc[v]; lm = es.lm[v]; }
        else { const double2 s0 = __ldg(stb + 2 * v); lc = s0.x; lm = s0.y; }
        capc = fmax(capc, lc); capm = fmax(capm, lm);
      }
      for (int o = 16; o > 0; o >>= 1) { capc = fmax(capc, __shfl_xor_sync(0xffffffffu, capc, o)); capm = fmax(capm, __shfl_xor_sync(0xffffffffu, capm, o)); }
      if ((threadIdx.x & 31) == 0) { red_c[threadIdx.x >> 5] = capc; red_m[threadIdx.x >> 5] = capm; }
      __syncthreads();
      for (int w = 0; w < NW; w++) { capc = fmax(capc, red_c[w]); capm = fmax(capm, red_m[w]); }
      __syncthreads();
    }
    for (int b = 0;; b++) {
      long long w0 = clock64();
      // rows of block b need S_{b-2}: published >= b-1 (which also covers bk0[b], bk0[b+1])
      if (threadIdx.x == 0) {
        if (b >= 2) {
          // relaxed polling (an acquire load would invalidate L1 on every poll), one fence after
          while ((int)ld_relaxed_u32(a.published) < b - 1) __nanosleep(32);
          __threadfence();
        }
        bk_s[0] = __ldcg(a.bk0 + b);
        bk_s[1] = __ldcg(a.bk0 + b + 1);
        if (bk_s[0] < a.n_cons) { smin_s[0] = a.smin_c[bk_s[0]]; smin_s[1] = a.smin_m[bk_s[0]]; }
      }
      __syncthreads();
      const int k0 = bk_s[0];
      const int k1 = min(bk_s[1], a.n_cons);
      const double minc = smin_s[0], minm = smin_s[1];
      __syncthreads();  // bk_s is rewritten for the next block
      if (k0 >= a.n_cons) break;
      long long w1 = clock64();
      // live mask of the lane's VMs for this block's snapshot (bit u: VM 32*warp + lane + 32*NW*u):
      // dead = even the smallest request among the jobs from k0 on does not fit (exact: the
      // assigned amounts only grow within a cycle)
      unsigned long long live = ~0ull;
      // most room left on any live VM at this snapshot (cpus, mem): a job that asks for more than that
      // fits nowhere, now or later in the cycle - its row is not scored at all (pre-test below)
      double maxfc = 1.7976931348623157e308, maxfm = 1.7976931348623157e308;
      if (a.of.O <= 64 * 32 * NW) {
        live = 0ull;
        double fc = -1.0, fm = -1.0;
        const double2* dyb = reinterpret_cast<const double2*>(a.dyn.d[b & 1]);
        const double2* stb = reinterpret_cast<const double2*>(a.of.vs);
        int u = 0;
        for (int v = 32 * (threadIdx.x >> 5) + (threadIdx.x & 31); v < a.of.O; v += 32 * NW, u++) {
          const double2 d0 = __ldcg(dyb + 2 * v);
          double lc, lm;
          if (es.lc) { lc = es.lc[v]; lm = es.lm[v]; }
          else { const double2 s0 = __ldg(stb + 2 * v); lc = s0.x; lm = s0.y; }
          bool dead = (d0.x + minc > lc) | (d0.y + minm > lm);
          bool special = false;   // a VM only jobs of a special kind can use: a reserved host, a k8s GPU node
          if (CONSTR) {
            const int4* vcp = reinterpret_cast<const int4*>(a.of.vc + v);
            const int4 c0 = __ldg(vcp), c1 = __ldg(vcp + 1);
            const int an = __ldcg(reinterpret_cast<const int*>(a.dyn.n[b & 1] + v));
            // max-tasks-per-host reached (assigned counts only grow): no job can ever go there
            if (c0.z >= 0 && !(c0.w + an < c0.z)) dead = true;
            special = (c1.y & VC_RESERVED) || ((c1.y & VC_K8S) && (c1.y >> 8) != 0);
          }
          if (!dead) {
            live |= 1ull << u;
            if (!special) { fc = fmax(fc, lc - d0.x); fm = fmax(fm, lm - d0.y); }
          }
        }
        for (int o = 16; o > 0; o >>= 1) { fc = fmax(fc, __shfl_xor_sync(0xffffffffu, fc, o)); fm = fmax(fm, __shfl_xor_sync(0xffffffffu, fm, o)); }
        if ((threadIdx.x & 31) == 0) { red_c[threadIdx.x >> 5] = fc; red_m[threadIdx.x >> 5] = fm; }
        // every CTA sees all VMs: when none is live nothing from k0 on can ever be placed
        // (state only tightens) - all evaluators stop here and the drivers end the cycle
        if (!__syncthreads_or(live != 0ull)) {
          if (threadIdx.x == 0) atomicMax(a.dead_blk, b + 1);
          break;
        }
        maxfc = maxfm = -1.0;
        for (int w = 0; w < NW; w++) { maxfc = fmax(maxfc, red_c[w]); maxfm = fmax(maxfm, red_m[w]); }
      }
      // live VMs of every chunk compacted into shared memory; sparse mode when all lists fit
      bool sparse = false;
      if (a.of.O <= 64 * 32 * NW && a.sb_words <= SBW_MAX && a.sparse_ok) {
        if (threadIdx.x < 32) SP.cnt[threadIdx.x] = 0;
        __syncthreads();
        const int ln = threadIdx.x & 31, wp = threadIdx.x >> 5;
        for (unsigned long long m = live; m; m &= m - 1) {
          const int u = __ffsll((long long)m) - 1;
          const int pos = atomicAdd(&SP.cnt[ln], 1);
          if (pos < SL_MAX) SP.t[ln][pos] = (unsigned short)(wp + NW * u);   // tile of VM 32 * (wp + NW * u) + ln
        }
        __syncthreads();
        if (threadIdx.x < 32) {
          int mx = SP.cnt[threadIdx.x];
          for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
          if (threadIdx.x == 0) SP.maxc = mx;
        }
        __syncthreads();
        sparse = SP.maxc <= SL_MAX;
      }
      // the next row's job columns are fetched while this row is scored
      int k = k0 + ei;
      JobRegs rn;
      bool gn = false;
      if (k < k1) { rn = load_job<CONSTR>(a, k); gn = CONSTR && (a.kflags[k] & 1); }
      for (; k < k1; k += n_eval) {
        const JobRegs r = rn;
        const bool grp = gn;
        if (k + n_eval < k1) { rn = load_job<CONSTR>(a, k + n_eval); gn = CONSTR && (a.kflags[k + n_eval] & 1); }
        // pre-test (uniform over the CTA): the request exceeds the most room any live VM has, by more than
        // any rounding of `assigned + request > limit` could hide (margin 1e-9 x scale against 2^-52) =>
        // every VM fails the resource check; the row keeps its stale (infeasible) stamp
        // (constraint kernel: the room is that of the VMs any job may use; a gpu job or a job holding a
        // reservation could still go to a k8s GPU node / its reserved host and is always scored)
        const bool plain = !CONSTR || (r.g == 0.0 && !(a.jb.reserved_host && a.jb.reserved_host[r.j] >= 0));
        if (plain && ((r.c - maxfc) > 1e-9 * (capc + r.c) || (r.m - maxfm) > 1e-9 * (capm + r.m))) {
          if (threadIdx.x == 0)
            asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(a.rows_ready + b), "r"(1u) : "memory");
          n_hopeless++;
          continue;
        }
        evaluate_row<CONSTR, PROF>(a, r, grp, b, k - k0, es, E, live, ep, SP, sparse);
      }
      wait += (unsigned long long)(w1 - w0);
      const unsigned long long dt = (unsigned long long)(clock64() - w1);
      work += dt;
      if (PROF) { if (k0 < a.n_cons / 4) { work_q1 += dt; rows_q1 += (k1 - k0 + n_eval - 1) / n_eval; } nblk_seen++; }
    }
    if (ei == 0 && threadIdx.x == 0) {
      a.stats[16] = work; a.stats[17] = wait;
      if (PROF) { a.stats[18] = ep[0]; a.stats[19] = ep[1]; a.stats[20] = ep[2]; a.stats[21] = work_q1; a.stats[22] = rows_q1; a.stats[23] = nblk_seen; a.stats[26] = n_hopeless; }
    }
  }
}

// ------------------------------------------------------------ considerable
struct ConsArgs {
  const int32_t* ranked; int n_ranked;
  JobDev jb;
  int n_users;
  const double *q_count, *q_cpus, *q_mem, *q_gpus;
  const double *u_count, *u_cpus, *u_mem, *u_gpus;
  const int32_t* tokens;
  int enforce_rate_limit;
  cook_pool_quota pool_q;
  int num_considerable;
};

struct LessUserPos {
  const int32_t* ranked;
  const int32_t* user;
  __device__ bool operator()(int32_t a, int32_t b) const {
    int ua = user[ranked[a]], ub = user[ranked[b]];
    if (ua != ub) return ua < ub;
    return a < b;
  }
};

// tools.clj:903-915 + :940-959: warp per user, lane-serial left fold over the
// user's queued jobs in queue order, starting from the user's running usage.
__global__ void __launch_bounds__(128) cons_user_kernel(ConsArgs a, const int32_t* pos_by_user,
                                                        const int32_t* seg_start,
                                                        const int32_t* seg_end, uint8_t* keep, const GridFlag* gf) {
  const int u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (u >= a.n_users) return;
  const int s = seg_start[u], e = seg_end[u];
  if (e <= s) return;
  double acc[4] = {a.u_count ? a.u_count[u] : 0.0, a.u_cpus ? a.u_cpus[u] : 0.0, a.u_mem ? a.u_mem[u] : 0.0,
                    a.u_gpus ? a.u_gpus[u] : 0.0};
  const double qn = a.q_count[u], qc = a.q_cpus[u], qm = a.q_mem[u], qg = a.q_gpus[u];
  const int tokens = a.tokens ? a.tokens[u] : 0x7fffffff;
  __shared__ double stage[4][4][32];
  // No quota on any resource (quota.clj default = Double/MAX_VALUE) and no rate limit in
  // force: every finite running sum passes, so the order-dependent fold is not needed.
  const double dmax = 1.7976931348623157e308;
  if (qn >= dmax && qc >= dmax && qm >= dmax && qg >= dmax && !a.enforce_rate_limit) {
    for (int p = s + lane; p < e; p += 32) keep[pos_by_user[p]] = 1;
    return;
  }
  int seen = 0;
  // every partial sum exact (addends and start values on the 2^-10 grid, total below 2^43): a
  // parallel scan yields the left fold's bits; otherwise the lane-serial chain keeps the association
  const bool exact = grid_exact(gf, e - s, fmax(fmax(acc[0], acc[1]), fmax(acc[2], acc[3]))) && grid_value_ok(acc[0]) &&
                     grid_value_ok(acc[1]) && grid_value_ok(acc[2]) && grid_value_ok(acc[3]);
  for (int base0 = s; base0 < e; base0 += 128) {   // four chunks of gathers in flight
    double x4[4][4];   // count, cpus, mem, gpus
    int pos4[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int p = base0 + 32 * q + lane;
      x4[q][0] = x4[q][1] = x4[q][2] = x4[q][3] = 0.0; pos4[q] = -1;
      if (p < e) {
        pos4[q] = pos_by_user[p];
        const int j = a.ranked[pos4[q]];
        x4[q][0] = 1.0; x4[q][1] = a.jb.cpus[j]; x4[q][2] = a.jb.mem[j]; x4[q][3] = a.jb.gpus ? a.jb.gpus[j] : 0.0;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int base = base0 + 32 * q;
      if (base >= e) break;
      const int p = base + lane;
      warp_fold_prefix(x4[q], acc, min(32, e - base), exact, stage[threadIdx.x >> 5]);
      bool ok = (p < e) && (x4[q][0] <= qn && x4[q][1] <= qc && x4[q][2] <= qm && x4[q][3] <= qg);
      unsigned ob = __ballot_sync(0xffffffffu, ok);
      int kth = seen + __popc(ob & (0xffffffffu >> (31 - lane)));  // k-th surviving job of the user
      bool limited = kth > tokens;
      if (ok && limited && a.enforce_rate_limit) ok = false;
      if (p < e) keep[pos4[q]] = ok ? 1 : 0;
      seen += __popc(ob);
    }
  }
}

// The considerable set and its per-k hot columns, slot by slot.
struct ConsOut {
  int32_t* cons; double *kc, *km, *kg; int32_t* kports; uint8_t* kflags;
  __device__ void put(const JobDev& jb, int j, int slot) const {
    cons[slot] = j;
    kc[slot] = jb.cpus[j];
    km[slot] = jb.mem[j];
    kg[slot] = jb.gpus ? jb.gpus[j] : 0.0;
    kports[slot] = jb.ports ? jb.ports[j] : 0;
    uint8_t fl = 0;
    if (jb.group_off && jb.group_off[j + 1] > jb.group_off[j]) fl |= 1;
    kflags[slot] = fl;
  }
};

// Queue-order pass (single warp): pool quota over survivors (tools.clj:917-933),
// allowed + launch-plugin masks (scheduler.clj:749-750), take N (:751).
// Out::put(jb, j, slot) receives the slot-th considerable job j.
template <class Out>
__global__ void cons_queue_kernel(ConsArgs a, const uint8_t* keep, Out out, int32_t* out_n) {
  const int lane = threadIdx.x;
  __shared__ double stage[4][32];
  double pool[4] = {0.0, 0.0, 0.0, 0.0};   // count, cpus, mem, gpus
  if (a.pool_q.enabled)  // (reduce (partial merge-with +) (vals user->usage)), tools.clj:969
    warp_fold_sum<4, 1>(pool, a.n_users, false, [&](int u, double (&x)[4]) {
      x[0] = a.u_count ? a.u_count[u] : 0.0; x[1] = a.u_cpus ? a.u_cpus[u] : 0.0;
      x[2] = a.u_mem ? a.u_mem[u] : 0.0; x[3] = a.u_gpus ? a.u_gpus[u] : 0.0;
      return true;
    }, stage);
  int n_out = 0;
  for (int base = 0; base < a.n_ranked && n_out < a.num_considerable; base += 32) {
    int i = base + lane;
    bool k = i < a.n_ranked && keep[i];
    int j = i < a.n_ranked ? a.ranked[i] : 0;
    if (a.pool_q.enabled) {
      double x[4] = {0.0, 0.0, 0.0, 0.0}, mine[4] = {0.0, 0.0, 0.0, 0.0};
      if (k) { x[0] = 1.0; x[1] = a.jb.cpus[j]; x[2] = a.jb.mem[j]; x[3] = a.jb.gpus ? a.jb.gpus[j] : 0.0; }
      warp_chain(x, pool, mine, __ballot_sync(0xffffffffu, k), stage);
      if (k) k = mine[0] <= a.pool_q.count && mine[1] <= a.pool_q.cpus && mine[2] <= a.pool_q.mem && mine[3] <= a.pool_q.gpus;
    }
    if (k && a.jb.allowed && !a.jb.allowed[j]) k = false;
    if (k && a.jb.plugin && !a.jb.plugin[j]) k = false;
    unsigned kb = __ballot_sync(0xffffffffu, k);
    int slot = n_out + __popc(kb & ((1u << lane) - 1u));
    if (k && slot < a.num_considerable) out.put(a.jb, j, slot);
    n_out += __popc(kb);
  }
  if (lane == 0) *out_n = min(n_out, a.num_considerable);
}

// Parallel form of the queue-order pass for the common case of NO global pool
// quota (tools.clj:923 `(if (nil? quota) queue ...)`): the filters are then
// element-wise and "take N" is a stable compaction.
template <class Out>
struct ConsSurvivors {
  ConsArgs a; const uint8_t* kept; Out out;
  __device__ bool keep(int i) const {
    if (!kept[i]) return false;
    const int j = a.ranked[i];
    if (a.jb.allowed && !a.jb.allowed[j]) return false;
    if (a.jb.plugin && !a.jb.plugin[j]) return false;
    return true;
  }
  __device__ void emit(int i, int slot) const { out.put(a.jb, a.ranked[i], slot); }
};

// The considerable set as job indices alone (the resident state's considerable call).
struct ConsIdx {
  int32_t* cons;
  __device__ void put(const JobDev&, int j, int slot) const { cons[slot] = j; }
};

// M0 over the rows a.ranked names, after the caller zeroed seg_s / seg_e [n_users + 1]: the per-user order, its
// segments, the grid check of the J job rows, the per-user folds, then the queue-order pass (pool quota: one warp;
// else the stable compaction).  *count receives the number of considerable jobs.  Shared by cook_match and
// cook_state_considerable, so both run the same launches on the same columns.
template <class Out>
cudaError_t cons_pass(const ConsArgs& ca, int J, int32_t* pos, int32_t* tmp, int32_t* seg_s, int32_t* seg_e,
                      uint8_t* keep, GridFlag* gf, const Out& out, int32_t* count, cudaStream_t st, int* launches) {
  const int TB = 256, n = ca.n_ranked, U = ca.n_users;
  cudaError_t e = csort::sort_indices(pos, tmp, n, LessUserPos{ca.ranked, ca.jb.user}, st, launches);
  if (e != cudaSuccess) return e;
  seg_bounds_kernel<<<(n + TB - 1) / TB, TB, 0, st>>>(SortedKey{pos, ca.ranked, ca.jb.user}, n, seg_s, seg_e, nullptr);
  (*launches)++;
  if ((e = cudaMemsetAsync(gf, 0, sizeof(GridFlag), st)) != cudaSuccess) return e;
  grid_check_kernel<<<(J + TB - 1) / TB, TB, 0, st>>>(ca.jb.cpus, ca.jb.mem, ca.jb.gpus, J, gf);
  (*launches)++;
  cons_user_kernel<<<(U + 3) / 4, 128, 0, st>>>(ca, pos, seg_s, seg_e, keep, gf);
  (*launches)++;
  if (ca.pool_q.enabled) {
    // global pool quota: an order-dependent f64 left fold over the survivors
    // (filter-sequential) => exact single-warp pass
    cons_queue_kernel<<<1, 32, 0, st>>>(ca, keep, out, count);
    (*launches)++;
  } else {
    compact(ConsSurvivors<Out>{ca, keep, out}, n, nullptr, tmp, count, ca.num_considerable, st, launches);
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------ setup
__global__ void gather_offers_kernel(const int32_t* perm, int O, const double* c, const double* m,
                                     const double* rc, const double* rm, VmStatic* vs) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= O) return;
  int o = perm[v];
  VmStatic x;
  x.lc = c[o]; x.lm = m[o];
  x.rc = rc ? rc[o] : 0.0; x.rm = rm ? rm[o] : 0.0;
  vs[v] = x;
}

// suffix minima of the considerable jobs' requests: block-local reverse scans, then every
// block folds in the minima of the blocks to its right
constexpr int SMIN_TB = 256;
__global__ void __launch_bounds__(SMIN_TB) suffix_min_local_kernel(const double* kc, const double* km, int n,
                                                                   double* sc, double* sm, double* bc, double* bm) {
  __shared__ double wc[SMIN_TB / 32], wm[SMIN_TB / 32];
  const double INF = 1.7976931348623157e308;
  const int k = blockIdx.x * SMIN_TB + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double c = k < n ? kc[k] : INF, m = k < n ? km[k] : INF;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {  // reverse inclusive scan inside the warp
    const double oc = __shfl_down_sync(0xffffffffu, c, o), om = __shfl_down_sync(0xffffffffu, m, o);
    if (lane + o < 32) { c = fmin(c, oc); m = fmin(m, om); }
  }
  if (lane == 0) { wc[warp] = c; wm[warp] = m; }
  __syncthreads();
  for (int w = warp + 1; w < SMIN_TB / 32; w++) { c = fmin(c, wc[w]); m = fmin(m, wm[w]); }
  if (k < n) { sc[k] = c; sm[k] = m; }
  if (threadIdx.x == 0) { bc[blockIdx.x] = c; bm[blockIdx.x] = m; }
}
__global__ void __launch_bounds__(SMIN_TB) suffix_min_apply_kernel(int n, int nblocks, double* sc, double* sm,
                                                                   const double* bc, const double* bm) {
  __shared__ double wc[SMIN_TB / 32], wm[SMIN_TB / 32];
  const double INF = 1.7976931348623157e308;
  double c = INF, m = INF;
  for (int j = blockIdx.x + 1 + threadIdx.x; j < nblocks; j += SMIN_TB) { c = fmin(c, bc[j]); m = fmin(m, bm[j]); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { c = fmin(c, __shfl_xor_sync(0xffffffffu, c, o)); m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o)); }
  if ((threadIdx.x & 31) == 0) { wc[threadIdx.x >> 5] = c; wm[threadIdx.x >> 5] = m; }
  __syncthreads();
  c = INF; m = INF;
  for (int w = 0; w < SMIN_TB / 32; w++) { c = fmin(c, wc[w]); m = fmin(m, wm[w]); }
  const int k = blockIdx.x * SMIN_TB + threadIdx.x;
  if (k < n) { sc[k] = fmin(sc[k], c); sm[k] = fmin(sm[k], m); }
}

// offer-side constraint inputs gathered into rank space (one record per VM) + attribute table
__global__ void gather_cons_kernel(OfferDev of, VmCons* vc, int32_t* attr_v) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= of.O) return;
  const int o = of.perm[v];
  VmCons c;
  c.hostname_id = of.hostname_id ? of.hostname_id[o] : -1;
  c.location = of.location ? of.location[o] : -1;
  c.max_tasks = of.max_tasks ? of.max_tasks[o] : -1;
  c.num_tasks = of.num_tasks ? of.num_tasks[o] : 0;
  c.run_count = of.run_count ? of.run_count[o] : 0;
  const int gn = of.gpu_off ? of.gpu_off[o + 1] - of.gpu_off[o] : 0;
  c.flags = ((of.is_k8s && of.is_k8s[o]) ? VC_K8S : 0) | ((of.reserved && of.reserved[o]) ? VC_RESERVED : 0) | (gn << 8);
  c.gpu_lo = of.gpu_off ? of.gpu_off[o] : 0;
  c.ports_total = of.ports_total ? of.ports_total[o] : 0;
  c.host_start = of.host_start ? of.host_start[o] : -1;
  c.disk_lo = of.disk_off ? of.disk_off[o] : 0;
  c.disk_n = of.disk_off ? of.disk_off[o + 1] - of.disk_off[o] : 0;
  vc[v] = c;
  for (int col = 0; col < of.n_attr_cols; col++) attr_v[(size_t)col * of.O + v] = of.attr[(size_t)col * of.O + o];
}

// per-cycle reset of the dynamic state (both buffers) + the reciprocals of the fitness
// denominators (static for the cycle)
__global__ void init_dyn_kernel(const VmStatic* vs, int O, VmDyn* d0, VmDyn* d1, VmCnt* n0, VmCnt* n1) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= O) return;
  const VmStatic x = vs[v];
  VmDyn d;
  d.ac = 0.0; d.am = 0.0;
  d.yc = safe_rcp(x.lc + x.rc);
  d.ym = safe_rcp(x.lm + x.rm);
  d0[v] = d; d1[v] = d;
  VmCnt c;
  c.an = 0; c.pu = 0;
  n0[v] = c; n1[v] = c;
}

__global__ void ports_total_kernel(const int32_t* off, const int32_t* b, const int32_t* e, int O,
                                   int32_t* total) {
  int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= O) return;
  int t = 0;
  for (int k = off[o]; k < off[o + 1]; k++) t += e[k] - b[k] + 1;
  total[o] = t;
}

// assign (rank space) -> original offer index; assigned port numbers
// (FENZO F6: first n free ports scanning ranges in lease order).
__global__ void finalize_kernel(MatchArgs a, int32_t* out_assign, int32_t* out_ports, int max_ports,
                                int32_t* used_flag) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.n_cons) return;
  // the cycle ended early: from dead_k0 on no VM could take even the smallest request left
  const int dk = *a.dead_k0;
  if (dk >= 0 && k >= dk) a.fail[k] = COOK_FAIL_RESOURCES;
  int v = a.assign[k];
  int o = v >= 0 ? a.of.perm[v] : -1;
  out_assign[k] = o;
  if (v >= 0) used_flag[v] = 1;
  if (out_ports && max_ports > 0) {
    for (int p = 0; p < max_ports; p++) out_ports[(size_t)k * max_ports + p] = -1;
    int want = (o >= 0 && a.jb.ports) ? a.jb.ports[a.cons[k]] : 0;
    if (want > 0 && a.of.port_off) {
      int skip = a.ports_start[k], got = 0;
      for (int r = a.of.port_off[o]; r < a.of.port_off[o + 1] && got < want; r++) {
        int len = a.of.port_end[r] - a.of.port_begin[r] + 1;
        if (skip >= len) { skip -= len; continue; }
        for (int p = a.of.port_begin[r] + skip; p <= a.of.port_end[r] && got < want; p++) {
          if (got < max_ports) out_ports[(size_t)k * max_ports + got] = p;
          got++;
        }
        skip = 0;
      }
    }
  }
}

// ---- placement-failure summaries (SURVEY §8f-3): why job k could not go to each VM at its turn.
// One CTA per requested job; thread per VM.  The VM's state at the job's turn is rebuilt exactly:
// a left fold, in queue order, over the earlier jobs of the cycle that were placed on it.
__global__ void __launch_bounds__(256) explain_kernel(MatchArgs a, const int32_t* k_list, int n_list,
                                                      cook_failure_counts* out) {
  __shared__ int s_cnt[COOK_FAILC_N + 2];
  const int k = k_list[blockIdx.x];
  if (threadIdx.x < COOK_FAILC_N + 2) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  if (k < 0 || k >= a.n_cons) {
    if (threadIdx.x == 0) { cook_failure_counts z; memset(&z, 0, sizeof(z)); z.n_vms = -1; out[blockIdx.x] = z; }
    return;
  }
  const int j = a.cons[k];
  JobRegs r;
  r.c = a.kc[k]; r.m = a.km[k]; r.j = j;
  r.g = a.kg ? a.kg[k] : 0.0; r.ports = a.kports ? a.kports[k] : 0;
  const bool has_cons = a.of.vc != nullptr && a.sb_words > 0;
  const bool grp = has_cons && (a.kflags[k] & 1);
  for (int v = threadIdx.x; v < a.of.O; v += blockDim.x) {
    const VmStatic vs = a.of.vs[v];
    double ac = 0.0, am = 0.0;
    int an = 0, pu = 0;
    for (int q = 0; q < k; q++)               // broadcast loads: every thread walks the same queue
      if (a.assign[q] == v) { ac = ac + a.kc[q]; am = am + a.km[q]; an++; pu += a.kports ? a.kports[q] : 0; }
    const bool no_c = ac + r.c > vs.lc, no_m = am + r.m > vs.lm;
    bool no_p = false;
    if (has_cons && r.ports > 0) no_p = r.ports > a.of.vc[v].ports_total - pu;
    if (no_c) atomicAdd(&s_cnt[COOK_FAILC_CPUS], 1);
    if (no_m) atomicAdd(&s_cnt[COOK_FAILC_MEM], 1);
    if (no_p) atomicAdd(&s_cnt[COOK_FAILC_N + 1], 1);
    if (no_c || no_m || no_p) continue;        // Fenzo evaluates constraints only when the resources fit
    int first = has_cons ? first_failing_constraint(a, r, v, an) : -1;
    if (first < 0 && grp)   // the members Fenzo knew at the job's turn: those placed by the jobs before k
      first = first_failing_group(a, j, v, [&](int g) {
        int n = 0;
        for (int k2 = 0; k2 < k; k2++) {
          if (!(a.kflags[k2] & 1) || a.assign[k2] < 0) continue;
          const int j2 = a.cons[k2];
          for (int e = a.jb.group_off[j2]; e < a.jb.group_off[j2 + 1]; e++) n += a.jb.group_idx[e] == g;
        }
        return n;
      });
    if (first >= 0) atomicAdd(&s_cnt[COOK_FAILC_FIRST_CONSTRAINT + first], 1);
    else atomicAdd(&s_cnt[COOK_FAILC_N], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    cook_failure_counts c;
    c.n_vms = a.of.O; c.n_passed = s_cnt[COOK_FAILC_N]; c.n_ports = s_cnt[COOK_FAILC_N + 1];
    for (int i = 0; i < COOK_FAILC_N; i++) c.counts[i] = s_cnt[i];
    out[blockIdx.x] = c;
  }
}

// ---- usage delta of a match round (SURVEY §8e): jobs placed this cycle, per user
__global__ void placed_flag_kernel(const int32_t* cons, const int32_t* out_assign, int n_cons, uint8_t* placed_job) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n_cons && out_assign[k] >= 0) placed_job[cons[k]] = 1;
}
// exact-grid amounts: the sums do not depend on the order, one atomic add per placed job and column
// (lanes of a warp that share the user are combined first)
__global__ void usage_delta_exact_kernel(ConsArgs a, const int32_t* cons, const int32_t* out_assign, int n_cons,
                                         double* delta /* [n_users][4] */, const GridFlag* gf) {
  if (!grid_exact(gf, n_cons)) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool placed = k < n_cons && out_assign[k] >= 0;
  const unsigned act = __ballot_sync(0xffffffffu, placed);
  if (!placed) return;
  const int j = cons[k], u = a.jb.user[j];
  double xn = 1.0, xc = a.jb.cpus[j], xm = a.jb.mem[j], xg = a.jb.gpus ? a.jb.gpus[j] : 0.0;
  const unsigned peers = __match_any_sync(act, u);
  const int leader = __ffs(peers) - 1;
  for (unsigned m = peers & ~(1u << leader); m; m &= m - 1) {   // the leader gathers its peers' amounts
    const int l = __ffs(m) - 1;
    const double yn = __shfl_sync(peers, xn, l), yc = __shfl_sync(peers, xc, l), ym = __shfl_sync(peers, xm, l), yg = __shfl_sync(peers, xg, l);
    if (lane == leader) { xn = xn + yn; xc = xc + yc; xm = xm + ym; xg = xg + yg; }
  }
  if (lane == leader) {
    atomicAdd(&delta[4 * u], xn); atomicAdd(&delta[4 * u + 1], xc); atomicAdd(&delta[4 * u + 2], xm); atomicAdd(&delta[4 * u + 3], xg);
  }
}
// warp per user: left fold over the user's queued jobs in queue order (pos_by_user), placed jobs only
__global__ void __launch_bounds__(128) usage_delta_kernel(ConsArgs a, const int32_t* pos_by_user, const int32_t* seg_start,
                                                          const int32_t* seg_end, const uint8_t* placed_job,
                                                          double* delta /* [n_users][4] */, const GridFlag* gf, int n_cons) {
  if (grid_exact(gf, n_cons)) return;   // usage_delta_exact_kernel did it
  const int u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (u >= a.n_users) return;
  const int s = seg_start[u], e = seg_end[u];
  __shared__ double stage[4][4][32];
  double d[4] = {0.0, 0.0, 0.0, 0.0};
  warp_fold_sum<4, 4>(d, e - s, grid_exact(gf, e - s), [&](int k, double (&x)[4]) {
    const int j = a.ranked[pos_by_user[s + k]];
    if (!placed_job[j]) return false;   // only the placed ones add (x + 0.0 == x anyway)
    x[0] = 1.0; x[1] = a.jb.cpus[j]; x[2] = a.jb.mem[j]; x[3] = a.jb.gpus ? a.jb.gpus[j] : 0.0;
    return true;
  }, stage[threadIdx.x >> 5]);
  if (lane == 0) { delta[4 * u] = d[0]; delta[4 * u + 1] = d[1]; delta[4 * u + 2] = d[2]; delta[4 * u + 3] = d[3]; }
}

__global__ void cons_job_id_kernel(const int32_t* cons, const int64_t* job_id, int n, int64_t* out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = job_id[cons[k]];
}

__global__ void count_flags_kernel(const int32_t* flags, int n, int32_t* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int v = (i < n && flags[i]) ? 1 : 0;
  unsigned b = __ballot_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(out, __popc(b));
}

}  // namespace

// ------------------------------------------------------------------ host side
// A MatchPlan is the device-resident image of one cook_match call's inputs plus
// all scratch.  With params->reuse_resident the upload stage is skipped (the
// inputs of the previous call on this handle are still in HBM) and only the
// kernels + result download run — the "inputs already resident" measurement.
struct MatchPlan {
  Arena arena;
  bool valid = false;
  int J = 0, O = 0, U = 0, n_ranked = 0, NC = 0, max_ports = 0, G = 0, B = 0;
  bool constr = false;
  size_t n_memb = 0;
  int64_t h2d_bytes = 0;
  ConsArgs ca;
  MatchArgs ma;
  // scratch
  int32_t *d_perm = nullptr, *d_pos = nullptr, *d_tmp = nullptr, *d_seg_s = nullptr, *d_seg_e = nullptr;
  uint8_t* d_keep = nullptr;
  uint8_t* d_placed = nullptr;
  GridFlag* d_gf = nullptr;
  int last_n_cons = 0;
  double *d_oc = nullptr, *d_om = nullptr, *d_orc = nullptr, *d_orm = nullptr;
  VmStatic* d_vs = nullptr;
  double* d_kg = nullptr;
  int32_t* d_kports = nullptr;
  int32_t* d_ports_total = nullptr;
  VmCons* d_vc = nullptr;
  int32_t* d_attr_v = nullptr;
  int32_t *d_cons = nullptr, *d_out_assign = nullptr, *d_out_ports = nullptr, *d_used = nullptr;
  double *d_kc = nullptr, *d_km = nullptr;
  uint8_t* d_kflags = nullptr;
  unsigned long long* d_stats = nullptr;
  int32_t* d_counters = nullptr;
  int* d_latest = nullptr;
  unsigned long long* d_gchain = nullptr;
  size_t lo_g_n = 0;
  double *d_smin_c = nullptr, *d_smin_m = nullptr, *d_smin_bc = nullptr, *d_smin_bm = nullptr;
  size_t max_blocks = 0;
  int32_t bk_init[3] = {0, 0, 0};
  int64_t* d_job_id = nullptr;    // device-source plans: job id per row, and per considerable job
  int64_t* d_cons_jid = nullptr;
  uint64_t runs = 0;              // match_run calls on this plan: what identifies a round (match_round)
};

static void plan_free(void* p) {
  MatchPlan* mp = static_cast<MatchPlan*>(p);
  if (mp) { mp->arena.release(); delete mp; }
}

// The pool's plan, made on first use.
static MatchPlan* plan_of(cook_pool* pool) {
  if (!pool->match_plan) {
    pool->match_plan = new MatchPlan();
    pool->match_plan_free = plan_free;
  }
  return static_cast<MatchPlan*>(pool->match_plan);
}

// A job column of the plan: carved when the shape has it, and filled from the host when the shape uploads.
template <class T>
static T* job_col(Carve& c, const JobShape& sh, const T* col, size_t n) {
  if (!col) return nullptr;
  T* d = c.take<T>(n ? n : 1);
  if (sh.upload) c.copy(d, col, n);
  return d;
}

OfferShape host_offer_shape(const cook_offers_soa* offers) {
  OfferShape s;
  const int O = offers->n;
  s.O = O;
  s.host = offers;
  s.hostname_id = offers->hostname_id;
  s.ports = offers->port_off; s.n_ports = s.ports ? offers->port_off[O] : 0;
  s.is_k8s = offers->is_k8s; s.location = offers->location;
  s.gpu = offers->gpu_off; s.n_gpu = s.gpu ? offers->gpu_off[O] : 0;
  s.disk = offers->disk_off; s.n_disk = s.disk ? offers->disk_off[O] : 0;
  s.max_tasks = offers->max_tasks; s.num_tasks = offers->num_tasks; s.host_start = offers->host_start_time;
  s.reserved = offers->reserved;
  s.n_attr_cols = offers->attr ? offers->n_attr_cols : 0;
  return s;
}

// An offer column of the plan: the host table's, uploaded, or carved for the caller when the shape has it.
template <class T>
static T* offer_col(Carve& c, const OfferShape& osh, const T* col, bool has, size_t n) {
  if (osh.host) return c.up(col, n);
  return has ? c.take<T>(n ? n : 1) : nullptr;
}

int32_t match_build(cook_pool* pool, const int32_t* ranked_idx, int32_t n_ranked, const JobShape& sh,
                    const OfferShape& osh, const cook_groups* groups, const cook_user_table* users,
                    const cook_pool_quota* pool_quota, const cook_match_params* params, int32_t max_ports,
                    MatchRows* rows) {
  cudaStream_t st = pool->stream;
  MatchPlan* mp = plan_of(pool);
  Arena& ar = mp->arena;
  const JobDev& jc = sh.cols;
  const int J = sh.J, O = osh.O, U = users->n_users, NC = params->num_considerable;
  const cook_offers_soa none = {};
  const cook_offers_soa* offers = osh.host ? osh.host : &none;
  mp->valid = false;
  // host-side prep: offers sorted by hostname rank (tie-break order); without a host table the VMs come in it
  std::vector<int32_t> perm(osh.host ? O : 0, -1);
  bool dense = true;  // name_rank is normally a permutation of 0..O-1: invert it directly
  for (int i = 0; i < (int)perm.size() && dense; i++) {
    const int32_t r = offers->name_rank[i];
    if (r < 0 || r >= O || perm[r] >= 0) dense = false; else perm[r] = i;
  }
  if (!dense) {
    std::iota(perm.begin(), perm.end(), 0);
    std::stable_sort(perm.begin(), perm.end(),
                     [&](int32_t x, int32_t y) { return offers->name_rank[x] < offers->name_rank[y]; });
  }
  // per-group capacity of the placed list = #member jobs
  const int G = groups ? groups->n_groups : 0;
  const bool grouped = jc.group_off && G;
  const size_t n_memb = grouped ? sh.gp_off[G] : 0;
  // The cpu+mem-only kernel is used when no constraint column can affect a
  // placement (all-zero ports/gpus columns count as absent).
  const bool constr_eff = jc.novel_off || jc.gpu_model || jc.disk_request || jc.attr_off || jc.est_end_ms ||
                          jc.ckpt_location || jc.reserved_host || grouped || osh.is_k8s || osh.max_tasks ||
                          osh.reserved || osh.gpu || sh.any_gpus_ports;

  // blocks: B jobs at the start, then sized by the resolver to ~btarget placements per block
  int B = 64, bmin = 64, bmax = MAXB, btarget = 32;
  // constraint pools: a scored row costs several times a cpu+mem row and a block is at most one row per
  // evaluator CTA while the cluster fills - longer blocks amortise the per-block hand-offs (on an H100
  // within 1 % of the best of 64 / 128 / 256-row blocks on config-#3 and config-#5 pools)
  if (constr_eff) { B = 128; bmin = 128; btarget = 64; }
  if (const char* eb = getenv("COOK_MATCH_B")) { int v = atoi(eb); if (v >= 8 && v <= MAXB) B = v; }
  if (const char* eb = getenv("COOK_MATCH_BMIN")) { int v = atoi(eb); if (v >= 8 && v <= MAXB) bmin = v; }
  if (const char* eb = getenv("COOK_MATCH_BMAX")) { int v = atoi(eb); if (v >= 8 && v <= MAXB) bmax = v; }
  if (const char* eb = getenv("COOK_MATCH_TARGET")) { int v = atoi(eb); if (v >= 1) btarget = v; }
  bmax = std::max(bmax, std::max(B, bmin));
  const size_t max_blocks = (size_t)NC / std::min(B, bmin) + 8;
  ConsArgs& ca = mp->ca;
  MatchArgs& ma = mp->ma;
  JobDev jb;
  OfferDev of;
  GroupDev gr;
  int32_t* ranked = nullptr;
  double* usage = nullptr;
  memset(&ca, 0, sizeof(ca));
  memset(&ma, 0, sizeof(ma));
  memset(&jb, 0, sizeof(jb));
  memset(&of, 0, sizeof(of));
  memset(&gr, 0, sizeof(gr));
  of.O = O;
  of.n_attr_cols = osh.n_attr_cols;
  OfferCols oc = {};
  mp->h2d_bytes = 0;
  const cudaError_t carved = carve(ar, st, nullptr, &mp->h2d_bytes, [&](Carve& c) {
    ranked = c.take<int32_t>(n_ranked ? n_ranked : 1);
    if (ranked_idx) c.copy(ranked, ranked_idx, n_ranked);
    jb.user = job_col(c, sh, jc.user, J);
    jb.cpus = job_col(c, sh, jc.cpus, J);
    jb.mem = job_col(c, sh, jc.mem, J);
    jb.gpus = job_col(c, sh, jc.gpus, J);
    jb.ports = job_col(c, sh, jc.ports, J);
    jb.allowed = job_col(c, sh, jc.allowed, J);
    jb.plugin = job_col(c, sh, jc.plugin, J);
    if (jc.novel_off) {
      jb.novel_off = job_col(c, sh, jc.novel_off, J + 1);
      jb.novel_host = job_col(c, sh, jc.novel_host, std::max<size_t>(1, sh.n_novel));
    }
    jb.gpu_model = job_col(c, sh, jc.gpu_model, J);
    jb.disk_request = job_col(c, sh, jc.disk_request, J);
    jb.disk_type = job_col(c, sh, jc.disk_type, J);
    if (jc.attr_off) {
      const size_t na = std::max<size_t>(1, sh.n_attr);
      jb.attr_off = job_col(c, sh, jc.attr_off, J + 1);
      jb.attr_col = job_col(c, sh, jc.attr_col, na);
      jb.attr_val = job_col(c, sh, jc.attr_val, na);
    }
    jb.est_end_ms = job_col(c, sh, jc.est_end_ms, J);
    jb.ckpt_location = job_col(c, sh, jc.ckpt_location, J);
    jb.reserved_host = job_col(c, sh, jc.reserved_host, J);
    if (grouped) {
      jb.group_off = job_col(c, sh, jc.group_off, J + 1);
      jb.group_idx = job_col(c, sh, jc.group_idx, std::max<size_t>(1, n_memb));
    }
    mp->d_job_id = sh.job_ids ? c.take<int64_t>(J + 1) : nullptr;
    mp->d_cons_jid = sh.job_ids ? c.take<int64_t>(NC + 1) : nullptr;

    mp->d_perm = offer_col(c, osh, perm.data(), true, O); of.perm = mp->d_perm;
    mp->d_oc = offer_col(c, osh, offers->cpus, true, O); mp->d_om = offer_col(c, osh, offers->mem, true, O);
    if (sh.dev.run) {
      mp->d_orc = c.take<double>(O ? O : 1); mp->d_orm = c.take<double>(O ? O : 1);
    } else {
      mp->d_orc = c.up(offers->run_cpus, O); mp->d_orm = c.up(offers->run_mem, O);
    }
    mp->d_vs = c.take<VmStatic>(O + 1); of.vs = mp->d_vs;
    of.hostname_id = c.up(osh.hostname_id, O);
    of.run_count = sh.dev.run ? c.take<int32_t>(O ? O : 1) : c.up(offers->run_count, O);
    mp->d_ports_total = nullptr;
    if (osh.ports) {
      const int np = std::max<int64_t>(1, osh.n_ports);
      of.port_off = offer_col(c, osh, offers->port_off, true, O + 1);
      of.port_begin = offer_col(c, osh, offers->port_begin, true, np);
      of.port_end = offer_col(c, osh, offers->port_end, true, np);
      mp->d_ports_total = c.take<int32_t>(O + 1); of.ports_total = mp->d_ports_total;
    }
    of.is_k8s = offer_col(c, osh, offers->is_k8s, osh.is_k8s, O);
    of.reserved = offer_col(c, osh, offers->reserved, osh.reserved, O);
    of.location = offer_col(c, osh, offers->location, osh.location, O);
    if (osh.gpu) {
      const int ng = std::max<int64_t>(1, osh.n_gpu);
      of.gpu_off = offer_col(c, osh, offers->gpu_off, true, O + 1);
      of.gpu_model = offer_col(c, osh, offers->gpu_model, true, ng);
      of.gpu_count = offer_col(c, osh, offers->gpu_count, true, ng);
    }
    if (osh.disk) {
      const int nd = std::max<int64_t>(1, osh.n_disk);
      of.disk_off = offer_col(c, osh, offers->disk_off, true, O + 1);
      of.disk_type = offer_col(c, osh, offers->disk_type, true, nd);
      of.disk_space = offer_col(c, osh, offers->disk_space, true, nd);
    }
    of.max_tasks = offer_col(c, osh, offers->max_tasks, osh.max_tasks, O);
    of.num_tasks = offer_col(c, osh, offers->num_tasks, osh.num_tasks, O);
    of.host_start = offer_col(c, osh, offers->host_start_time, osh.host_start, O);
    if (of.n_attr_cols > 0) of.attr = offer_col(c, osh, offers->attr, true, (size_t)of.n_attr_cols * O);
    if (!osh.host)
      oc = OfferCols{mp->d_perm, mp->d_oc, mp->d_om, writable(of.port_off), writable(of.port_begin),
                     writable(of.port_end), writable(of.is_k8s), writable(of.location), writable(of.gpu_off),
                     writable(of.gpu_model), writable(of.gpu_count), writable(of.disk_off), writable(of.disk_type),
                     writable(of.disk_space), writable(of.max_tasks), writable(of.num_tasks),
                     writable(of.host_start), writable(of.attr), writable(of.reserved)};
    mp->d_vc = c.take<VmCons>(O + 1);
    mp->d_attr_v = c.take<int32_t>((size_t)of.n_attr_cols * O + 1);
    of.vc = mp->d_vc; of.attr_v = mp->d_attr_v;

    if (grouped) {
      gr.n_groups = G;
      gr.kind = c.up(groups->kind, G);
      gr.attr_col = c.up(groups->attr_col, G);
      gr.minimum = c.up(groups->minimum, G);
      if (sh.dev.cot) {
        const size_t nc = std::max<int64_t>(1, sh.dev.n_cot);
        gr.cot_off = c.take<int32_t>(G + 1);
        gr.cot_host = c.take<int32_t>(nc); gr.cot_attr = c.take<int32_t>(nc);
      } else {
        gr.cot_off = c.up(groups->cot_off, G + 1);
        const int nc = std::max(1, groups->cot_off[G]);
        gr.cot_host = c.up(groups->cot_hostname_id, nc);
        gr.cot_attr = c.up(groups->cot_attr_val, nc);
      }
      gr.gp_off = c.up(sh.gp_off.data(), G + 1);
      gr.gp_n = c.take<int32_t>(G + 1);
      gr.gp_vm = c.take<int32_t>(n_memb + 1);
    }
    ca.q_count = c.up(users->quota_count, U); ca.q_cpus = c.up(users->quota_cpus, U);
    ca.q_mem = c.up(users->quota_mem, U); ca.q_gpus = c.up(users->quota_gpus, U);
    if (sh.dev.usage) {
      usage = c.take<double>(4 * (size_t)U);
      ca.u_count = usage; ca.u_cpus = usage ? usage + U : nullptr;
      ca.u_mem = usage ? usage + 2 * U : nullptr; ca.u_gpus = usage ? usage + 3 * U : nullptr;
    } else {
      ca.u_count = c.up(users->usage_count, U); ca.u_cpus = c.up(users->usage_cpus, U);
      ca.u_mem = c.up(users->usage_mem, U); ca.u_gpus = c.up(users->usage_gpus, U);
    }
    ca.tokens = c.up(users->tokens, U);

    for (int b = 0; b < 2; b++) {
      ma.dyn.d[b] = c.take<VmDyn>(O + 1);
      ma.dyn.n[b] = c.take<VmCnt>(O + 1);
    }
    mp->d_pos = c.take<int32_t>(n_ranked + 1);
    mp->d_tmp = c.take<int32_t>(n_ranked + 1);
    mp->d_seg_s = c.take<int32_t>(U + 1);
    mp->d_seg_e = c.take<int32_t>(U + 1);
    mp->d_keep = c.take<uint8_t>(n_ranked + 1);
    mp->d_placed = c.take<uint8_t>(J + 1);
    mp->d_gf = c.take<GridFlag>(1);
    mp->d_cons = c.take<int32_t>(NC + 1);
    mp->d_kc = c.take<double>(NC + 1);
    mp->d_km = c.take<double>(NC + 1);
    mp->d_kflags = c.take<uint8_t>(NC + 1);
    ma.rows = c.take<unsigned char>((size_t)2 * bmax * ROW_BYTES);
    ma.sbits = c.take<unsigned>((size_t)2 * bmax * ((O + 31) / 32) + 4);
    mp->d_kg = c.take<double>(NC + bmax + 1);
    mp->d_kports = c.take<int32_t>(NC + bmax + 1);
    ma.feas = c.take<int32_t>(2 * bmax + 16);
    mp->d_smin_c = c.take<double>(NC + 1);
    mp->d_smin_m = c.take<double>(NC + 1);
    mp->d_smin_bc = c.take<double>(NC / 256 + 2);
    mp->d_smin_bm = c.take<double>(NC / 256 + 2);
    ma.rows_ready = c.take<unsigned>(max_blocks + 8);
    ma.bk0 = c.take<int32_t>(max_blocks + 8);
    ma.assign = c.take<int32_t>(NC + 1);
    ma.ports_start = c.take<int32_t>(NC + 1);
    ma.fail = c.take<uint8_t>(NC + 1);
    mp->d_out_assign = c.take<int32_t>(NC + 1);
    mp->d_out_ports = c.take<int32_t>((size_t)NC * std::max(max_ports, 1) + 1);
    mp->d_used = c.take<int32_t>(O + 1);
    mp->d_stats = c.take<unsigned long long>(32);
    mp->d_counters = c.take<int32_t>(16);
    mp->d_latest = c.take<int>((size_t)(MAX_SPEC_CTAS + 1) * (O + 1));
    ma.glog = c.take<LogEnt>(LOGN);
    ma.glogx = c.take<int4>(LOGN);
    mp->d_gchain = c.take<unsigned long long>(4);
    ma.lo_g = c.take<int32_t>(max_blocks + 8);
    ma.gres = c.take<SpecOut>(GRING);
    ma.gres_seq = c.take<unsigned>(GRING);
  });
  CK(pool, carved);
  ca.ranked = ranked; ca.n_ranked = n_ranked; ca.jb = jb; ca.n_users = U;
  ca.enforce_rate_limit = params->enforce_rate_limit;
  cook_pool_quota qoff{0, 0, 0, 0, 0};
  ca.pool_q = pool_quota ? *pool_quota : qoff;
  ca.num_considerable = NC;
  ma.kg = mp->d_kg; ma.kports = mp->d_kports;
  ma.smin_c = mp->d_smin_c; ma.smin_m = mp->d_smin_m;
  mp->max_blocks = max_blocks;
  ma.gchain = mp->d_gchain;
  mp->lo_g_n = max_blocks + 8;
  ma.jb = jb; ma.of = of; ma.gr = gr;
  ma.cons = mp->d_cons; ma.kc = mp->d_kc; ma.km = mp->d_km; ma.kflags = mp->d_kflags;
  ma.B = B; ma.bmin = bmin; ma.bmax = bmax; ma.btarget = btarget;
  ma.host_lifetime_mins = params->host_lifetime_mins;
  ma.published = reinterpret_cast<unsigned*>(mp->d_counters + 8); ma.stats = mp->d_stats;
  ma.dead_blk = mp->d_counters + 9; ma.dead_k0 = mp->d_counters + 10;
  ma.lookahead = 31;   // the most the 32-lane first look allows: the results' way back is about a dozen job-times long
  ma.poll_ns = 200;
  ma.max_spec_warp = RES_THREADS / 32;
  ma.spec_kmin = 12;
  if (const char* ek = getenv("COOK_KMIN")) ma.spec_kmin = atoi(ek);
  if (const char* ew = getenv("COOK_MAX_SPEC_WARP")) ma.max_spec_warp = atoi(ew);
  if (const char* ep = getenv("COOK_POLL_NS")) ma.poll_ns = atoi(ep);
  if (const char* el = getenv("COOK_LOOKAHEAD")) { int v = atoi(el); if (v >= 2 && v <= RING - 1) ma.lookahead = v; }
  mp->J = J; mp->O = O; mp->U = U; mp->n_ranked = n_ranked; mp->NC = NC; mp->max_ports = max_ports;
  mp->G = G; mp->B = B; mp->constr = constr_eff; mp->n_memb = n_memb;
  if (rows) {
    const bool run = sh.dev.run, cot = sh.dev.cot && grouped;
    *rows = MatchRows{jb, ranked, mp->d_job_id, usage, run ? mp->d_orc : nullptr, run ? mp->d_orm : nullptr,
                      run ? writable(of.run_count) : nullptr, cot ? writable(gr.cot_off) : nullptr,
                      cot ? writable(gr.cot_host) : nullptr, cot ? writable(gr.cot_attr) : nullptr, of.hostname_id,
                      of.attr, gr.attr_col, oc};
  }
  return COOK_OK;
}

// out_job_id (plans with job ids): the job id of every considerable job
int32_t match_run(cook_pool* pool, int32_t* out_considerable, int64_t* out_job_id, int32_t* out_assign,
                  int32_t* out_ports, uint8_t* out_fail_reason, cook_match_stats* out_stats, bool uploaded, int max_ctas) {
  MatchPlan* mp = plan_of(pool);
  mp->valid = true;   // the plan's inputs are complete: a caller that writes its rows did so before the run
  mp->runs++;
  cudaStream_t st = pool->stream;
  const int O = mp->O, U = mp->U, max_ports = mp->max_ports;
  MatchArgs& ma = mp->ma;
  ConsArgs& ca = mp->ca;
  int launches = 0;
  // ---- reset of per-cycle dynamic state
  if (ma.gr.gp_n) CK(pool, cudaMemsetAsync(ma.gr.gp_n, 0, sizeof(int32_t) * (mp->G + 1), st));
  CK(pool, cudaMemsetAsync(mp->d_seg_s, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(mp->d_seg_e, 0, sizeof(int32_t) * (U + 1), st));
  CK(pool, cudaMemsetAsync(mp->d_used, 0, sizeof(int32_t) * (O + 1), st));
  CK(pool, cudaMemsetAsync(mp->d_stats, 0, sizeof(unsigned long long) * 32, st));
  CK(pool, cudaMemsetAsync(mp->d_counters, 0, sizeof(int32_t) * 16, st));
  CK(pool, cudaMemsetAsync(mp->d_counters + 10, 0xff, sizeof(int32_t), st));   // dead_k0 = -1
  CK(pool, cudaMemsetAsync(mp->d_gchain, 0, sizeof(unsigned long long) * 4, st));
  CK(pool, cudaMemsetAsync(ma.gres_seq, 0, sizeof(unsigned) * GRING, st));
  CK(pool, cudaMemsetAsync(ma.lo_g, 0, sizeof(int32_t) * 4, st));
  CK(pool, cudaMemsetAsync(ma.rows_ready, 0, sizeof(unsigned) * (mp->max_blocks + 8), st));
  CK(pool, cudaMemsetAsync(ma.feas, 0, sizeof(int32_t) * (2 * (size_t)mp->ma.bmax + 16), st));
  {  // first three block bounds; the resolver appends the rest while it runs
    mp->bk_init[0] = 0; mp->bk_init[1] = mp->B; mp->bk_init[2] = 2 * mp->B;
    CK(pool, cudaMemcpyAsync(ma.bk0, mp->bk_init, sizeof(mp->bk_init), cudaMemcpyHostToDevice, st));
  }
  CK(pool, cudaEventRecord(pool->ev[1], st));

  // ---- M0 considerable
  const int TB = 256;
  if (O > 0) {
    gather_offers_kernel<<<(O + TB - 1) / TB, TB, 0, st>>>(mp->d_perm, O, mp->d_oc, mp->d_om, mp->d_orc,
                                                           mp->d_orm, mp->d_vs);
    launches++;
    init_dyn_kernel<<<(O + TB - 1) / TB, TB, 0, st>>>(mp->d_vs, O, ma.dyn.d[0], ma.dyn.d[1], ma.dyn.n[0], ma.dyn.n[1]);
    launches++;
    if (mp->d_ports_total) {
      ports_total_kernel<<<(O + TB - 1) / TB, TB, 0, st>>>(ma.of.port_off, ma.of.port_begin,
                                                           ma.of.port_end, O, mp->d_ports_total);
      launches++;
    }
    if (mp->constr) {
      gather_cons_kernel<<<(O + TB - 1) / TB, TB, 0, st>>>(ma.of, mp->d_vc, mp->d_attr_v);
      launches++;
    }
  }
  const ConsOut cons_out{mp->d_cons, mp->d_kc, mp->d_km, mp->d_kg, mp->d_kports, mp->d_kflags};
  CK(pool, cons_pass(ca, mp->J, mp->d_pos, mp->d_tmp, mp->d_seg_s, mp->d_seg_e, mp->d_keep, mp->d_gf, cons_out,
                     mp->d_counters, st, &launches));
  int32_t n_cons = 0;
  int64_t d2h = 0;
  CK(pool, download(&n_cons, mp->d_counters, 1, st, &d2h));
  CK(pool, cudaEventRecord(pool->ev[2], st));
  CK(pool, cudaStreamSynchronize(st));

  // ---- M3 matcher
  ma.n_cons = n_cons;
  int n_used = 0;
  unsigned long long hstats[32] = {0};
  const bool prof_on = getenv("COOK_PROF") != nullptr;
  const char* trace_path = prof_on ? getenv("COOK_PROF_TRACE") : nullptr;
  // The timeline's pointers are device globals of this module: PROF runs go one at a time per process, so
  // that two pools on one device do not arm them over each other.  The buffer is freed on every return.
  static std::mutex prof_mu;
  std::unique_lock<std::mutex> prof_lock(prof_mu, std::defer_lock);
  if (prof_on) prof_lock.lock();
  struct TraceBuf {
    unsigned long long* p = nullptr;
    ~TraceBuf() { if (p) cudaFree(p); }
  } trace;
  int trace_caps[2] = {0, 0};
  CK(pool, cudaEventRecord(pool->ev[5], st));
  if (n_cons > 0) {
    if (O == 0) {
      CK(pool, cudaMemsetAsync(ma.assign, 0xff, sizeof(int32_t) * n_cons, st));
      CK(pool, cudaMemsetAsync(ma.fail, COOK_FAIL_NO_OFFERS, n_cons, st));
    } else {
      {
        const int nsb = (n_cons + SMIN_TB - 1) / SMIN_TB;
        suffix_min_local_kernel<<<nsb, SMIN_TB, 0, st>>>(mp->d_kc, mp->d_km, n_cons, mp->d_smin_c, mp->d_smin_m,
                                                         mp->d_smin_bc, mp->d_smin_bm);
        suffix_min_apply_kernel<<<nsb, SMIN_TB, 0, st>>>(n_cons, nsb, mp->d_smin_c, mp->d_smin_m, mp->d_smin_bc,
                                                         mp->d_smin_bm);
        launches += 2;
      }
      // defaults for feasible-but-unplaced jobs; the kernel overwrites placed and skipped ones
      CK(pool, cudaMemsetAsync(ma.assign, 0xff, sizeof(int32_t) * n_cons, st));
      CK(pool, cudaMemsetAsync(ma.fail, COOK_FAIL_CONSTRAINT, n_cons, st));
      // resolver CTA: shared structures + the per-VM newest-log-entry table (global when too big)
      ma.sb_words = mp->constr ? (O + 31) / 32 : 0;
      const size_t res_base = ((sizeof(ResolverShared) + 15) & ~size_t(15)) +
                              (((size_t)NCW_CONSTR * ma.sb_words * 4 + 15) & ~size_t(15));   // sb_words: constraint pools only
      size_t smem = res_base;
      ma.latest_global = nullptr;
      if (res_base + sizeof(int) * (size_t)O <= 200 * 1024) smem = std::max(smem, res_base + sizeof(int) * (size_t)O);
      else ma.latest_global = mp->d_latest;
      // evaluator CTAs: the static VM table (4 f64 per VM, SoA) when it fits
      const size_t ev_base = (sizeof(EvalShared) + 127) & ~size_t(127);
      ma.vs_in_smem = ev_base + (size_t)O * 32 + sizeof(SparseLive) <= 224 * 1024 ? 1 : 0;
      if (getenv("COOK_NO_SMEM_STATIC")) ma.vs_in_smem = 0;
      ma.sparse_ok = getenv("COOK_NO_SPARSE") ? 0 : 1;
      smem = std::max(smem, ev_base + (ma.vs_in_smem ? (size_t)O * 32 : 0) + sizeof(SparseLive));
      void* kfn = mp->constr ? (prof_on ? (void*)match_kernel<true, true> : (void*)match_kernel<true, false>)
                             : (prof_on ? (void*)match_kernel<false, true> : (void*)match_kernel<false, false>);
      {
        // The attribute belongs to the function on the device, not to this handle, and handles of
        // one GPU may run concurrently: raise it monotonically under a process-wide lock so that
        // a pool with a smaller offer table never lowers it under another pool's launch.
        static std::mutex mu;
        static int cur[16][4] = {};
        std::lock_guard<std::mutex> lk(mu);
        const int vi = (mp->constr ? 2 : 0) + (prof_on ? 1 : 0), di = pool->device & 15;
        if ((int)smem > cur[di][vi]) {
          int optin = 0;
          CK(pool, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, pool->device));
          cudaFuncAttributes fa;
          CK(pool, cudaFuncGetAttributes(&fa, kfn));
          optin -= (int)fa.sharedSizeBytes;   // the opt-in limit covers static + dynamic shared memory
          const int want = std::max((int)smem, optin);
          CK(pool, cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, std::min(want, optin)));
          cur[di][vi] = std::min(want, optin);
        }
        if ((int)smem > cur[di][vi])
          return set_err(pool, COOK_E_TOO_LARGE,
                         "cook_match: the offer table does not fit the kernel's shared memory (constraint pools: the verdict-bit "
                         "rows of the four owners bound a pool at about 130k offers) - split the pool");
      }
      int grid = pool->sm_count;
      if (max_ctas > 0) grid = std::min(grid, max_ctas);  // pools sharing one GPU
      int occ = 0;
      CK(pool, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, RES_THREADS, smem));
      if (occ < 1) return set_err(pool, COOK_E_CUDA, "cook_match: kernel does not fit on an SM");
      // roles: block 0 resolves, blocks 1..n_spec compute candidate sets, the rest score rows
      if (grid < 3) grid = 3;
      int n_spec = 3;
      if (const char* es = getenv("COOK_NSPEC")) n_spec = atoi(es);
      n_spec = std::max(1, std::min(n_spec, std::min(MAX_SPEC_CTAS, std::max(1, grid / 8))));
      n_spec = std::min(n_spec, grid - 2);
      ma.n_spec = n_spec;
      if (prof_on) {  // per-turn timeline: armed only when a file asks for it
        int caps[2] = {0, 0};
        if (trace_path) {
          caps[0] = n_cons + mp->max_blocks + 8;
          caps[1] = mp->max_blocks + 8;
          CK(pool, cudaMalloc(&trace.p, sizeof(unsigned long long) * ((size_t)caps[0] * TURN_WORDS + caps[1])));
          CK(pool, cudaMemsetAsync(trace.p, 0, sizeof(unsigned long long) * ((size_t)caps[0] * TURN_WORDS + caps[1]), st));
        }
        unsigned long long* d_blk = trace.p ? trace.p + (size_t)caps[0] * TURN_WORDS : nullptr;
        CK(pool, cudaMemcpyToSymbolAsync(g_turn_trace, &trace.p, sizeof(trace.p), 0, cudaMemcpyHostToDevice, st));
        CK(pool, cudaMemcpyToSymbolAsync(g_blk_trace, &d_blk, sizeof(d_blk), 0, cudaMemcpyHostToDevice, st));
        CK(pool, cudaMemcpyToSymbolAsync(g_turn_cap, &caps[0], sizeof(int), 0, cudaMemcpyHostToDevice, st));
        CK(pool, cudaMemcpyToSymbolAsync(g_blk_cap, &caps[1], sizeof(int), 0, cudaMemcpyHostToDevice, st));
        CK(pool, cudaStreamSynchronize(st));   // the caps live on this stack frame
        trace_caps[0] = caps[0]; trace_caps[1] = caps[1];
      }
      void* kargs[] = {&ma};
      CK(pool, cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(RES_THREADS), kargs, smem, st));
      launches++;
    }
  }
  CK(pool, cudaEventRecord(pool->ev[6], st));
  if (n_cons > 0) {
    finalize_kernel<<<(n_cons + TB - 1) / TB, TB, 0, st>>>(ma, mp->d_out_assign,
                                                           out_ports ? mp->d_out_ports : nullptr,
                                                           max_ports, mp->d_used);
    count_flags_kernel<<<(O + TB) / TB, TB, 0, st>>>(mp->d_used, O, mp->d_counters + 1);
    launches += 2;
    if (out_job_id && mp->d_cons_jid) {
      cons_job_id_kernel<<<(n_cons + TB - 1) / TB, TB, 0, st>>>(mp->d_cons, mp->d_job_id, n_cons, mp->d_cons_jid);
      launches++;
    }
    CK(pool, cudaGetLastError());
  }
  CK(pool, cudaEventRecord(pool->ev[3], st));
  if (n_cons > 0) {
    if (out_considerable) CK(pool, download(out_considerable, mp->d_cons, n_cons, st, &d2h));
    if (out_job_id && mp->d_cons_jid) CK(pool, download(out_job_id, mp->d_cons_jid, n_cons, st, &d2h));
    CK(pool, download(out_assign, mp->d_out_assign, n_cons, st, &d2h));
    if (out_ports && max_ports > 0) CK(pool, download(out_ports, mp->d_out_ports, (size_t)n_cons * max_ports, st, &d2h));
    if (out_fail_reason) CK(pool, download(out_fail_reason, ma.fail, n_cons, st, &d2h));
    CK(pool, download(hstats, mp->d_stats, 32, st, &d2h));
    CK(pool, download(&n_used, mp->d_counters + 1, 1, st, &d2h));
  }
  CK(pool, cudaEventRecord(pool->ev[4], st));
  CK(pool, cudaStreamSynchronize(st));
  if (prof_on) {
    const char* nm[27] = {"fast", "chunk_rescan", "group_jobs", "matched", "fallbacks", "trunc_specs",
                          "skipped", "slow_turns", "c_wait_result", "c_follow_log", "c_decide_commit", "c_to_argmax",
                          "c_end_block", "c_fallback", "res_total", "res_q1_done", "eval_work", "eval_wait",
                          "eval_loop", "eval_sync", "eval_merge", "eval_work_q1", "eval_rowslots_q1", "blocks", "z_takes", "relooks", "rows_pretest_ei0"};
    for (int i = 0; i < 27; i++) fprintf(stderr, "[cook_prof] %-14s %llu\n", nm[i], hstats[i]);
  }
  if (trace.p) {
    // header (8 x i64): magic, turn rows, block rows, words per turn row, resolver clocks, n_cons, matched, 0
    const size_t nw = (size_t)trace_caps[0] * TURN_WORDS + trace_caps[1];
    std::vector<unsigned long long> h(8 + nw);
    h[0] = 0x314e5254ull; h[1] = trace_caps[0]; h[2] = trace_caps[1]; h[3] = TURN_WORDS;
    h[4] = hstats[14]; h[5] = (unsigned long long)n_cons; h[6] = hstats[3]; h[7] = 0;
    CK(pool, cudaMemcpy(h.data() + 8, trace.p, nw * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (FILE* f = fopen(trace_path, "wb")) {
      fwrite(h.data(), sizeof(unsigned long long), h.size(), f);
      fclose(f);
    }
  }
  mp->last_n_cons = n_cons;
  record_phase(pool, COOK_PHASE_MATCH, uploaded ? pool->ev[0] : nullptr, pool->ev[1], pool->ev[3], pool->ev[4],
               uploaded ? mp->h2d_bytes : 0, d2h, launches);
  if (out_stats) {
    const cook_phase_stats& ps = pool->phase[COOK_PHASE_MATCH];
    out_stats->n_considerable = n_cons;
    out_stats->n_matched = (int)hstats[3];
    out_stats->head_matched = (n_cons > 0 && out_assign[0] >= 0) ? 1 : 0;
    out_stats->n_offers_used = n_used;
    out_stats->evals = (int64_t)n_cons * O;
    out_stats->n_fast = (int64_t)(hstats[0] + hstats[6]);
    out_stats->n_chunk_rescan = (int64_t)(hstats[1] + hstats[4]);
    out_stats->n_full_rescan = (int64_t)hstats[2];
    out_stats->ms_h2d = ps.ms_h2d;
    out_stats->ms_considerable = ev_ms(pool->ev[1], pool->ev[2]);
    out_stats->ms_match = ev_ms(pool->ev[2], pool->ev[3]);
    out_stats->ms_match_kernel = ev_ms(pool->ev[5], pool->ev[6]);
    out_stats->ms_d2h = ps.ms_d2h;
    out_stats->n_launches = ps.n_launches;
    out_stats->h2d_bytes = ps.h2d_bytes;
    out_stats->d2h_bytes = ps.d2h_bytes;
  }
  return COOK_OK;
}

uint64_t match_runs(cook_pool* pool) { return pool->match_plan ? static_cast<MatchPlan*>(pool->match_plan)->runs : 0; }

bool match_round(cook_pool* pool, uint64_t run, int32_t* n_cons, const int32_t** cons, const int32_t** assign) {
  const MatchPlan* mp = static_cast<const MatchPlan*>(pool->match_plan);
  if (!mp || !mp->valid || mp->runs != run) return false;
  *n_cons = mp->last_n_cons;
  *cons = mp->d_cons;
  *assign = mp->d_out_assign;
  return true;
}

cudaError_t considerable_rows(const ConsRows& r, cudaStream_t st, int* launches) {
  ConsArgs ca;
  memset(&ca, 0, sizeof(ca));
  ca.ranked = r.ranked; ca.n_ranked = r.n;
  ca.jb.user = r.user; ca.jb.cpus = r.cpus; ca.jb.mem = r.mem; ca.jb.gpus = r.gpus;
  ca.jb.allowed = r.allowed; ca.jb.plugin = r.plugin;
  ca.n_users = r.n_users;
  ca.q_count = r.quota[0]; ca.q_cpus = r.quota[1]; ca.q_mem = r.quota[2]; ca.q_gpus = r.quota[3];
  ca.u_count = r.usage[0]; ca.u_cpus = r.usage[1]; ca.u_mem = r.usage[2]; ca.u_gpus = r.usage[3];
  ca.tokens = r.tokens;
  ca.enforce_rate_limit = r.enforce_rate_limit;
  ca.pool_q = r.pool_q;
  ca.num_considerable = r.num_considerable;
  const size_t segs = sizeof(int32_t) * ((size_t)r.n_users + 1);
  cudaError_t e = cudaMemsetAsync(r.seg_s, 0, segs, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(r.seg_e, 0, segs, st);
  if (e != cudaSuccess) return e;
  return cons_pass(ca, r.n, r.pos, r.tmp, r.seg_s, r.seg_e, r.keep, r.gf, ConsIdx{r.out_row}, r.out_n, st, launches);
}

bool match_last_usage(cook_pool* pool, int n_users, const double* (&usage)[4]) {
  const MatchPlan* mp = static_cast<const MatchPlan*>(pool->match_plan);
  if (!mp || !mp->valid || mp->U != n_users) return false;
  usage[0] = mp->ca.u_count; usage[1] = mp->ca.u_cpus; usage[2] = mp->ca.u_mem; usage[3] = mp->ca.u_gpus;
  return true;
}

int32_t check_match_inputs(cook_pool* pool, const char* who, const cook_offers_soa* offers, const cook_groups* groups,
                           const cook_user_table* users, const cook_match_params* params, int32_t max_ports,
                           bool tables, bool novel, bool grouped, bool cot_derived) {
  if (params->good_enough_fitness < 1.0)
    return set_err(pool, COOK_E_BADARG,
                   "%s: good_enough_fitness < 1.0 is Fenzo's racy early-exit mode; "
                   "only the deterministic mode (>= 1.0) is supported", who);
  if (params->fitness_kind != 0) return set_err(pool, COOK_E_UNSUPPORTED_CONSTRAINT, "%s: only cpuMemBinPacker", who);
  const int O = offers->n;
  if (O < 0 || users->n_users <= 0 || params->num_considerable < 0 || max_ports < 0)
    return set_err(pool, COOK_E_BADARG, "%s: bad sizes", who);
  if (!tables) return COOK_OK;
  if (!offers->name_rank && O > 0) return set_err(pool, COOK_E_BADARG, "%s: offers.name_rank required", who);
  if (groups && !idx_in_range(groups->attr_col, groups->n_groups, -1, std::max(1, offers->n_attr_cols)))
    return set_err(pool, COOK_E_BADARG, "%s: groups.attr_col out of range", who);
  grouped = grouped && groups && groups->n_groups;
  if ((novel || offers->reserved || grouped) && !offers->hostname_id)
    return set_err(pool, COOK_E_BADARG, "%s: hostname_id column required by constraints", who);
  if (grouped && ((!cot_derived && !groups->cot_off) || !groups->kind)) return set_err(pool, COOK_E_BADARG, "%s: incomplete cook_groups", who);
  return COOK_OK;
}

// The shape of host-table jobs: their columns as given, uploaded; the group members counted per group.
static int32_t host_shape(cook_pool* pool, const cook_jobs_soa* jobs, int G, JobShape* sh) {
  const int J = jobs->n;
  sh->J = J;
  sh->cols = JobDev{jobs->user, jobs->cpus, jobs->mem, jobs->gpus, jobs->ports, jobs->allowed, jobs->plugin_accept,
                    jobs->novel_off, jobs->novel_host, jobs->gpu_model, jobs->disk_request, jobs->disk_type,
                    jobs->attr_off, jobs->attr_col, jobs->attr_val, jobs->est_end_ms, jobs->ckpt_location,
                    jobs->reserved_host, jobs->group_off, jobs->group_idx};
  sh->upload = true;
  sh->n_novel = jobs->novel_off ? jobs->novel_off[J] : 0;
  sh->n_attr = jobs->attr_off ? jobs->attr_off[J] : 0;
  sh->n_group = jobs->group_off ? jobs->group_off[J] : 0;
  if (G && jobs->group_off) {
    sh->gp_off.assign(G + 1, 0);
    for (int64_t i = 0; i < sh->n_group; i++) {
      const int g = jobs->group_idx[i];
      if (g < 0 || g >= G) return set_err(pool, COOK_E_BADARG, "cook_match: bad group index");
      sh->gp_off[g + 1]++;
    }
    for (int g = 0; g < G; g++) sh->gp_off[g + 1] += sh->gp_off[g];
  }
  if (jobs->gpus)
    for (int j = 0; j < J && !sh->any_gpus_ports; j++) sh->any_gpus_ports = jobs->gpus[j] != 0.0;
  if (jobs->ports)
    for (int j = 0; j < J && !sh->any_gpus_ports; j++) sh->any_gpus_ports = jobs->ports[j] != 0;
  return COOK_OK;
}

extern "C" int32_t cook_match(cook_pool* pool, const int32_t* ranked_idx, int32_t n_ranked,
                              const cook_jobs_soa* jobs, const cook_offers_soa* offers,
                              const cook_groups* groups, const cook_user_table* users,
                              const cook_pool_quota* pool_quota, const cook_match_params* params,
                              int32_t* out_considerable, int32_t* out_assign, int32_t* out_ports,
                              int32_t max_ports, uint8_t* out_fail_reason,
                              cook_match_stats* out_stats) {
  if (!pool) return COOK_E_BADARG;
  if (!ranked_idx || !jobs || !offers || !users || !params || !out_considerable || !out_assign)
    return set_err(pool, COOK_E_BADARG, "cook_match: null argument");
  const int J = jobs->n, O = offers->n, U = users->n_users;
  const int NC = params->num_considerable;
  int32_t rc = check_match_inputs(pool, "cook_match", offers, groups, users, params, max_ports,
                                  !params->reuse_resident && n_ranked > 0 && NC > 0, jobs->novel_off, jobs->group_off);
  if (rc != COOK_OK) return rc;
  if (J < 0 || n_ranked < 0) return set_err(pool, COOK_E_BADARG, "cook_match: bad sizes");
  if (out_stats) memset(out_stats, 0, sizeof(*out_stats));
  if (n_ranked == 0 || NC == 0) return COOK_OK;
  if (!params->reuse_resident) {   // index columns are dereferenced on the device: check them here
    if (!idx_in_range(ranked_idx, n_ranked, 0, J)) return set_err(pool, COOK_E_BADARG, "cook_match: ranked_idx out of range");
    if (!idx_in_range(jobs->user, J, 0, U)) return set_err(pool, COOK_E_BADARG, "cook_match: jobs.user out of range");
    if (jobs->attr_off && !idx_in_range(jobs->attr_col, jobs->attr_off[J], 0, std::max(1, offers->n_attr_cols)))
      return set_err(pool, COOK_E_BADARG, "cook_match: jobs.attr_col out of range");
  }
  CK(pool, cudaSetDevice(pool->device));
  MatchPlan* mp = plan_of(pool);
  const bool reuse = params->reuse_resident && mp->valid && mp->J == J && mp->O == O && mp->U == U &&
                     mp->n_ranked == n_ranked && mp->NC == NC && mp->max_ports == max_ports;
  if (params->reuse_resident && !reuse)
    return set_err(pool, COOK_E_BADARG,
                   "cook_match: reuse_resident set but no matching resident inputs on this handle");
  CK(pool, cudaEventRecord(pool->ev[0], pool->stream));
  if (!reuse) {
    mp->valid = false;
    JobShape sh;
    rc = host_shape(pool, jobs, groups ? groups->n_groups : 0, &sh);
    if (rc == COOK_OK)
      rc = match_build(pool, ranked_idx, n_ranked, sh, host_offer_shape(offers), groups, users, pool_quota, params,
                       max_ports, nullptr);
    if (rc != COOK_OK) return rc;
  }
  return match_run(pool, out_considerable, nullptr, out_assign, out_ports, out_fail_reason, out_stats, !reuse,
                   params->max_ctas);
}

// §8e: usage delta of this handle's last match round (device) -> one all-gather -> host.
// the per-user usage delta of `src`'s last match round into d_local[n_pad] (zeroed by the caller), on stream st
static int32_t usage_delta_launch(cook_pool* pool, cook_pool* src, cudaStream_t st, double* d_local, int32_t n_pad,
                                  int* launches) {
  MatchPlan* mp = static_cast<MatchPlan*>(src->match_plan);
  const bool have = mp && mp->valid;
  if (have && 4 * mp->U > n_pad) return set_err(pool, COOK_E_BADARG, "cook_exchange_usage: n_pad < 4 * n_users");
  if (have && mp->last_n_cons > 0) {
    const int TB = 256, nc = mp->last_n_cons;
    CK(pool, cudaMemsetAsync(mp->d_placed, 0, mp->J + 1, st));
    placed_flag_kernel<<<(nc + TB - 1) / TB, TB, 0, st>>>(mp->d_cons, mp->d_out_assign, nc, mp->d_placed);
    usage_delta_exact_kernel<<<(nc + TB - 1) / TB, TB, 0, st>>>(mp->ca, mp->d_cons, mp->d_out_assign, nc, d_local, mp->d_gf);
    usage_delta_kernel<<<(mp->U + 3) / 4, 128, 0, st>>>(mp->ca, mp->d_pos, mp->d_seg_s, mp->d_seg_e, mp->d_placed, d_local, mp->d_gf, nc);
    *launches += 3;
    CK(pool, cudaGetLastError());
  }
  return COOK_OK;
}

// deltas of n_pools handles of this rank (slot i = pools[i], the slots beyond n_pools stay zero), ONE all-gather
static int32_t exchange_run(cook_pool* const* pools, int32_t n_pools, void* comm, int32_t world, int32_t n_pad,
                            int32_t n_slots, double* out_all) {
  cook_pool* pool = pools[0];
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  const size_t per_rank = (size_t)n_slots * n_pad;
  const size_t need = (size_t)(world + 1) * per_rank;
  if (need > pool->xchg_cap) {
    if (pool->xchg) cudaFree(pool->xchg);
    pool->xchg = nullptr; pool->xchg_cap = 0;
    CK(pool, cudaMalloc(&pool->xchg, need * sizeof(double)));
    pool->xchg_cap = need;
  }
  double* d_local = pool->xchg;
  double* d_all = pool->xchg + per_rank;
  int launches = 0;
  CK(pool, cudaEventRecord(pool->ev[16], st));
  CK(pool, cudaMemsetAsync(d_local, 0, sizeof(double) * per_rank, st));
  for (int i = 0; i < n_pools; i++) {
    // the other handles' match rounds have completed (cook_match returns after its stream is idle):
    // their result arrays are read from this handle's stream
    int32_t rc = usage_delta_launch(pool, pools[i], st, d_local + (size_t)i * n_pad, n_pad, &launches);
    if (rc != COOK_OK) return rc;
  }
  if (world > 1 && comm) {
    int32_t rc = cook_allgather_usage(comm, st, d_local, d_all, (int64_t)per_rank);
    if (rc != COOK_OK) return set_err(pool, rc, "cook_exchange_usage: ncclAllGather failed");
    launches += 1;
  } else {
    d_all = d_local;
    if (world != 1) return set_err(pool, COOK_E_BADARG, "cook_exchange_usage: world > 1 needs a communicator");
  }
  CK(pool, cudaEventRecord(pool->ev[17], st));
  int64_t d2h = 0;
  CK(pool, download(out_all, d_all, (size_t)world * per_rank, st, &d2h));
  CK(pool, cudaEventRecord(pool->ev[18], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_EXCHANGE, nullptr, pool->ev[16], pool->ev[17], pool->ev[18], 0, d2h, launches);
  return COOK_OK;
}

extern "C" int32_t cook_exchange_usage(cook_pool* pool, void* comm, int32_t world, int32_t n_pad, double* out_all) {
  if (!pool || !out_all || world <= 0 || n_pad <= 0) return set_err(pool, COOK_E_BADARG, "cook_exchange_usage: bad argument");
  cook_pool* one[1] = {pool};
  return exchange_run(one, 1, comm, world, n_pad, 1, out_all);
}

extern "C" int32_t cook_exchange_usage_batch(cook_pool* const* pools, int32_t n_pools, void* comm, int32_t world,
                                             int32_t n_pad, int32_t n_slots, double* out_all) {
  if (!pools || n_pools <= 0 || !pools[0]) return COOK_E_BADARG;
  cook_pool* pool = pools[0];
  if (!out_all || world <= 0 || n_pad <= 0 || n_slots < n_pools)
    return set_err(pool, COOK_E_BADARG, "cook_exchange_usage_batch: bad argument");
  for (int i = 1; i < n_pools; i++)
    if (!pools[i] || pools[i]->device != pool->device)
      return set_err(pool, COOK_E_BADARG, "cook_exchange_usage_batch: the handles of one call live on one device");
  return exchange_run(pools, n_pools, comm, world, n_pad, n_slots, out_all);
}


// §8f-3: per-job placement-failure counters of the last match on this handle.
extern "C" int32_t cook_match_failures(cook_pool* pool, const int32_t* k_idx, int32_t n, cook_failure_counts* out) {
  if (!pool || !k_idx || !out || n < 0) return set_err(pool, COOK_E_BADARG, "cook_match_failures: bad argument");
  MatchPlan* mp = static_cast<MatchPlan*>(pool->match_plan);
  if (!mp || !mp->valid || mp->last_n_cons <= 0)
    return set_err(pool, COOK_E_BADARG, "cook_match_failures: no match round on this handle");
  if (n == 0) return COOK_OK;
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  int32_t* d_k = nullptr;
  cook_failure_counts* d_out = nullptr;
  CK(pool, cudaMalloc(&d_k, sizeof(int32_t) * n));
  cudaError_t e = cudaMalloc(&d_out, sizeof(cook_failure_counts) * n);
  if (e != cudaSuccess) { cudaFree(d_k); return set_err(pool, COOK_E_OOM, "cook_match_failures: out of memory"); }
  cudaMemcpyAsync(d_k, k_idx, sizeof(int32_t) * n, cudaMemcpyHostToDevice, st);
  MatchArgs ma = mp->ma;
  ma.n_cons = mp->last_n_cons;
  if (!mp->constr) ma.sb_words = 0;
  explain_kernel<<<n, 256, 0, st>>>(ma, d_k, n, d_out);
  cudaMemcpyAsync(out, d_out, sizeof(cook_failure_counts) * n, cudaMemcpyDeviceToHost, st);
  e = cudaStreamSynchronize(st);
  cudaFree(d_k);
  cudaFree(d_out);
  if (e != cudaSuccess) return set_err(pool, COOK_E_CUDA, "cook_match_failures: %s", cudaGetErrorString(e));
  return COOK_OK;
}
