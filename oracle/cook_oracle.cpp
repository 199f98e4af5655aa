// cook_oracle.cpp — CPU restatement of Cook's per-cycle scheduling hot path.
//
// *** TEST INFRASTRUCTURE ONLY. ***  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load this library.  The
// product path (cook_b200/, libcookgpu.so) never links or calls it and has no
// CPU fallback.
//
// Parity status: the reference (Clojure on the JVM + Netflix Fenzo 0.10.0)
// cannot run in this container (no JVM, no Maven cache; SURVEY.md §8c).  This
// file is a line-by-line restatement of the cited Clojure sources, PINNED
// against the reference's own known-answer tests transcribed in tests/golden/
// and tests/*_golden*.py (K1-K8 rank, K9/K14 considerable jobs, K10/K12/K13/K15
// matcher sets, K11/K16 constraint truth tables, K17 init-state, K18 pending-job
// DRU, K19/K20/K22 rebalancer decisions, K21 next-state).  The Fenzo rules (section "FENZO" below) are restated from the
// published Netflix/Fenzo 0.10.0 algorithm; they are pinned by Cook's
// set-level tests only (K10, K12, K13, K15): job->host parity with a real
// Fenzo is UNPINNED (no test in the reference reads hostnames of multi-host
// matches), and the equal-fitness tie-break (lowest hostname) is OURS.
//
// All citations are relative to /root/reference/scheduler/src/cook/.
//
// Build: see oracle/Makefile  (g++ -O2 -shared -fPIC, -ffp-contract=off).

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <map>
#include <queue>
#include <set>
#include <vector>
#include <atomic>
#include <thread>

#include "../include/cook_gpu.h"

static inline void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
  __builtin_ia32_pause();
#endif
}

namespace {

struct Usage {
  double count = 0, cpus = 0, mem = 0, gpus = 0;
};

// tools.clj:876-881 below-quota?: every usage key <= quota key (missing => 0,
// which the host shim materialises as 0.0 in the dense tables).  `gpus` only
// participates when some job contributed a :gpus key (tools.clj:883-889);
// with gpus == 0.0 and quota >= 0 the comparison is vacuous, so the 4-vector
// form is equivalent.
inline bool below_quota(double qc, double qcpu, double qmem, double qgpu, const Usage& u) {
  return u.count <= qc && u.cpus <= qcpu && u.mem <= qmem && u.gpus <= qgpu;
}
inline bool below_quota(const cook_pool_quota* q, const Usage& u) {
  return below_quota(q->count, q->cpus, q->mem, q->gpus, u);
}

// merge-with + : (+ acc x) left fold (dru.clj:43-48, scheduler.clj:2063).
inline void add_usage(Usage& acc, double cpus, double mem, double gpus) {
  acc.count = acc.count + 1.0;
  acc.cpus = acc.cpus + cpus;
  acc.mem = acc.mem + mem;
  acc.gpus = acc.gpus + gpus;
}

struct TaskView {  // running ++ pending, combined index space
  const cook_tasks_soa* r;
  const cook_tasks_soa* p;
  int R, J;
  int user(int i) const { return i < R ? r->user[i] : p->user[i - R]; }
  int prio(int i) const { return i < R ? r->priority[i] : p->priority[i - R]; }
  int64_t start(int i) const { return i < R ? r->start_time[i] : p->start_time[i - R]; }
  int64_t tid(int i) const { return i < R ? r->task_id[i] : p->task_id[i - R]; }
  int64_t jid(int i) const { return i < R ? r->job_id[i] : p->job_id[i - R]; }
  double cpus(int i) const { return i < R ? r->cpus[i] : p->cpus[i - R]; }
  double mem(int i) const { return i < R ? r->mem[i] : p->mem[i - R]; }
  double gpus(int i) const { return i < R ? r->gpus[i] : p->gpus[i - R]; }
};

// tools.clj:614-641: compare of [-priority start-time task-id job-id] vectors.
inline bool task_less(const TaskView& v, int a, int b) {
  int pa = -v.prio(a), pb = -v.prio(b);
  if (pa != pb) return pa < pb;
  if (v.start(a) != v.start(b)) return v.start(a) < v.start(b);
  if (v.tid(a) != v.tid(b)) return v.tid(a) < v.tid(b);
  return v.jid(a) < v.jid(b);
}

int g_naive_merge = 0;

}  // namespace

extern "C" {

// Test knob: 1 => dru.clj:82-104 sorted-merge restated literally (stable
// re-sort of all heads per emitted task, O(N*U log U)); 0 => heap with the
// equivalent key (dru asc, arrival desc, name asc).  tests compare both.
void oracle_set_naive_merge(int on) { g_naive_merge = on; }

const char* oracle_version(void) { return "cook_oracle 1 (CPU restatement; test infrastructure)"; }

// ---------------------------------------------------------------------------
// RANK  (scheduler.clj:2057-2194, dru.clj, tools.clj:614-668, :876-933)
// ---------------------------------------------------------------------------
int32_t oracle_rank(int32_t dru_mode, const cook_tasks_soa* running,
                    const cook_tasks_soa* pending, const cook_user_table* users,
                    const cook_pool_quota* pool_quota, const cook_pool_quota* group_quota,
                    const double* group_usage, const cook_rank_params* params,
                    int32_t* out_ranked_idx, int32_t* out_n, double* out_dru,
                    int32_t* out_order, int32_t* out_order_n) {
  if (!running || !pending || !users || !params || !out_ranked_idx || !out_n) return COOK_E_BADARG;
  TaskView v{running, pending, running->n, pending->n};
  const int R = v.R, J = v.J, N = R + J, U = users->n_users;
  const double NaN = std::numeric_limits<double>::quiet_NaN();

  // scheduler.clj:2080-2083 group-by user, sort with same-user-task-comparator
  std::vector<std::vector<int>> by_user(U);
  for (int i = 0; i < N; i++) {
    int u = v.user(i);
    if (u < 0 || u >= U) return COOK_E_BADARG;
    by_user[u].push_back(i);
  }
  std::vector<double> dru(N, NaN);
  for (int u = 0; u < U; u++) {
    auto& ts = by_user[u];
    std::stable_sort(ts.begin(), ts.end(), [&](int a, int b) { return task_less(v, a, b); });
    // scheduler.clj:2057-2071 limit-over-quota-jobs
    Usage total;
    int over = 0;
    size_t kept = 0;
    for (; kept < ts.size(); kept++) {
      int t = ts[kept];
      add_usage(total, v.cpus(t), v.mem(t), v.gpus(t));
      if (!below_quota(users->quota_count[u], users->quota_cpus[u], users->quota_mem[u],
                       users->quota_gpus[u], total))
        over++;
      if (over > params->max_over_quota_jobs) break;
    }
    ts.resize(kept);
    // dru.clj:50-66 / :68-80 cumulative sums (left fold) then one divide each
    double cm = 0.0, cc = 0.0, cg = 0.0;
    for (int t : ts) {
      cm = cm + v.mem(t);
      cc = cc + v.cpus(t);
      cg = cg + v.gpus(t);
      if (dru_mode == 0) {
        double a = cm / users->div_mem[u], b = cc / users->div_cpus[u];
        dru[t] = a > b ? a : b;  // clojure.core/max
      } else {
        dru[t] = cg / users->div_gpus[u];
      }
    }
  }
  if (out_dru) std::memcpy(out_dru, dru.data(), sizeof(double) * N);

  // dru.clj:82-126: k-way merge by ascending dru.  Users first ordered by name
  // (`(sort-by first)` :123; GPU mode has no such sort in the reference =>
  // hash order, unspecified: we use the same name order).  Each step stable-
  // sorts the remaining per-user seqs by head key and pops the first; the
  // popped user's remainder is consed to the FRONT (:94) => among equal heads
  // the most recently emitted user wins, else earlier relative order.
  std::vector<int> order;
  order.reserve(N);
  std::vector<int> users_by_name(U);
  for (int u = 0; u < U; u++) users_by_name[u] = u;
  std::sort(users_by_name.begin(), users_by_name.end(),
            [&](int a, int b) { return users->name_rank[a] < users->name_rank[b]; });
  if (g_naive_merge) {
    struct Seq { int u; size_t pos; };
    std::vector<Seq> colls;
    for (int u : users_by_name)
      if (!by_user[u].empty()) colls.push_back({u, 0});
    while (!colls.empty()) {
      std::stable_sort(colls.begin(), colls.end(), [&](const Seq& a, const Seq& b) {
        return dru[by_user[a.u][a.pos]] < dru[by_user[b.u][b.pos]];
      });
      Seq s = colls.front();
      order.push_back(by_user[s.u][s.pos]);
      colls.erase(colls.begin());
      if (s.pos + 1 < by_user[s.u].size()) colls.insert(colls.begin(), Seq{s.u, s.pos + 1});
    }
  } else {
    struct Head { double d; int64_t arrival; int nrank; int u; size_t pos; };
    auto cmp = [](const Head& a, const Head& b) {  // "greater" => min-heap
      if (a.d != b.d) return a.d > b.d;
      if (a.arrival != b.arrival) return a.arrival < b.arrival;  // later arrival first
      return a.nrank > b.nrank;
    };
    std::priority_queue<Head, std::vector<Head>, decltype(cmp)> heap(cmp);
    for (int u : users_by_name)
      if (!by_user[u].empty()) heap.push({dru[by_user[u][0]], 0, users->name_rank[u], u, 0});
    int64_t step = 0;
    while (!heap.empty()) {
      Head h = heap.top();
      heap.pop();
      step++;
      order.push_back(by_user[h.u][h.pos]);
      if (h.pos + 1 < by_user[h.u].size())
        heap.push({dru[by_user[h.u][h.pos + 1]], step, h.nrank, h.u, h.pos + 1});
    }
  }
  if (out_order) {
    for (size_t i = 0; i < order.size(); i++) out_order[i] = order[i];
  }
  if (out_order_n) *out_order_n = (int32_t)order.size();

  // scheduler.clj:2089-2090 keep pending only, task -> job
  std::vector<int> queue;
  queue.reserve(J);
  for (int t : order)
    if (t >= R) queue.push_back(t - R);

  // scheduler.clj:2134-2157 filter-based-on-quota -> tools.clj:917-933 with
  // filter-sequential (tools.clj:654-668): state advances for rejected jobs too.
  auto pool_filter = [&](const cook_pool_quota* q, Usage init) {
    if (!q || !q->enabled) return;
    std::vector<int> keep;
    Usage u = init;
    for (int j : queue) {
      add_usage(u, pending->cpus[j], pending->mem[j], pending->gpus[j]);
      if (below_quota(q, u)) keep.push_back(j);
    }
    queue.swap(keep);
  };
  Usage pool_usage;  // scheduler.clj:2118-2123 task-ents->usage of running tasks
  for (int i = 0; i < R; i++) add_usage(pool_usage, running->cpus[i], running->mem[i], running->gpus[i]);
  pool_filter(pool_quota, pool_usage);
  if (group_quota && group_quota->enabled && group_usage) {
    Usage gu;
    gu.count = group_usage[0]; gu.cpus = group_usage[1]; gu.mem = group_usage[2]; gu.gpus = group_usage[3];
    pool_filter(group_quota, gu);
  }
  // scheduler.clj:2198-2229 filter-offensive-jobs
  int n = 0;
  for (int j : queue) {
    if (params->filter_offensive &&
        (pending->mem[j] > params->offensive_max_mem_mb || pending->cpus[j] > params->offensive_max_cpus))
      continue;
    out_ranked_idx[n++] = j;
  }
  *out_n = n;
  return COOK_OK;
}

// ---------------------------------------------------------------------------
// MATCH  (scheduler.clj:617-762, tools.clj:903-973, constraints.clj, FENZO)
// ---------------------------------------------------------------------------
namespace {

struct MatchState {
  const cook_jobs_soa* jobs;
  const cook_offers_soa* of;
  const cook_groups* groups;
  const cook_match_params* prm;
  std::vector<double> asg_cpus, asg_mem;  // Σ assigned this cycle per VM
  std::vector<int> asg_count, ports_used, ports_total;
  // cotasks placed this cycle per group: (hostname id, vm index)
  std::vector<std::vector<int>> group_vms;
};

inline double csr_lookup(const int32_t* off, const int32_t* key, const double* val, int v, int k) {
  if (!off) return 0.0;
  for (int i = off[v]; i < off[v + 1]; i++)
    if (key[i] == k) return val[i];
  return 0.0;
}

// One (job, VM) evaluation = Fenzo AssignableVirtualMachine.tryRequest:
// resource fit, hard constraints, fitness (FENZO rules 3-4).  Returns fitness
// (> 0) or 0.0 on failure; *res_fail set when the failure was a resource.
thread_local int g_first_fail = -1;   // index of the first failing hard constraint of the last eval_pair (explain)
inline double cfail(int i) { g_first_fail = i; return 0.0; }
double eval_pair(const MatchState& s, int j, int v, bool* res_fail) {
  const cook_jobs_soa* jb = s.jobs;
  const cook_offers_soa* of = s.of;
  *res_fail = true;
  // FENZO 3a: used-this-cycle + request > lease total => fail
  if (s.asg_cpus[v] + jb->cpus[j] > of->cpus[v]) return 0.0;
  if (s.asg_mem[v] + jb->mem[j] > of->mem[v]) return 0.0;
  int want_ports = jb->ports ? jb->ports[j] : 0;
  if (want_ports > s.ports_total[v] - s.ports_used[v]) return 0.0;
  *res_fail = false;
  g_first_fail = -1;
  // FENZO 3b hard constraints, Cook's effective order (scheduler.clj:493-501,
  // constraints.clj:487-495): checkpoint-locality, estimated-completion,
  // user-defined, disk, gpu, novel-host, max-tasks-per-host, reservation, groups
  if (jb->ckpt_location && jb->ckpt_location[j] >= 0) {  // constraints.clj:201-240
    int loc = of->location ? of->location[v] : -1;
    if (loc != jb->ckpt_location[j]) return cfail(0);
  }
  if (jb->est_end_ms && jb->est_end_ms[j] >= 0 && of->host_start_time &&
      of->host_start_time[v] >= 0) {  // constraints.clj:385-401
    int64_t death = 1000 * of->host_start_time[v] + (int64_t)60 * 1000 * s.prm->host_lifetime_mins;
    if (!(jb->est_end_ms[j] < death)) return cfail(1);
  }
  if (jb->attr_off) {  // constraints.clj:355-376 user-defined EQUALS
    for (int k = jb->attr_off[j]; k < jb->attr_off[j + 1]; k++) {
      int col = jb->attr_col[k], val = jb->attr_val[k];
      if (col < 0 || col >= of->n_attr_cols) return cfail(2);
      int hv = of->attr[(size_t)col * of->n + v];
      if (val <= 0 || hv != val) return cfail(2);
    }
  }
  bool k8s = of->is_k8s && of->is_k8s[v];
  if (jb->disk_request && jb->disk_request[j] >= 0.0 && k8s) {  // constraints.clj:164-186
    double space = csr_lookup(of->disk_off, of->disk_type, of->disk_space, v,
                              jb->disk_type ? jb->disk_type[j] : -1);
    if (!(space >= jb->disk_request[j])) return cfail(3);
  }
  {  // constraints.clj:122-157 gpu-host-constraint (always built)
    double g = jb->gpus ? jb->gpus[j] : 0.0;
    if (k8s) {
      if (g > 0.0) {
        double have = csr_lookup(of->gpu_off, of->gpu_model, of->gpu_count, v,
                                 jb->gpu_model ? jb->gpu_model[j] : -1);
        int on_vm = (of->run_count ? of->run_count[v] : 0) + s.asg_count[v];
        if (!(have == g && on_vm == 0)) return cfail(4);
      } else {
        int nmodels = of->gpu_off ? of->gpu_off[v + 1] - of->gpu_off[v] : 0;
        if (nmodels != 0) return cfail(4);
      }
    } else if (!(g == 0.0)) {
      return cfail(4);
    }
  }
  if (jb->novel_off) {  // constraints.clj:68-94
    for (int k = jb->novel_off[j]; k < jb->novel_off[j + 1]; k++)
      if (jb->novel_host[k] == of->hostname_id[v]) return cfail(5);
  }
  if (of->max_tasks && of->max_tasks[v] >= 0) {  // constraints.clj:433-456
    int total = (of->num_tasks ? of->num_tasks[v] : 0) + s.asg_count[v];
    if (!(total < of->max_tasks[v])) return cfail(6);
  }
  if (of->reserved && of->reserved[v]) {  // constraints.clj:242-252, scheduler.clj:645-653
    int mine = jb->reserved_host ? jb->reserved_host[j] : -1;
    if (mine != of->hostname_id[v]) return cfail(7);
  }
  if (jb->group_off && s.groups) {  // constraints.clj:586-678
    const cook_groups* gr = s.groups;
    for (int k = jb->group_off[j]; k < jb->group_off[j + 1]; k++) {
      int g = jb->group_idx[k];
      int kind = gr->kind[g];
      const std::vector<int>& placed = s.group_vms[g];
      if (kind == COOK_GROUP_UNIQUE) {
        int h = of->hostname_id[v];
        for (int c = gr->cot_off[g]; c < gr->cot_off[g + 1]; c++)
          if (gr->cot_hostname_id[c] == h) return cfail(8);
        for (int pv : placed)
          if (of->hostname_id[pv] == h) return cfail(8);
      } else {
        int col = gr->attr_col[g];
        auto vm_attr = [&](int vm) { return (col >= 0 && col < of->n_attr_cols) ? of->attr[(size_t)col * of->n + vm] : 0; };
        int target = vm_attr(v);
        std::map<int, int> freq;  // value id (0 = nil) -> count
        for (int c = gr->cot_off[g]; c < gr->cot_off[g + 1]; c++) freq[gr->cot_attr_val[c]]++;
        for (int pv : placed) freq[vm_attr(pv)]++;
        if (kind == COOK_GROUP_BALANCED) {
          if (!freq.empty()) {
            auto it = freq.find(target);
            if (it != freq.end()) {
              int mn = std::numeric_limits<int>::max(), mx = 0;
              for (auto& kv : freq) { mn = std::min(mn, kv.second); mx = std::max(mx, kv.second); }
              if (gr->minimum[g] > (int)freq.size()) mn = 0;
              if (!(mn == mx || it->second < mx)) return cfail(9);
            }
          }
        } else {  // attribute-equals
          if (!freq.empty() && freq.find(target) == freq.end()) return cfail(10);
        }
      }
    }
  }
  // FENZO 4: cpuMemBinPacker = (cpuFit + memFit) / 2,
  // xFit = (req + Σassigned-this-cycle + Σrunning) / (leaseTotal + Σrunning)
  // ASSOCIATION: Fenzo's calculateResourceFitness folds req + a1 + a2 + ... one previous assignment at a time;
  // here (and in the CUDA path) Σassigned-this-cycle is kept as a running sum: (req + Σassigned) + Σrunning.
  // Identical on the binary grid the ABI asks for (include/cook_gpu.h: amounts are multiples of 2^-10 with
  // exact sums), possibly one ulp apart otherwise - with Fenzo absent from /root/reference that case cannot
  // be pinned either way (header: job -> host against a real Fenzo is unpinned).
  double rc = of->run_cpus ? of->run_cpus[v] : 0.0, rm = of->run_mem ? of->run_mem[v] : 0.0;
  double cpu_fit = ((jb->cpus[j] + s.asg_cpus[v]) + rc) / (of->cpus[v] + rc);
  double mem_fit = ((jb->mem[j] + s.asg_mem[v]) + rm) / (of->mem[v] + rm);
  return (cpu_fit + mem_fit) / 2.0;
}

}  // namespace

// M0: pending-jobs->considerable-jobs (scheduler.clj:729-762) =
// filter-based-on-user-quota (tools.clj:903-915) -> ratelimit (:940-959) ->
// filter-based-on-pool-quota (:917-933) -> allowed -> launch plugin -> take N.
int32_t oracle_considerable(const int32_t* ranked_idx, int32_t n_ranked,
                            const cook_jobs_soa* jobs, const cook_user_table* users,
                            const cook_pool_quota* pool_quota,
                            const cook_match_params* params, int32_t* out_considerable,
                            int32_t* out_n) {
  const int U = users->n_users;
  std::vector<Usage> usage(U);
  Usage pool_usage;  // tools.clj:969 (reduce (partial merge-with +) (vals user->usage))
  for (int u = 0; u < U; u++) {
    if (users->usage_count) {
      usage[u].count = users->usage_count[u]; usage[u].cpus = users->usage_cpus[u];
      usage[u].mem = users->usage_mem[u]; usage[u].gpus = users->usage_gpus[u];
    }
    pool_usage.count = pool_usage.count + usage[u].count;
    pool_usage.cpus = pool_usage.cpus + usage[u].cpus;
    pool_usage.mem = pool_usage.mem + usage[u].mem;
    pool_usage.gpus = pool_usage.gpus + usage[u].gpus;
  }
  std::vector<int> seen(U, 0);
  int n = 0;
  for (int i = 0; i < n_ranked && n < params->num_considerable; i++) {
    int j = ranked_idx[i];
    if (j < 0 || j >= jobs->n) return COOK_E_BADARG;
    int u = jobs->user[j];
    double g = jobs->gpus ? jobs->gpus[j] : 0.0;
    // user quota: state advances whether or not the job is kept
    add_usage(usage[u], jobs->cpus[j], jobs->mem[j], g);
    if (!below_quota(users->quota_count[u], users->quota_cpus[u], users->quota_mem[u],
                     users->quota_gpus[u], usage[u]))
      continue;
    // launch-rate limit: k-th surviving job of the user passes iff k <= tokens
    seen[u]++;
    bool limited = users->tokens ? (seen[u] > users->tokens[u]) : false;
    if (limited && params->enforce_rate_limit) continue;
    // pool quota over survivors
    if (pool_quota && pool_quota->enabled) {
      add_usage(pool_usage, jobs->cpus[j], jobs->mem[j], g);
      if (!below_quota(pool_quota, pool_usage)) continue;
    }
    if (jobs->allowed && !jobs->allowed[j]) continue;
    if (jobs->plugin_accept && !jobs->plugin_accept[j]) continue;
    out_considerable[n++] = j;
  }
  *out_n = n;
  return COOK_OK;
}

// ---------------------------------------------------------------------------
// FENZO restatement (com.netflix.fenzo/fenzo-core 0.10.0, project.clj:50; not
// vendored in /root/reference).  Rules (SURVEY.md §8c):
//  F1 every hostname with a live lease is one assignable VM; available = Σ leases.
//  F3 for each request IN LIST ORDER every VM is tried: resource fit against
//     (available - assigned this cycle), then hard constraints, then fitness;
//     fitness == 0.0 is a failure.
//  F4 cpuMemBinPacker (config.clj:108).
//  F5 good-enough-fitness >= 1.0 (zz_simulator.clj:84) => all VMs evaluated,
//     winner = max fitness; equal fitness => LOWEST hostname (OUR fixed
//     tie-break; Fenzo's is hash-order, unspecified).
//  F6 on success the VM's assigned cpus/mem/ports/count advance; ports are the
//     first n free ports scanning ranges in lease order.
// ---------------------------------------------------------------------------
struct ExplainReq { const int32_t* k_idx; int32_t n; cook_failure_counts* out; };
static thread_local const ExplainReq* g_explain = nullptr;

static int32_t oracle_match_impl(const int32_t* ranked_idx, int32_t n_ranked, const cook_jobs_soa* jobs,
                     const cook_offers_soa* offers, const cook_groups* groups,
                     const cook_user_table* users, const cook_pool_quota* pool_quota,
                     const cook_match_params* params, int32_t* out_considerable,
                     int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                     uint8_t* out_fail_reason, cook_match_stats* st, int n_threads) {
  if (!ranked_idx || !jobs || !offers || !users || !params || !out_considerable || !out_assign)
    return COOK_E_BADARG;
  if (params->good_enough_fitness < 1.0) return COOK_E_BADARG;
  if (params->fitness_kind != 0) return COOK_E_UNSUPPORTED_CONSTRAINT;
  int32_t nc = 0;
  int32_t rc = oracle_considerable(ranked_idx, n_ranked, jobs, users, pool_quota, params,
                                   out_considerable, &nc);
  if (rc != COOK_OK) return rc;
  const int O = offers->n;
  MatchState s;
  s.jobs = jobs; s.of = offers; s.groups = groups; s.prm = params;
  s.asg_cpus.assign(O, 0.0); s.asg_mem.assign(O, 0.0);
  s.asg_count.assign(O, 0); s.ports_used.assign(O, 0); s.ports_total.assign(O, 0);
  if (offers->port_off)
    for (int v = 0; v < O; v++)
      for (int k = offers->port_off[v]; k < offers->port_off[v + 1]; k++)
        s.ports_total[v] += offers->port_end[k] - offers->port_begin[k] + 1;
  if (groups) s.group_vms.resize(groups->n_groups);
  int n_matched = 0;
  // The per-task VM loop is the only thing Fenzo itself runs on a thread pool;
  // n_threads > 1 splits exactly that loop (used by bench.py --impl reference).
  struct Partial { int best; double fit; bool res_ok; char pad[64]; };
  auto scan = [&](int j, int v0, int v1, Partial& out) {
    int best = -1; double best_fit = 0.0; bool any_res_ok = false;
    for (int v = v0; v < v1; v++) {
      bool res_fail;
      double f = eval_pair(s, j, v, &res_fail);
      if (!res_fail) any_res_ok = true;
      if (f == 0.0) continue;  // FENZO 3c
      if (best < 0 || f > best_fit ||
          (f == best_fit && offers->name_rank[v] < offers->name_rank[best])) {
        best = v; best_fit = f;
      }
    }
    out.best = best; out.fit = best_fit; out.res_ok = any_res_ok;
  };
  const int T = std::max(1, std::min(n_threads, 64));
  std::vector<Partial> parts(T);
  // one cache line per flag: the workers spin on `gen` while the finished ones bump `done`
  struct alignas(64) Flag { std::atomic<int> v{0}; };
  Flag gen_f, done_f, job_f, stop_f;
  std::atomic<int>&gen = gen_f.v, &done = done_f.v, &cur_job = job_f.v, &stop = stop_f.v;
  std::vector<std::thread> workers;
  for (int t = 1; t < T; t++)
    workers.emplace_back([&, t]() {
      int seen = 0;
      while (true) {
        while (gen.load(std::memory_order_acquire) == seen) {
          if (stop.load(std::memory_order_relaxed)) return;
          cpu_relax();
        }
        seen++;
        int j = cur_job.load(std::memory_order_relaxed);
        scan(j, (int)((long long)O * t / T), (int)((long long)O * (t + 1) / T), parts[t]);
        done.fetch_add(1, std::memory_order_release);
      }
    });
  if (g_explain)
    for (int q = 0; q < g_explain->n; q++) {
      std::memset(&g_explain->out[q], 0, sizeof(cook_failure_counts));
      g_explain->out[q].n_vms = (g_explain->k_idx[q] >= 0 && g_explain->k_idx[q] < nc) ? O : -1;
    }
  for (int k = 0; k < nc; k++) {
    int j = out_considerable[k];
    if (g_explain)   // fenzo_utils.clj:45-57: per VM, every short resource, else the first failing constraint
      for (int q = 0; q < g_explain->n; q++) {
        if (g_explain->k_idx[q] != k) continue;
        cook_failure_counts& c = g_explain->out[q];
        for (int v = 0; v < O; v++) {
          const bool no_c = s.asg_cpus[v] + jobs->cpus[j] > offers->cpus[v];
          const bool no_m = s.asg_mem[v] + jobs->mem[j] > offers->mem[v];
          const bool no_p = (jobs->ports ? jobs->ports[j] : 0) > s.ports_total[v] - s.ports_used[v];
          if (no_c) c.counts[COOK_FAILC_CPUS]++;
          if (no_m) c.counts[COOK_FAILC_MEM]++;
          if (no_p) c.n_ports++;
          if (no_c || no_m || no_p) continue;
          bool rf;
          const double f = eval_pair(s, j, v, &rf);
          if (f == 0.0 && g_first_fail >= 0) c.counts[COOK_FAILC_FIRST_CONSTRAINT + g_first_fail]++;
          else c.n_passed++;
        }
      }
    if (T > 1) {
      done.store(0, std::memory_order_relaxed);
      cur_job.store(j, std::memory_order_relaxed);
      gen.fetch_add(1, std::memory_order_release);
    }
    scan(j, 0, (int)((long long)O * 1 / T), parts[0]);
    if (T > 1)
      while (done.load(std::memory_order_acquire) != T - 1) cpu_relax();
    int best = -1;
    double best_fit = 0.0;
    bool any_res_ok = false;
    for (int t = 0; t < T; t++) {
      any_res_ok = any_res_ok || parts[t].res_ok;
      int v = parts[t].best;
      if (v < 0) continue;
      if (best < 0 || parts[t].fit > best_fit ||
          (parts[t].fit == best_fit && offers->name_rank[v] < offers->name_rank[best])) {
        best = v; best_fit = parts[t].fit;
      }
    }
    out_assign[k] = best;
    if (out_fail_reason)
      out_fail_reason[k] = best >= 0 ? COOK_FAIL_NONE
                           : (O == 0 ? COOK_FAIL_NO_OFFERS
                                     : (any_res_ok ? COOK_FAIL_CONSTRAINT : COOK_FAIL_RESOURCES));
    if (best >= 0) {
      n_matched++;
      s.asg_cpus[best] = s.asg_cpus[best] + jobs->cpus[j];
      s.asg_mem[best] = s.asg_mem[best] + jobs->mem[j];
      s.asg_count[best]++;
      int want = jobs->ports ? jobs->ports[j] : 0;
      if (out_ports && max_ports > 0)
        for (int p = 0; p < max_ports; p++) out_ports[(size_t)k * max_ports + p] = -1;
      if (want > 0) {  // FENZO F6
        int skip = s.ports_used[best], got = 0;
        for (int r = offers->port_off[best]; r < offers->port_off[best + 1] && got < want; r++) {
          int len = offers->port_end[r] - offers->port_begin[r] + 1;
          if (skip >= len) { skip -= len; continue; }
          for (int p = offers->port_begin[r] + skip; p <= offers->port_end[r] && got < want; p++) {
            if (out_ports && got < max_ports) out_ports[(size_t)k * max_ports + got] = p;
            got++;
          }
          skip = 0;
        }
        s.ports_used[best] += want;
      }
      if (jobs->group_off && groups)
        for (int g = jobs->group_off[j]; g < jobs->group_off[j + 1]; g++)
          s.group_vms[jobs->group_idx[g]].push_back(best);
    } else if (out_ports && max_ports > 0) {
      for (int p = 0; p < max_ports; p++) out_ports[(size_t)k * max_ports + p] = -1;
    }
  }
  stop.store(1);
  for (auto& w : workers) w.join();
  if (st) {
    std::memset(st, 0, sizeof(*st));
    st->n_considerable = nc;
    st->n_matched = n_matched;
    st->head_matched = (nc > 0 && out_assign[0] >= 0) ? 1 : 0;
    int used = 0;
    for (int v = 0; v < O; v++) used += s.asg_count[v] > 0;
    st->n_offers_used = used;
    st->evals = (int64_t)nc * O;
  }
  return COOK_OK;
}

int32_t oracle_match(const int32_t* ranked_idx, int32_t n_ranked, const cook_jobs_soa* jobs,
                     const cook_offers_soa* offers, const cook_groups* groups,
                     const cook_user_table* users, const cook_pool_quota* pool_quota,
                     const cook_match_params* params, int32_t* out_considerable,
                     int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                     uint8_t* out_fail_reason, cook_match_stats* st) {
  return oracle_match_impl(ranked_idx, n_ranked, jobs, offers, groups, users, pool_quota, params,
                           out_considerable, out_assign, out_ports, max_ports, out_fail_reason, st, 1);
}

// TEST TWIN of cook_match_failures: the same match, counting at the requested jobs' turns.
int32_t oracle_match_failures(const int32_t* ranked_idx, int32_t n_ranked, const cook_jobs_soa* jobs,
                              const cook_offers_soa* offers, const cook_groups* groups,
                              const cook_user_table* users, const cook_pool_quota* pool_quota,
                              const cook_match_params* params, const int32_t* k_idx, int32_t n,
                              cook_failure_counts* out) {
  std::vector<int32_t> cons(std::max(1, params->num_considerable)), asg(std::max(1, params->num_considerable));
  ExplainReq req{k_idx, n, out};
  g_explain = &req;
  int32_t rc = oracle_match_impl(ranked_idx, n_ranked, jobs, offers, groups, users, pool_quota, params, cons.data(),
                                 asg.data(), nullptr, 0, nullptr, nullptr, 1);
  g_explain = nullptr;
  return rc;
}

int32_t oracle_match_mt(const int32_t* ranked_idx, int32_t n_ranked, const cook_jobs_soa* jobs,
                        const cook_offers_soa* offers, const cook_groups* groups,
                        const cook_user_table* users, const cook_pool_quota* pool_quota,
                        const cook_match_params* params, int32_t* out_considerable,
                        int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                        uint8_t* out_fail_reason, cook_match_stats* st, int32_t n_threads) {
  return oracle_match_impl(ranked_idx, n_ranked, jobs, offers, groups, users, pool_quota, params,
                           out_considerable, out_assign, out_ports, max_ports, out_fail_reason, st,
                           n_threads);
}

}  // extern "C"

// ---------------------------------------------------------------------------
// REBALANCE  (rebalancer.clj:144-467, dru.clj:128-144, constraints.clj:504-515,
// :680-697).  Default DRU mode only: in GPU mode the reference's
// compute-preemption-decision dereferences (:dru <number>) = nil and throws
// (rebalancer.clj:339-349 over the [task cumulative-gpus] pairs of :245-247),
// so there is no reference behaviour to restate.
// ---------------------------------------------------------------------------
namespace {

struct RTask {
  int user, prio, host;
  int64_t start, tid, jid;
  double cpus, mem, gpus, dru;
  bool alive;
};

struct RebState {
  std::vector<RTask> tasks;                 // running, then synthetic tasks of decisions
  std::vector<std::vector<int>> by_user;    // sorted (tools.clj:614-641)
  std::vector<uint8_t> has_spare;
  std::vector<double> spare_cpus, spare_mem, spare_gpus;
  std::vector<int> preempted_hosts;         // hosts of tasks preempted so far (constraints.clj:690-692)
};

inline bool rtask_less(const RTask& a, const RTask& b) {
  if (-a.prio != -b.prio) return -a.prio < -b.prio;
  if (a.start != b.start) return a.start < b.start;
  if (a.tid != b.tid) return a.tid < b.tid;
  return a.jid < b.jid;
}

// dru.clj:50-66 for one user (next-task->scored-task re-scores changed users)
void rescore_user(RebState& st, const cook_user_table* users, int u) {
  double cm = 0.0, cc = 0.0;
  for (int t : st.by_user[u]) {
    cm = cm + st.tasks[t].mem;
    cc = cc + st.tasks[t].cpus;
    double a = cm / users->div_mem[u], b = cc / users->div_cpus[u];
    st.tasks[t].dru = a > b ? a : b;
  }
}

// The six job-constraint-constructors evaluated on the cached agent attributes
// of `h` (constraints.clj:504-515); `have_attrs` is false when the host has no
// task in task->scored-task (preemptable-host->slave-id lookup yields nil,
// rebalancer.clj:371-377), i.e. every attribute reads as nil.
bool reb_host_passes(const cook_jobs_soa* jb, int j, const cook_host_table* ht, int h, bool have_attrs,
                     const cook_rebalance_params* prm) {
  // novel-host: (get nil "HOSTNAME") => nil => passes
  if (have_attrs && jb->novel_off)
    for (int k = jb->novel_off[j]; k < jb->novel_off[j + 1]; k++)
      if (jb->novel_host[k] == ht->hostname_id[h]) return false;
  bool k8s = have_attrs && ht->is_k8s && ht->is_k8s[h];
  double g = jb->gpus ? jb->gpus[j] : 0.0;
  if (k8s) {  // gpu-host 3-arity: vm-tasks-assigned = []
    if (g > 0.0) {
      double have = csr_lookup(ht->gpu_off, ht->gpu_model, ht->gpu_count, h, jb->gpu_model ? jb->gpu_model[j] : -1);
      if (!(have == g)) return false;
    } else {
      int nm = ht->gpu_off ? ht->gpu_off[h + 1] - ht->gpu_off[h] : 0;
      if (nm != 0) return false;
    }
  } else if (!(g == 0.0)) {
    return false;
  }
  if (jb->disk_request && jb->disk_request[j] >= 0.0 && k8s) {
    double space = csr_lookup(ht->disk_off, ht->disk_type, ht->disk_space, h, jb->disk_type ? jb->disk_type[j] : -1);
    if (!(space >= jb->disk_request[j])) return false;
  }
  if (jb->attr_off)
    for (int k = jb->attr_off[j]; k < jb->attr_off[j + 1]; k++) {
      int col = jb->attr_col[k], val = jb->attr_val[k];
      if (!have_attrs || col < 0 || col >= ht->n_attr_cols) return false;
      int hv = ht->attr[(size_t)col * ht->n + h];
      if (val <= 0 || hv != val) return false;
    }
  if (jb->est_end_ms && jb->est_end_ms[j] >= 0 && have_attrs && ht->host_start_time && ht->host_start_time[h] >= 0) {
    int64_t death = 1000 * ht->host_start_time[h] + (int64_t)60 * 1000 * prm->host_lifetime_mins;
    if (!(jb->est_end_ms[j] < death)) return false;
  }
  if (jb->ckpt_location && jb->ckpt_location[j] >= 0) {
    int loc = (have_attrs && ht->location) ? ht->location[h] : -1;
    if (loc != jb->ckpt_location[j]) return false;
  }
  return true;
}

}  // namespace

// Test-only view into the rebalancer state, for the reference tests that read
// it directly: compute-pending-default-job-dru (K18, test/cook/test/rebalancer.clj:115-157)
// and next-state (K21, :813-988).  With n_forced > 0 the decision search is
// skipped and the given decisions are applied with next-state (:270-309), as
// the reference test does.
struct oracle_reb_trace {
  int32_t n_forced;
  const cook_decision* forced;     // pending_idx, host, victim slice, mem/cpus/gpus
  const int32_t* forced_victims;
  double* pending_dru;             // [pending->n], NaN for jobs the walk did not reach
  double* task_dru;                // [R + max_preemption] after the last transition
  uint8_t* task_alive;             // same length
  int32_t* order;                  // task->scored-task key order (priority map) afterwards
  int32_t* n_order;
  uint8_t* has_spare;              // [H] host->spare-resources afterwards
  double *spare_mem, *spare_cpus, *spare_gpus;
  int32_t forced_only;             // 1: walk only the forced jobs (K21); 0: the forced jobs take their
                                   // given decision, every other pending job is searched as usual (K20:
                                   // "one host has already been preempted this cycle")
  uint8_t* below_quota;            // [pending->n] job-below-quota (:210-220) for the jobs the walk reached
};

static int32_t rebalance_impl(int32_t dru_mode, const cook_running_soa* running,
                                    const cook_jobs_soa* pending, const int64_t* pending_job_id,
                                    const int32_t* pending_priority, const cook_host_table* hosts,
                                    const cook_groups* groups, const cook_user_table* users,
                                    const cook_rebalance_params* prm, cook_decision* out_dec,
                                    int32_t* out_victims, int32_t* out_n, const oracle_reb_trace* tr) {
  if (!running || !pending || !hosts || !users || !prm || !out_dec || !out_victims || !out_n) return COOK_E_BADARG;
  if (dru_mode != 0) return COOK_E_UNSUPPORTED_CONSTRAINT;
  const int R = running->t.n, H = hosts->n, U = users->n_users;
  RebState st;
  st.tasks.resize(R);
  st.by_user.resize(U);
  for (int i = 0; i < R; i++) {
    const cook_tasks_soa& t = running->t;
    st.tasks[i] = RTask{t.user[i], t.priority[i], running->host[i], t.start_time[i], t.task_id[i], t.job_id[i],
                        t.cpus[i], t.mem[i], t.gpus ? t.gpus[i] : 0.0, 0.0, true};
    st.by_user[t.user[i]].push_back(i);
  }
  for (int u = 0; u < U; u++) {  // rebalancer.clj:237-243 sorted-set-by same-user-task-comparator
    std::stable_sort(st.by_user[u].begin(), st.by_user[u].end(),
                     [&](int a, int b) { return rtask_less(st.tasks[a], st.tasks[b]); });
    rescore_user(st, users, u);
  }
  st.has_spare.assign(H, 0); st.spare_cpus.assign(H, 0.0); st.spare_mem.assign(H, 0.0); st.spare_gpus.assign(H, 0.0);
  for (int h = 0; h < H; h++)
    if (hosts->has_spare && hosts->has_spare[h]) {
      st.has_spare[h] = 1; st.spare_cpus[h] = hosts->spare_cpus[h]; st.spare_mem[h] = hosts->spare_mem[h];
      st.spare_gpus[h] = hosts->spare_gpus ? hosts->spare_gpus[h] : 0.0;
    }
  std::vector<int> hosts_by_name(H);  // (sort-by first) rebalancer.clj:383
  for (int h = 0; h < H; h++) hosts_by_name[h] = h;
  std::sort(hosts_by_name.begin(), hosts_by_name.end(),
            [&](int a, int b) { return hosts->name_rank[a] < hosts->name_rank[b]; });
  const double DMAX = std::numeric_limits<double>::max();
  int n_dec = 0, n_vict = 0;
  // rebalancer.clj:442-458: walk the pending jobs while preemptions remain
  if (tr && tr->pending_dru)
    for (int p = 0; p < pending->n; p++) tr->pending_dru[p] = std::numeric_limits<double>::quiet_NaN();
  const bool any_forced = tr && tr->n_forced > 0;
  const bool forced_only = any_forced && tr->forced_only != 0;
  const int n_walk = forced_only ? tr->n_forced : pending->n;
  for (int w = 0; w < n_walk && n_dec < prm->max_preemption; w++) {
    const int p = forced_only ? tr->forced[w].pending_idx : w;
    const cook_decision* fdec = nullptr;
    if (any_forced)
      for (int q = 0; q < tr->n_forced; q++)
        if (tr->forced[q].pending_idx == p) fdec = &tr->forced[q];
    const bool forced = fdec != nullptr;
    const int pu = pending->user[p];
    const double pmem = pending->mem[p], pcpus = pending->cpus[p], pgpus = pending->gpus ? pending->gpus[p] : 0.0;
    // job-below-quota :210-220
    Usage fu;
    add_usage(fu, pcpus, pmem, pgpus);
    for (int t : st.by_user[pu]) add_usage(fu, st.tasks[t].cpus, st.tasks[t].mem, st.tasks[t].gpus);
    const bool below = below_quota(users->quota_count[pu], users->quota_cpus[pu], users->quota_mem[pu],
                                   users->quota_gpus[pu], fu);
    if (tr && tr->below_quota) tr->below_quota[p] = below ? 1 : 0;
    // compute-pending-default-job-dru :182-208: nearest = last task <= synthetic pending task
    RTask synth{pu, pending_priority[p], -1, std::numeric_limits<int64_t>::max(), -1, pending_job_id[p],
                pcpus, pmem, pgpus, 0.0, true};
    double nearest = 0.0;
    for (int t : st.by_user[pu]) {
      if (rtask_less(synth, st.tasks[t])) break;  // t > synth
      nearest = st.tasks[t].dru;
    }
    const double pd_mem = nearest + pmem / users->div_mem[pu], pd_cpu = nearest + pcpus / users->div_cpus[pu];
    const double pending_dru = pd_mem > pd_cpu ? pd_mem : pd_cpu;
    if (tr && tr->pending_dru) tr->pending_dru[p] = pending_dru;
    // victims in priority-map order: (-dru, user) ascending (:252-256); equal
    // (dru, user) is unordered in the reference => OURS: later same-user position first
    std::vector<int> order;
    for (size_t t = 0; t < st.tasks.size(); t++)
      if (st.tasks[t].alive) order.push_back((int)t);
    std::vector<int> pos_in_user(st.tasks.size(), 0);
    for (int u = 0; u < U; u++)
      for (size_t i = 0; i < st.by_user[u].size(); i++) pos_in_user[st.by_user[u][i]] = (int)i;
    std::sort(order.begin(), order.end(), [&](int a, int b) {
      const RTask &x = st.tasks[a], &y = st.tasks[b];
      if (x.dru != y.dru) return x.dru > y.dru;
      if (x.user != y.user) return users->name_rank[x.user] < users->name_rank[y.user];
      return pos_in_user[a] > pos_in_user[b];
    });
    std::vector<std::vector<int>> host_victims(H);
    std::vector<uint8_t> host_has_task(H, 0);
    for (int t : order) {
      const RTask& x = st.tasks[t];
      host_has_task[x.host] = 1;
      if (!(below || x.user == pu)) continue;
      if (x.dru < prm->safe_dru_threshold) continue;
      if (!((x.dru - pending_dru) > prm->min_dru_diff)) continue;
      host_victims[x.host].push_back(t);
    }
    // group cohosts: running cotasks + hosts of everything preempted so far
    auto group_ok = [&](int h, bool have_attrs) {
      if (!pending->group_off || !groups) return true;
      for (int k = pending->group_off[p]; k < pending->group_off[p + 1]; k++) {
        int g = pending->group_idx[k];
        int kind = groups->kind[g];
        int col = groups->attr_col ? groups->attr_col[g] : -1;
        auto host_attr = [&](int hh) { return (col >= 0 && col < hosts->n_attr_cols) ? hosts->attr[(size_t)col * H + hh] : 0; };
        if (kind == COOK_GROUP_UNIQUE) {
          if (!have_attrs) return false;  // (and target-hostname ...) with nil hostname
          int hn = hosts->hostname_id[h];
          for (int ph : st.preempted_hosts) if (hosts->hostname_id[ph] == hn) return false;
          for (int c = groups->cot_off[g]; c < groups->cot_off[g + 1]; c++)
            if (groups->cot_hostname_id[c] == hn) return false;
        } else {
          std::map<int, int> freq;
          for (int ph : st.preempted_hosts) freq[host_attr(ph)]++;
          for (int c = groups->cot_off[g]; c < groups->cot_off[g + 1]; c++) freq[groups->cot_attr_val[c]]++;
          int target = have_attrs ? host_attr(h) : 0;
          if (freq.empty()) continue;
          auto it = freq.find(target);
          if (kind == COOK_GROUP_ATTR_EQUALS) { if (it == freq.end()) return false; }
          else if (it != freq.end()) {
            int mn = std::numeric_limits<int>::max(), mx = 0;
            for (auto& kv : freq) { mn = std::min(mn, kv.second); mx = std::max(mx, kv.second); }
            if (groups->minimum[g] > (int)freq.size()) mn = 0;
            if (!(mn == mx || it->second < mx)) return false;
          }
        }
      }
      return true;
    };
    // :380-404 per host (name order): [spare ; victims desc dru], prefix sums,
    // keep sufficient prefixes, max-key :dru with ties -> LAST
    bool found = false;
    double best_dru = 0.0, best_mem = 0, best_cpus = 0, best_gpus = 0;  // (fnil :dru {:dru 0.0}) nil
    int best_host = -1;
    std::vector<int> best_tasks;
    for (int h : hosts_by_name) {
      if (!st.has_spare[h] && host_victims[h].empty()) continue;
      const bool have_attrs = host_has_task[h];
      if (!reb_host_passes(pending, p, hosts, h, have_attrs, prm)) continue;
      if (!group_ok(h, have_attrs)) continue;
      double sm = 0.0, sc = 0.0, sg = 0.0;
      std::vector<int> prefix;
      auto consider = [&](double dru) {
        if (sm >= pmem && sc >= pcpus && (pgpus > 0.0 ? sg >= pgpus : true)) {
          if (dru >= best_dru) {  // max-key: >= keeps the LAST of equal keys; nil counts as 0.0
            found = true; best_dru = dru; best_host = h; best_tasks = prefix;
            best_mem = sm; best_cpus = sc; best_gpus = sg;
          }
        }
      };
      if (st.has_spare[h]) {
        sg = sg + st.spare_gpus[h]; sm = sm + st.spare_mem[h]; sc = sc + st.spare_cpus[h];
        consider(DMAX);
      }
      for (int t : host_victims[h]) {
        sg = sg + st.tasks[t].gpus; sm = sm + st.tasks[t].mem; sc = sc + st.tasks[t].cpus;
        prefix.push_back(t);
        consider(st.tasks[t].dru);
      }
    }
    if (forced) {  // the test hands next-state its decision (:906, :931, :951)
      const cook_decision& f = *fdec;
      found = true; best_host = f.host; best_dru = f.dru; best_mem = f.mem; best_cpus = f.cpus; best_gpus = f.gpus;
      best_tasks.assign(tr->forced_victims + f.victim_begin, tr->forced_victims + f.victim_begin + f.victim_count);
    }
    if (!found) continue;
    // ---- next-state :270-309
    cook_decision& d = out_dec[n_dec];
    d.pending_idx = p; d.host = best_host; d.dru = best_dru; d.mem = best_mem; d.cpus = best_cpus; d.gpus = best_gpus;
    d.victim_begin = n_vict; d.victim_count = (int)best_tasks.size();
    for (int i = (int)best_tasks.size() - 1; i >= 0; i--) out_victims[n_vict++] = best_tasks[i];  // conj onto list => ascending dru
    std::set<int> changed;
    changed.insert(pu);
    for (int t : best_tasks) {
      RTask& x = st.tasks[t];
      x.alive = false;
      auto& lst = st.by_user[x.user];
      lst.erase(std::find(lst.begin(), lst.end(), t));
      changed.insert(x.user);
      st.preempted_hosts.push_back(x.host);
    }
    RTask nt = synth;
    nt.host = best_host;
    st.tasks.push_back(nt);
    const int nti = (int)st.tasks.size() - 1;
    auto& lst = st.by_user[pu];
    lst.insert(std::upper_bound(lst.begin(), lst.end(), nti,
                                [&](int a, int b) { return rtask_less(st.tasks[a], st.tasks[b]); }), nti);
    for (int u : changed) rescore_user(st, users, u);
    st.has_spare[best_host] = 1;
    st.spare_mem[best_host] = best_mem - pmem;
    st.spare_gpus[best_host] = best_gpus - pgpus;
    st.spare_cpus[best_host] = best_cpus - pcpus;
    n_dec++;
  }
  *out_n = n_dec;
  if (tr) {
    const int nt = (int)st.tasks.size();
    std::vector<int> pos_in_user(nt, 0);
    for (int u = 0; u < U; u++)
      for (size_t i = 0; i < st.by_user[u].size(); i++) pos_in_user[st.by_user[u][i]] = (int)i;
    std::vector<int> order;
    for (int t = 0; t < nt; t++) {
      if (tr->task_dru) tr->task_dru[t] = st.tasks[t].dru;
      if (tr->task_alive) tr->task_alive[t] = st.tasks[t].alive;
      if (st.tasks[t].alive) order.push_back(t);
    }
    std::sort(order.begin(), order.end(), [&](int a, int b) {  // same rule as the victim order above
      const RTask &x = st.tasks[a], &y = st.tasks[b];
      if (x.dru != y.dru) return x.dru > y.dru;
      if (x.user != y.user) return users->name_rank[x.user] < users->name_rank[y.user];
      return pos_in_user[a] > pos_in_user[b];
    });
    if (tr->order) for (size_t i = 0; i < order.size(); i++) tr->order[i] = order[i];
    if (tr->n_order) *tr->n_order = (int)order.size();
    for (int h = 0; h < H; h++) {
      if (tr->has_spare) tr->has_spare[h] = st.has_spare[h];
      if (tr->spare_mem) tr->spare_mem[h] = st.spare_mem[h];
      if (tr->spare_cpus) tr->spare_cpus[h] = st.spare_cpus[h];
      if (tr->spare_gpus) tr->spare_gpus[h] = st.spare_gpus[h];
    }
  }
  return COOK_OK;
}

extern "C" int32_t oracle_rebalance(int32_t dru_mode, const cook_running_soa* running,
                                    const cook_jobs_soa* pending, const int64_t* pending_job_id,
                                    const int32_t* pending_priority, const cook_host_table* hosts,
                                    const cook_groups* groups, const cook_user_table* users,
                                    const cook_rebalance_params* prm, cook_decision* out_dec,
                                    int32_t* out_victims, int32_t* out_n) {
  return rebalance_impl(dru_mode, running, pending, pending_job_id, pending_priority, hosts, groups, users, prm,
                        out_dec, out_victims, out_n, nullptr);
}

extern "C" int32_t oracle_rebalance_trace(int32_t dru_mode, const cook_running_soa* running,
                                          const cook_jobs_soa* pending, const int64_t* pending_job_id,
                                          const int32_t* pending_priority, const cook_host_table* hosts,
                                          const cook_groups* groups, const cook_user_table* users,
                                          const cook_rebalance_params* prm, cook_decision* out_dec,
                                          int32_t* out_victims, int32_t* out_n, const oracle_reb_trace* tr) {
  return rebalance_impl(dru_mode, running, pending, pending_job_id, pending_priority, hosts, groups, users, prm,
                        out_dec, out_victims, out_n, tr);
}

// ---------------------------------------------------------------------------
// Check used by tests/test_fastdiv.py: the CUDA kernels divide by the (static)
// fitness denominators through their correctly rounded reciprocals,
//   y = RN(1/den), q0 = x*y, q = fma(fma(-den, q0, x), y, q0)
// (cook_b200/csrc/match.cu div_y).  This counts the inputs for which that differs
// from the IEEE quotient x/den the reference computes (clojure `/` on doubles,
// via Fenzo's cpuMemBinPacker) over three families: Cook's value grids, random
// doubles, and denominators with (nearly) all-ones significands.  oracle_check_fastdiv_guard
// covers the dividend guard (fitness.cuh fit_guard): dividends at the edges of what a guarded cycle
// can divide, [2^-600, 2^602), against every denominator safe_rcp accepts, and below the guard.
#include <cmath>
static inline double fastdiv_q(double x, double den, double y) {
  const double q0 = x * y;
  return std::fma(std::fma(-den, q0, x), y, q0);
}
extern "C" int64_t oracle_check_fastdiv(int64_t n_random, uint64_t seed) {
  int64_t bad = 0;
  uint64_t s = seed ? seed : 88172645463325252ull;
  auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
  auto rd = [&](int emin, int emax) {
    const uint64_t m = rnd() & ((1ull << 52) - 1);
    const int e = emin + (int)(rnd() % (uint64_t)(emax - emin + 1));
    const uint64_t bits = ((uint64_t)(e + 1023) << 52) | m;
    double d;
    memcpy(&d, &bits, 8);
    return d;
  };
  for (int bi = 1; bi <= 512; bi++)
    for (int ai = 1; ai <= 1024; ai++) {
      const double b = bi * 0.5, x = ai * 0.5;
      if (fastdiv_q(x, b, 1.0 / b) != x / b) bad++;
    }
  for (int bi = 1; bi <= 2048; bi++)
    for (int ai = 1; ai <= 2048; ai++) {
      const double b = bi * 512.0, x = ai * 512.0;
      if (fastdiv_q(x, b, 1.0 / b) != x / b) bad++;
    }
  for (int64_t i = 0; i < n_random; i++) {
    const double x = rd(-20, 30), b = rd(-20, 30);
    if (fastdiv_q(x, b, 1.0 / b) != x / b) bad++;
  }
  for (int64_t i = 0; i < n_random / 4; i++) {
    const uint64_t m = ((1ull << 52) - 1) - (rnd() % 4);
    const uint64_t bits = ((uint64_t)(1023 + (int)(rnd() % 20)) << 52) | m;
    double b;
    memcpy(&b, &bits, 8);
    const double x = rd(-5, 25);
    if (fastdiv_q(x, b, 1.0 / b) != x / b) bad++;
  }
  return bad;
}

// family 0: dividends guarded amounts can give -- 0, the least binades from 2^-600 up, the largest below
//   2^602 -- by denominators across (1e-100, 1e100), with the bottom and top binades of each drawn often, so
//   that the quotients reach down to 2^-933 and up to 2^934: every one must equal IEEE division.
// family 1: dividends below the guard (subnormal, and normal up to 2^-960), by denominators across the range:
//   the mismatches this counts are why the guard exists.
extern "C" int64_t oracle_check_fastdiv_guard(int64_t n, uint64_t seed, int family) {
  int64_t bad = 0;
  uint64_t s = seed ? seed : 88172645463325252ull;
  auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
  auto rd = [&](int emin, int emax) {   // normal double, exponent uniform in [emin, emax]
    const uint64_t m = rnd() & ((1ull << 52) - 1);
    const int e = emin + (int)(rnd() % (uint64_t)(emax - emin + 1));
    const uint64_t bits = ((uint64_t)(e + 1023) << 52) | m;
    double d;
    memcpy(&d, &bits, 8);
    return d;
  };
  auto safe = [](double den) {          // fitness.cuh safe_rcp
    uint64_t bits;
    memcpy(&bits, &den, 8);
    const uint64_t frac = bits & 0x000fffffffffffffULL;
    return (den > 1e-100 && den < 1e100 && frac != 0x000fffffffffffffULL) ? 1.0 / den : 0.0;
  };
  for (int64_t i = 0; i < n; i++) {
    double x;
    const uint64_t pick = rnd() % 8;
    if (family == 0) {
      x = pick == 0 ? 0.0 : pick < 4 ? rd(-600, -590) : pick < 7 ? rd(590, 601) : rd(-600, 601);
    } else {
      if (pick < 4) {
        const uint64_t bits = 1 + rnd() % ((1ull << 52) - 1);   // subnormal
        memcpy(&x, &bits, 8);
      } else {
        x = rd(-1022, -960);
      }
    }
    const uint64_t dp = rnd() % 4;
    const double den = dp == 0 ? rd(-333, -320) : dp == 1 ? rd(320, 332) : rd(-333, 332);
    const double y = safe(den);
    if (y == 0.0) continue;
    if (fastdiv_q(x, den, y) != x / den) bad++;
  }
  return bad;
}
