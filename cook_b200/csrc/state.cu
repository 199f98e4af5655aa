// state.cu — the resident pool state (SURVEY §8f-1, device half): a pool's pending jobs and running
// tasks kept on the device between cycles, changed by deltas, ranked and matched in place.
//
// Host, O(delta) per batch: the id -> slot maps and free lists, per-slot facts (user code, list lengths,
// which columns hold a non-absent value, the group and attribute-column codes) and the counts and code
// maxima derived from them.  Device: one SoA table per kind whose capacity doubles with device-to-device
// copies, a live flag and a generation stamp per slot, and one append-only arena per CSR list with a
// per-slot (off, len), compacted once its dead entries outnumber the live ones.
// Rank and match gather dense columns from the tables with fold.cuh's compaction and order-wide scan and
// run cook_rank's and cook_match's own code on them: rank_impl over the gathered task columns, and the
// match plan's build, the gathers into the job columns it carved, then its run.  The ranked queue stays
// on the device as (slot, generation) pairs; a match keeps the entries whose slot still holds that
// generation, so a job removed or replaced since the rank leaves the queue.  A rebalance takes the first
// allowed jobs of that queue and every live running task on its host, gathered into the columns the
// rebalancer's build carved, and runs cook_rebalance's walk on them.
// By job id, without re-sending rows: a launch moves pending rows to the running table on the device and
// leaves the state a delta would; a patch writes the match-time columns (allowed, plugin_accept,
// reserved_host) in place and keeps the generation, so the job keeps its queue entry.
// Running usage per user, of the pool and per listed host: the live running rows compacted, sorted by (key, task
// id) and folded per segment, each sum a left fold in ascending task id (DESIGN.md §2).
// Running rows carry their job's group list (a fourth arena, filled by running upserts and moved on the device
// by a launch).  A group's cotasks: the live running rows with a known host expanded into one entry per group,
// sorted by (group, task id).
// Considerable jobs without a match: the live queue entries with their queue positions, their M0 columns gathered,
// cook_match's considerable pass (match.cu) run on them; a consuming call retires the taken entries' generations.
#include <algorithm>
#include <map>
#include <unordered_map>
#include <unordered_set>

#include "fold.cuh"
#include "sort.cuh"

namespace {

// ---- device tables: column k of a table is cols[k] (sz bytes per slot)
enum PCol {
  P_USER, P_PRIO, P_JID, P_CPUS, P_MEM, P_GPUS, P_PORTS, P_ALLOWED, P_PLUGIN, P_GPU_MODEL, P_DISK_REQ, P_DISK_TYPE,
  P_EST, P_CKPT, P_RESERVED, P_NDATA,   // the columns a delta row carries
  P_LIVE = P_NDATA, P_GEN, P_NOFF, P_NLEN, P_AOFF, P_ALEN, P_GOFF, P_GLEN, P_NCOL
};
constexpr int P_SZ[P_NCOL] = {4, 4, 8, 8, 8, 8, 4, 1, 1, 4, 8, 4, 8, 4, 4, 1, 4, 4, 4, 4, 4, 4, 4};
enum RCol { R_USER, R_PRIO, R_START, R_TID, R_JID, R_CPUS, R_MEM, R_GPUS, R_HOST, R_NDATA, R_LIVE = R_NDATA, R_GEN,
            R_GOFF, R_GLEN, R_NCOL };
constexpr int R_SZ[R_NCOL] = {4, 4, 8, 8, 8, 8, 8, 8, 4, 1, 4, 4, 4};

// the pending rows' three lists, then the running rows' group list
enum { L_NOVEL = 0, L_ATTR = 1, L_GROUP = 2, L_RGROUP = 3, L_N };

// ---- scatter: row i of a batch to slot[i].  Upserts write the columns (a null source writes the
// column's absent value) and the rows' list ranges; removals clear the live flag.  Both bump the
// generation, which is what retires a queue entry.  A patch (live null) writes its columns only: the
// slot keeps its live flag and generation, so its queue entry stays.
constexpr int MAXC = 16;
struct ScatterCol { char* dst; const char* src; long long dflt; int sz; };
struct ScatterArgs {
  ScatterCol c[MAXC];
  int nc, n, upsert;
  const int32_t* slot;
  uint8_t* live;           // null: a patch
  uint32_t* gen;
  int32_t* loff[3];        // per-slot list range; null: the table has no lists
  int32_t* llen[3];
  const int32_t* doff[3];  // the batch's CSR offsets (null: empty lists)
  int32_t tail[3];         // where the batch's lists were appended
};

__global__ void scatter_kernel(ScatterArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int s = a.slot[i];
#pragma unroll
  for (int k = 0; k < MAXC; k++) {
    if (k >= a.nc) break;
    const ScatterCol& c = a.c[k];
    if (c.sz == 1) reinterpret_cast<uint8_t*>(c.dst)[s] = c.src ? reinterpret_cast<const uint8_t*>(c.src)[i] : (uint8_t)c.dflt;
    else if (c.sz == 4) reinterpret_cast<int32_t*>(c.dst)[s] = c.src ? reinterpret_cast<const int32_t*>(c.src)[i] : (int32_t)c.dflt;
    else reinterpret_cast<long long*>(c.dst)[s] = c.src ? reinterpret_cast<const long long*>(c.src)[i] : c.dflt;
  }
  if (!a.live) return;
  a.live[s] = a.upsert ? 1 : 0;
  a.gen[s] += 1u;
#pragma unroll
  for (int l = 0; l < 3; l++)
    if (a.loff[l]) {
      const bool has = a.upsert && a.doff[l];
      const int o = has ? a.doff[l][i] : 0;
      a.loff[l][s] = a.tail[l] + o;
      a.llen[l][s] = has ? a.doff[l][i + 1] - o : 0;
    }
}

// ---- launch: pending slot pslot[i] becomes running slot rslot[i].  What the task shares with its job moves
// from the pending table; task id, start time and host (null: -1) come from the call.  The group list starts
// empty at the running arena's tail `rtail`; launch_lists_kernel moves the job's list there when some launched
// job has one.  The pending slot is retired afterwards by a removal scatter.
__global__ void launch_kernel(const int32_t* pslot, const int32_t* rslot, const int64_t* tid, const int64_t* start,
                              const int32_t* host, void* const* pc, void* const* rc, int n, int32_t rtail) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = pslot[i], r = rslot[i];
  static_cast<int32_t*>(rc[R_USER])[r] = static_cast<const int32_t*>(pc[P_USER])[s];
  static_cast<int32_t*>(rc[R_PRIO])[r] = static_cast<const int32_t*>(pc[P_PRIO])[s];
  static_cast<int64_t*>(rc[R_JID])[r] = static_cast<const int64_t*>(pc[P_JID])[s];
  static_cast<double*>(rc[R_CPUS])[r] = static_cast<const double*>(pc[P_CPUS])[s];
  static_cast<double*>(rc[R_MEM])[r] = static_cast<const double*>(pc[P_MEM])[s];
  static_cast<double*>(rc[R_GPUS])[r] = static_cast<const double*>(pc[P_GPUS])[s];
  static_cast<int64_t*>(rc[R_START])[r] = start[i];
  static_cast<int64_t*>(rc[R_TID])[r] = tid[i];
  static_cast<int32_t*>(rc[R_HOST])[r] = host ? host[i] : -1;
  static_cast<uint8_t*>(rc[R_LIVE])[r] = 1;
  static_cast<uint32_t*>(rc[R_GEN])[r] += 1u;
  static_cast<int32_t*>(rc[R_GOFF])[r] = rtail;
  static_cast<int32_t*>(rc[R_GLEN])[r] = 0;
}

// ---- list lengths for the order-wide scan (integer sums: any association is exact)
struct SlotLen {   // arena compaction: slot p, dead slots hold nothing
  const uint8_t* live; const int32_t* len;
  __device__ void operator()(int p, int (&x)[1]) const { x[0] = live[p] ? len[p] : 0; }
};
struct RowLen {    // the match's row p is slot m_slot[p]
  const int32_t* m_slot; const int32_t* len;
  __device__ void operator()(int p, int (&x)[1]) const { x[0] = len[m_slot[p]]; }
};

// warp per live slot: its list moves to the exclusive scan of the live lengths in the new arena
__global__ void list_compact_kernel(OrderScan<int, 1> os, const uint8_t* live, int32_t* off, const int32_t* len, int n,
                                    const int32_t* src0, const int32_t* src1, int32_t* dst0, int32_t* dst1) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n || !live[w]) return;
  const int l = len[w], start = os.at(0, w) - l, o = off[w];
  for (int i = lane; i < l; i += 32) {
    dst0[start + i] = src0[o + i];
    if (dst1) dst1[start + i] = src1[o + i];
  }
  __syncwarp();
  if (lane == 0) off[w] = start;
}

// warp per launched row: pending slot pslot[w]'s group list moves to the running arena at rtail + the exclusive scan
// of the launched rows' lengths, where the equivalent delta's CSR puts it, and becomes running slot rslot[w]'s list
__global__ void launch_lists_kernel(OrderScan<int, 1> os, const int32_t* pslot, const int32_t* rslot, int n,
                                    const int32_t* poff, const int32_t* plen, const int32_t* src, int32_t* roff,
                                    int32_t* rlen, int32_t* dst, int32_t rtail) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n) return;
  const int s = pslot[w], l = plen[s], start = rtail + os.at(0, w) - l, o = poff[s];
  for (int i = lane; i < l; i += 32) dst[start + i] = src[o + i];
  if (lane == 0) {
    roff[rslot[w]] = start;
    rlen[rslot[w]] = l;
  }
}

// warp per match row: the row's list into the dense CSR (doff[n + 1], values) cook_match reads
__global__ void csr_gather_kernel(OrderScan<int, 1> os, const int32_t* m_slot, int n, const int32_t* off,
                                  const int32_t* len, const int32_t* src0, const int32_t* src1, int32_t* doff,
                                  int32_t* dst0, int32_t* dst1) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n) return;
  const int s = m_slot[w], l = len[s], end = os.at(0, w), start = end - l, o = off[s];
  for (int i = lane; i < l; i += 32) {
    dst0[start + i] = src0[o + i];
    if (dst1) dst1[start + i] = src1[o + i];
  }
  if (lane == 0) {
    doff[w + 1] = end;
    if (w == 0) doff[0] = 0;
  }
}

// ---- rank: live rows -> dense task columns (running first), compacted in slot order
struct RunningRows {
  void* const* col; TaskCols o;
  __device__ bool keep(int i) const { return static_cast<const uint8_t*>(col[R_LIVE])[i]; }
  __device__ void emit(int i, int d) const {
    writable(o.user)[d] = static_cast<const int32_t*>(col[R_USER])[i];
    writable(o.prio)[d] = static_cast<const int32_t*>(col[R_PRIO])[i];
    writable(o.start)[d] = static_cast<const int64_t*>(col[R_START])[i];
    writable(o.tid)[d] = static_cast<const int64_t*>(col[R_TID])[i];
    writable(o.jid)[d] = static_cast<const int64_t*>(col[R_JID])[i];
    writable(o.cpus)[d] = static_cast<const double*>(col[R_CPUS])[i];
    writable(o.mem)[d] = static_cast<const double*>(col[R_MEM])[i];
    writable(o.gpus)[d] = static_cast<const double*>(col[R_GPUS])[i];
  }
};
struct PendingRows {
  void* const* col; TaskCols o;
  int32_t* pslot;   // dense pending index -> slot
  int R;
  __device__ bool keep(int i) const { return static_cast<const uint8_t*>(col[P_LIVE])[i]; }
  __device__ void emit(int i, int d) const {
    pslot[d] = i;
    d += R;
    writable(o.user)[d] = static_cast<const int32_t*>(col[P_USER])[i];
    writable(o.prio)[d] = static_cast<const int32_t*>(col[P_PRIO])[i];
    writable(o.start)[d] = INT64_MAX;   // a pending job's synthetic task (tools.clj:582-588)
    writable(o.tid)[d] = -1;
    writable(o.jid)[d] = static_cast<const int64_t*>(col[P_JID])[i];
    writable(o.cpus)[d] = static_cast<const double*>(col[P_CPUS])[i];
    writable(o.mem)[d] = static_cast<const double*>(col[P_MEM])[i];
    writable(o.gpus)[d] = static_cast<const double*>(col[P_GPUS])[i];
  }
};

// the ranked queue (dense pending indices) as (slot, generation) pairs, and its job ids
__global__ void queue_kernel(const int32_t* ranked, const int32_t* n, const int32_t* pslot, const uint32_t* gen,
                             const int64_t* jid, int32_t* q_slot, uint32_t* q_gen, int64_t* q_jid) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= *n) return;
  const int s = pslot[ranked[k]];
  q_slot[k] = s; q_gen[k] = gen[s]; q_jid[k] = jid[s];
}

// ---- match: the queue entries whose slot still holds their generation, in queue order
struct QueueLive {
  const int32_t* q_slot; const uint32_t* q_gen; const uint8_t* live; const uint32_t* gen; int32_t* m_slot;
  __device__ bool keep(int k) const { const int s = q_slot[k]; return live[s] && gen[s] == q_gen[k]; }
  __device__ void emit(int k, int d) const { m_slot[d] = q_slot[k]; }
};

// ---- considerable: the live queue entries with their queue positions
struct QueueLivePos {
  QueueLive q; int32_t* qpos;
  __device__ bool keep(int k) const { return q.keep(k); }
  __device__ void emit(int k, int d) const { q.emit(k, d); qpos[d] = k; }
};
// row d of a considerable call is slot m_slot[d]: the columns M0 reads (a null mask is not gathered)
__global__ void cons_rows_kernel(void* const* col, const int32_t* m_slot, int n, int32_t* ranked, int32_t* user,
                                 double* cpus, double* mem, double* gpus, uint8_t* allowed, uint8_t* plugin) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n) return;
  const int s = m_slot[d];
  ranked[d] = d;
  user[d] = static_cast<const int32_t*>(col[P_USER])[s];
  cpus[d] = static_cast<const double*>(col[P_CPUS])[s];
  mem[d] = static_cast<const double*>(col[P_MEM])[s];
  gpus[d] = static_cast<const double*>(col[P_GPUS])[s];
  if (allowed) allowed[d] = static_cast<const uint8_t*>(col[P_ALLOWED])[s];
  if (plugin) plugin[d] = static_cast<const uint8_t*>(col[P_PLUGIN])[s];
}
// the k-th considerable job (row row[k] < *n): its job id and, with `consume`, its queue entry retired by writing the
// rank-time generation minus one: a slot's generation only grows, so the entry stays stale until the next rank
__global__ void cons_take_kernel(const int32_t* row, const int32_t* n, const int32_t* qpos, const int64_t* q_jid,
                                 uint32_t* q_gen, int consume, int64_t* out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= *n) return;
  const int q = qpos[row[k]];
  out[k] = q_jid[q];
  if (consume) q_gen[q] -= 1u;
}

// row d of the match is slot m_slot[d]: its columns into the plan's
__global__ void fill_rows_kernel(MatchRows r, void* const* col, const int32_t* m_slot, int n) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n) return;
  const int s = m_slot[d];
  const JobDev& o = r.jb;
  r.ranked[d] = d;
  writable(o.user)[d] = static_cast<const int32_t*>(col[P_USER])[s];
  writable(o.cpus)[d] = static_cast<const double*>(col[P_CPUS])[s];
  writable(o.mem)[d] = static_cast<const double*>(col[P_MEM])[s];
  writable(o.gpus)[d] = static_cast<const double*>(col[P_GPUS])[s];
  r.job_id[d] = static_cast<const int64_t*>(col[P_JID])[s];
  if (o.ports) writable(o.ports)[d] = static_cast<const int32_t*>(col[P_PORTS])[s];
  if (o.allowed) writable(o.allowed)[d] = static_cast<const uint8_t*>(col[P_ALLOWED])[s];
  if (o.plugin) writable(o.plugin)[d] = static_cast<const uint8_t*>(col[P_PLUGIN])[s];
  if (o.gpu_model) writable(o.gpu_model)[d] = static_cast<const int32_t*>(col[P_GPU_MODEL])[s];
  if (o.disk_request) {
    writable(o.disk_request)[d] = static_cast<const double*>(col[P_DISK_REQ])[s];
    writable(o.disk_type)[d] = static_cast<const int32_t*>(col[P_DISK_TYPE])[s];
  }
  if (o.est_end_ms) writable(o.est_end_ms)[d] = static_cast<const int64_t*>(col[P_EST])[s];
  if (o.ckpt_location) writable(o.ckpt_location)[d] = static_cast<const int32_t*>(col[P_CKPT])[s];
  if (o.reserved_host) writable(o.reserved_host)[d] = static_cast<const int32_t*>(col[P_RESERVED])[s];
}

// ---- rebalance: the live running rows, host = the index of the row's hostname code in the host table
__global__ void host_map_kernel(const int32_t* hostname_id, int H, int32_t* host_of) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < H) host_of[hostname_id[h]] = h;
}
struct RebRunningRows {
  RunningRows r; int32_t* host; const int32_t* host_of;
  __device__ bool keep(int i) const { return r.keep(i); }
  __device__ void emit(int i, int d) const {
    r.emit(i, d);
    host[d] = host_of[static_cast<const int32_t*>(r.col[R_HOST])[i]];
  }
};
// jobs-to-make-room-for: the live queue entries whose job is allowed to start
struct QueueAllowed {
  QueueLive q; const uint8_t* allowed;
  __device__ bool keep(int k) const { return q.keep(k) && allowed[q.q_slot[k]]; }
  __device__ void emit(int k, int d) const { q.emit(k, d); }
};
// pending job d of the rebalance is slot m_slot[d]: its columns into the build's
__global__ void reb_pending_kernel(RebRows r, void* const* col, const int32_t* m_slot, int n) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n) return;
  const int s = m_slot[d];
  const JobDev& o = r.jb;
  writable(o.user)[d] = static_cast<const int32_t*>(col[P_USER])[s];
  writable(o.cpus)[d] = static_cast<const double*>(col[P_CPUS])[s];
  writable(o.mem)[d] = static_cast<const double*>(col[P_MEM])[s];
  writable(o.gpus)[d] = static_cast<const double*>(col[P_GPUS])[s];
  writable(r.jid)[d] = static_cast<const int64_t*>(col[P_JID])[s];
  writable(r.prio)[d] = static_cast<const int32_t*>(col[P_PRIO])[s];
  writable(o.gpu_model)[d] = static_cast<const int32_t*>(col[P_GPU_MODEL])[s];
  writable(o.disk_request)[d] = static_cast<const double*>(col[P_DISK_REQ])[s];
  writable(o.disk_type)[d] = static_cast<const int32_t*>(col[P_DISK_TYPE])[s];
  writable(o.est_end_ms)[d] = static_cast<const int64_t*>(col[P_EST])[s];
  writable(o.ckpt_location)[d] = static_cast<const int32_t*>(col[P_CKPT])[s];
}

// ---- running usage: the live running rows, dense in slot order; host = the index of the row's hostname
// code in the caller's list, or H when the row's host is -1 or not listed (a segment no output reads)
struct UsageRows {
  void* const* col;
  int32_t* user; int64_t* tid; int32_t* host; double* amt[3];   // host null: no host list
  const int32_t* host_of; int32_t n_codes, H;
  __device__ bool keep(int i) const { return static_cast<const uint8_t*>(col[R_LIVE])[i]; }
  __device__ void emit(int i, int d) const {
    user[d] = static_cast<const int32_t*>(col[R_USER])[i];
    tid[d] = static_cast<const int64_t*>(col[R_TID])[i];
    amt[0][d] = static_cast<const double*>(col[R_CPUS])[i];
    amt[1][d] = static_cast<const double*>(col[R_MEM])[i];
    amt[2][d] = static_cast<const double*>(col[R_GPUS])[i];
    if (host) {
      const int32_t code = static_cast<const int32_t*>(col[R_HOST])[i];
      const int32_t h = code >= 0 && code < n_codes ? host_of[code] : -1;
      host[d] = h < 0 ? H : h;
    }
  }
};
// (key, task id); key null: task id alone.  Task ids are unique among live rows, so the order is total.
struct LessKeyTid {
  const int32_t* key; const int64_t* tid;
  __device__ bool operator()(int32_t a, int32_t b) const {
    if (key && key[a] != key[b]) return key[a] < key[b];
    return tid[a] < tid[b];
  }
};
struct LoadSorted {   // the order-wide scan's addends: cpus, mem, gpus of the row at position p
  const int32_t* ord; const double* amt[3];
  __device__ void operator()(int p, double (&x)[3]) const {
    const int i = ord[p];
    x[0] = amt[0][i]; x[1] = amt[1][i]; x[2] = amt[2][i];
  }
};
// The segments of one kind: segment g is positions [start[g], end[g]) of `ord` (start null: [0, R)).
// `scan`: os holds the order-wide scan of ord, read when the whole order is on the grid.
struct UsageSegs {
  const int32_t* ord; const int32_t* start; const int32_t* end;
  OrderScan<double, 3> os; int scan, n;
};
enum { US_USER, US_HOST, US_POOL, US_N };
struct UsageArgs {
  UsageSegs seg[US_N];
  const double* amt[3];
  const GridFlag* gf; int R;
  double* user_out; int U;                                 // [4][U]: count, cpus, mem, gpus
  double* host_cpus; double* host_mem; int32_t* host_count; // [H]
  double* pool_out;                                        // [4]
};

// Warp per segment (users, then hosts, then the pool): the left fold of cpus, mem and gpus in the segment's
// order (ascending task id within it).  The whole order on the grid: the two ends of the order-wide scan;
// else warp_fold_sum, association-free when the segment alone is on the grid, else the serial chain.
__global__ void __launch_bounds__(128) usage_fold_kernel(UsageArgs a) {
  __shared__ double stage[4][3][32];
  int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, kind = 0;
  while (kind < US_N && g >= a.seg[kind].n) g -= a.seg[kind++].n;
  if (kind == US_N) return;
  const UsageSegs& q = a.seg[kind];
  const int s = q.start ? q.start[g] : 0, e = q.start ? q.end[g] : a.R;
  double acc[3] = {0.0, 0.0, 0.0};
  if (q.scan && grid_exact(a.gf, a.R)) {
    if (e > s)
#pragma unroll
      for (int k = 0; k < 3; k++) acc[k] = q.os.segment_sum(k, e - 1, s);
  } else {
    warp_fold_sum<3, 4>(acc, e - s, grid_exact(a.gf, e - s), [&](int k, double (&x)[3]) {
      const int i = q.ord[s + k];
      x[0] = a.amt[0][i]; x[1] = a.amt[1][i]; x[2] = a.amt[2][i];
      return true;
    }, stage[threadIdx.x >> 5]);
  }
  if (threadIdx.x & 31) return;
  if (kind == US_USER) {
    a.user_out[g] = (double)(e - s);
    a.user_out[a.U + g] = acc[0]; a.user_out[2 * a.U + g] = acc[1]; a.user_out[3 * a.U + g] = acc[2];
  } else if (kind == US_HOST) {
    a.host_count[g] = e - s; a.host_cpus[g] = acc[0]; a.host_mem[g] = acc[1];
  } else {
    a.pool_out[0] = (double)(e - s); a.pool_out[1] = acc[0]; a.pool_out[2] = acc[1]; a.pool_out[3] = acc[2];
  }
}

// ---- cotasks: the live running slots whose host is known and whose group list is not empty, in slot order
struct CotaskRows {
  const uint8_t* live; const int32_t* host; const int32_t* len; int32_t* slot;
  __device__ bool keep(int i) const { return live[i] && host[i] != -1 && len[i] > 0; }
  __device__ void emit(int i, int d) const { slot[d] = i; }
};
struct CotaskArgs {
  OrderScan<int, 1> os;     // inclusive scan of the compacted rows' list lengths
  const int32_t* slot; int K;
  const int32_t* goff; const int32_t* glen; const int32_t* arena; const int32_t* host; const int64_t* tid;
  const int32_t* host_of; int32_t n_codes;   // hostname code -> index of the listed host, or -1; null: none listed
  const int32_t* gcol;      // [n_groups] the group's column among the uploaded ones, or -1
  const int32_t* attr; int H;   // the uploaded columns, [columns][H]
  int32_t* e_grp; int64_t* e_tid; int32_t* e_host; int32_t* e_attr;
};
// thread per compacted row: one entry per group of its list, placed where the scan puts the row
__global__ void cotask_expand_kernel(CotaskArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.K) return;
  const int s = a.slot[k], l = a.glen[s], start = a.os.at(0, k) - l, o = a.goff[s];
  const int32_t code = a.host[s];
  const int32_t h = a.host_of && code < a.n_codes ? a.host_of[code] : -1;
  const int64_t t = a.tid[s];
  for (int i = 0; i < l; i++) {
    const int32_t g = a.arena[o + i], c = a.gcol[g];
    a.e_grp[start + i] = g;
    a.e_tid[start + i] = t;
    a.e_host[start + i] = code;
    a.e_attr[start + i] = c >= 0 && h >= 0 ? a.attr[(size_t)c * a.H + h] : 0;
  }
}
// Position p < N of the (group, task id) order into the value columns; p <= G: the first position of group p,
// i.e. the entries of smaller groups (a binary search), so a group without entries gets an empty range.
__global__ void cotask_out_kernel(const int32_t* ord, const int32_t* e_grp, const int32_t* e_host,
                                  const int32_t* e_attr, int N, int G, int32_t* off, int32_t* o_host, int32_t* o_attr) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < N) {
    const int i = ord[p];
    o_host[p] = e_host[i];
    o_attr[p] = e_attr[i];
  }
  if (p <= G) {
    int lo = 0, hi = N;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (e_grp[ord[m]] < p) lo = m + 1;
      else hi = m;
    }
    off[p] = lo;
  }
}

// ---- host side
// the non-absent values of a pending row, counted per column (the match's constraint switch)
enum { F_GPUS, F_PORTS, F_NOT_ALLOWED, F_NOT_PLUGIN, F_GPU_MODEL, F_DISK, F_EST, F_CKPT, F_RESERVED, F_N };

struct PendingInfo {
  int32_t user = 0;
  int32_t len[3] = {0, 0, 0};
  uint16_t flags = 0;
  std::vector<int32_t> groups, attr_cols;
};

struct Table {
  int ncol = 0;
  const int* sz = nullptr;
  void* col[P_NCOL] = {};
  void** d_col = nullptr;        // the column pointers on the device (for the gather kernels)
  int32_t cap = 0, hw = 0;       // slots allocated, slots ever used
  int nlist = 0, lcol[3] = {};   // the per-slot (off, len) column pairs of the table's lists: off at lcol[l]
  std::unordered_map<int64_t, int32_t> slot_of;
  std::vector<int32_t> free;

  template <class T>
  const T* at(int k) const { return static_cast<const T*>(col[k]); }
  // capacity >= n: new columns, zeroed, the old contents copied (device to device)
  cudaError_t grow(int32_t n, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    const int32_t ncap = std::max<int32_t>(n, std::max<int32_t>(2 * cap, 1024));
    void* nc[P_NCOL] = {};
    for (int k = 0; k < ncol; k++) {
      cudaError_t e = cudaMalloc(&nc[k], (size_t)ncap * sz[k]);
      if (e == cudaSuccess) e = cudaMemsetAsync(nc[k], 0, (size_t)ncap * sz[k], st);
      if (e == cudaSuccess && col[k]) e = cudaMemcpyAsync(nc[k], col[k], (size_t)cap * sz[k], cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) {
        for (int j = 0; j <= k; j++) if (nc[j]) cudaFree(nc[j]);
        return e;
      }
    }
    if (!d_col) {
      cudaError_t e = cudaMalloc(&d_col, sizeof(void*) * P_NCOL);
      if (e != cudaSuccess) return e;
    }
    cudaError_t e = cudaMemcpyAsync(d_col, nc, sizeof(void*) * P_NCOL, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return e;
    for (int k = 0; k < ncol; k++) {
      if (col[k]) cudaFree(col[k]);
      col[k] = nc[k];
    }
    cap = ncap;
    return cudaSuccess;
  }
  int32_t take_slot() {
    if (!free.empty()) { const int32_t s = free.back(); free.pop_back(); return s; }
    return hw++;
  }
  void release() {
    for (int k = 0; k < ncol; k++) if (col[k]) cudaFree(col[k]);
    if (d_col) cudaFree(d_col);
  }
};

struct ListArena {
  int k = 1;                      // value arrays: 2 for (attribute column, value)
  int32_t* v[2] = {};
  int32_t* alt[2] = {};           // compaction target, same capacity
  int64_t cap = 0, tail = 0, live = 0;
  cudaError_t grow(int64_t n, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    const int64_t ncap = std::max<int64_t>(n, std::max<int64_t>(2 * cap, 4096));
    for (int i = 0; i < k; i++) {
      int32_t* p = nullptr;
      cudaError_t e = cudaMalloc(&p, sizeof(int32_t) * ncap);
      if (e == cudaSuccess && tail) e = cudaMemcpyAsync(p, v[i], sizeof(int32_t) * tail, cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) { if (p) cudaFree(p); return e; }
      if (v[i]) cudaFree(v[i]);
      v[i] = p;
      if (alt[i]) cudaFree(alt[i]);
      alt[i] = nullptr;
    }
    cap = ncap;
    return cudaSuccess;
  }
  void release() {
    for (int i = 0; i < 2; i++) { if (v[i]) cudaFree(v[i]); if (alt[i]) cudaFree(alt[i]); }
  }
};

void count_add(std::map<int32_t, int64_t>& m, int32_t code, int64_t d) {
  auto it = m.emplace(code, 0).first;
  if ((it->second += d) == 0) m.erase(it);
}
int32_t count_max(const std::map<int32_t, int64_t>& m) { return m.empty() ? -1 : m.rbegin()->first; }

struct PoolState {
  Table pend, run;
  std::vector<PendingInfo> pinfo;    // by pending slot
  std::vector<int32_t> ruser, rhost; // by running slot
  std::vector<std::vector<int32_t>> rgroups;   // by running slot: its group list
  ListArena lists[L_N];
  std::map<int32_t, int64_t> users_p, users_r, attr_cols, groups;   // code -> live uses
  std::map<int32_t, int64_t> hosts_r;                               // running rows' hostname codes (-1 too)
  std::map<int32_t, int64_t> groups_r;                              // running rows' group codes
  int64_t cot_rows = 0, cot_n = 0;   // live running rows with a known host and a group list, and their entries
  int64_t nflag[F_N] = {};
  std::unordered_set<int32_t> reserved;   // the live pending slots whose reserved_host is not -1
  Arena stage;                        // one batch's uploads
  Arena scratch;                      // one call's device buffers
  Arena derive;                       // a derived match's or rebalance's running-side scratch (scratch is live then)
  Arena queue;                        // the ranked queue, carved by rank only: it lives until the match
  int32_t* counters = nullptr;        // [0] running rows, [1] pending rows, [2] live queue entries
  GridFlag* gf0 = nullptr;            // stays zero: integer scans are always exact
  const int32_t* q_slot = nullptr; const uint32_t* q_gen = nullptr; const int64_t* q_jid = nullptr;
  int32_t n_q = 0;
  bool ranked = false;

  PoolState() {
    pend.ncol = P_NCOL; pend.sz = P_SZ;
    run.ncol = R_NCOL; run.sz = R_SZ;
    pend.nlist = 3; pend.lcol[L_NOVEL] = P_NOFF; pend.lcol[L_ATTR] = P_AOFF; pend.lcol[L_GROUP] = P_GOFF;
    run.nlist = 1; run.lcol[0] = R_GOFF;
    lists[L_ATTR].k = 2;
  }
  void release() {
    pend.release(); run.release();
    for (auto& l : lists) l.release();
    stage.release(); scratch.release(); derive.release(); queue.release();
    if (counters) cudaFree(counters);
    if (gf0) cudaFree(gf0);
  }
  void add_pending(int32_t slot, const PendingInfo& pi, int64_t sign) {
    count_add(users_p, pi.user, sign);
    for (int32_t g : pi.groups) count_add(groups, g, sign);
    for (int32_t c : pi.attr_cols) count_add(attr_cols, c, sign);
    for (int l = 0; l < 3; l++) lists[l].live += sign * pi.len[l];
    for (int f = 0; f < F_N; f++) if ((pi.flags >> f) & 1) nflag[f] += sign;
    if ((pi.flags >> F_RESERVED) & 1) {
      if (sign > 0) reserved.insert(slot);
      else reserved.erase(slot);
    }
  }
  // running slot `slot`'s row (ruser, rhost, rgroups) enters (+1) or leaves (-1) the counts
  void add_running(int32_t slot, int64_t sign) {
    count_add(users_r, ruser[slot], sign);
    count_add(hosts_r, rhost[slot], sign);
    const std::vector<int32_t>& g = rgroups[slot];
    for (int32_t c : g) count_add(groups_r, c, sign);
    lists[L_RGROUP].live += sign * (int64_t)g.size();
    if (rhost[slot] != -1 && !g.empty()) {
      cot_rows += sign;
      cot_n += sign * (int64_t)g.size();
    }
  }
  void running_room(int32_t slot) {
    if ((size_t)slot < ruser.size()) return;
    const size_t n = std::max<size_t>(slot + 1, 2 * ruser.size());
    ruser.resize(n); rhost.resize(n); rgroups.resize(n);
  }
  // a live pending slot's flag f after a patch of its column
  void set_flag(int32_t slot, int f, bool on) {
    PendingInfo& pi = pinfo[slot];
    if ((bool)((pi.flags >> f) & 1) == on) return;
    pi.flags ^= (uint16_t)(1u << f);
    nflag[f] += on ? 1 : -1;
    if (f == F_RESERVED) {
      if (on) reserved.insert(slot);
      else reserved.erase(slot);
    }
  }
};

void state_free(void* p) {
  PoolState* s = static_cast<PoolState*>(p);
  if (s) { s->release(); delete s; }
}

PoolState* state_of(cook_pool* pool, bool create) {
  if (!pool->state && create) {
    PoolState* s = new PoolState();
    if (cudaMalloc(&s->counters, sizeof(int32_t) * 8) != cudaSuccess ||
        cudaMalloc(&s->gf0, sizeof(GridFlag)) != cudaSuccess || cudaMemset(s->gf0, 0, sizeof(GridFlag)) != cudaSuccess) {
      state_free(s);
      return nullptr;
    }
    pool->state = s;
    pool->state_free = state_free;
  }
  return static_cast<PoolState*>(pool->state);
}

bool csr_ok(const int32_t* off, int n, const int32_t* v0, const int32_t* v1, bool two) {
  if (!off) return true;
  if (off[0] != 0) return false;
  for (int i = 0; i < n; i++) if (off[i + 1] < off[i]) return false;
  return off[n] == 0 || (v0 && (!two || v1));
}

long long bits_of(double x) { long long b; memcpy(&b, &x, 8); return b; }

// hostname codes that are non-negative and distinct; *n_codes: one past the largest
bool host_codes(const int32_t* code, int H, int32_t* n_codes) {
  std::unordered_set<int32_t> seen;
  seen.reserve((size_t)H);
  *n_codes = 0;
  for (int h = 0; h < H; h++) {
    if (code[h] < 0 || !seen.insert(code[h]).second) return false;
    *n_codes = std::max(*n_codes, code[h] + 1);
  }
  return true;
}

// the CSR lists of rows m_slot[0, n) into the dense lists of `o` that are carved (non-null)
void gather_lists(const PoolState* S, const JobDev& o, const int32_t* m_slot, int n, const OrderScan<int, 1>& os,
                  cudaStream_t st, int* nl) {
  const int32_t* doff[3] = {o.novel_off, o.attr_off, o.group_off};
  const int32_t* dst[3][2] = {{o.novel_host, nullptr}, {o.attr_col, o.attr_val}, {o.group_idx, nullptr}};
  const int loff[3] = {P_NOFF, P_AOFF, P_GOFF};
  for (int l = 0; l < 3; l++) {
    if (!doff[l]) continue;
    const int32_t* len = S->pend.at<int32_t>(loff[l] + 1);
    order_scan(os, RowLen{m_slot, len}, n, S->gf0, st, nl);
    csr_gather_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, m_slot, n, S->pend.at<int32_t>(loff[l]), len, S->lists[l].v[0],
                                                   S->lists[l].v[1], writable(doff[l]), writable(dst[l][0]),
                                                   writable(dst[l][1]));
    (*nl)++;
  }
}

// compaction of every list arena whose dead entries outnumber its live ones
int32_t compact_lists(cook_pool* pool, PoolState* S, cudaStream_t st, int* nl) {
  for (int l = 0; l < L_N; l++) {
    ListArena& A = S->lists[l];
    if (A.tail - A.live <= A.live) continue;
    const bool run = l == L_RGROUP;
    const Table& t = run ? S->run : S->pend;
    const int n = t.hw, oc = t.lcol[run ? 0 : l];
    if (A.live > 0 && n > 0) {
      for (int i = 0; i < A.k; i++)
        if (!A.alt[i]) CK(pool, cudaMalloc(&A.alt[i], sizeof(int32_t) * std::max<int64_t>(A.cap, 1)));
      OrderScan<int, 1> os;
      CK(pool, carve(S->scratch, st, nullptr, nullptr, [&](Carve& c) {
        os.part[0] = c.take<int32_t>(n);
        os.tile[0] = c.take<int32_t>((n + OS_TILE - 1) / OS_TILE + 1);
      }));
      const uint8_t* live = static_cast<const uint8_t*>(t.col[run ? (int)R_LIVE : (int)P_LIVE]);
      int32_t* off = static_cast<int32_t*>(t.col[oc]);
      const int32_t* len = static_cast<const int32_t*>(t.col[oc + 1]);
      order_scan(os, SlotLen{live, len}, n, S->gf0, st, nl);
      list_compact_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, live, off, len, n, A.v[0], A.v[1], A.alt[0],
                                                       A.k > 1 ? A.alt[1] : nullptr);
      (*nl)++;
      CK(pool, cudaGetLastError());
      for (int i = 0; i < A.k; i++) std::swap(A.v[i], A.alt[i]);
    }
    A.tail = A.live;
  }
  return COOK_OK;
}

// one scatter_kernel launch of a batch's n rows into table t.  live_col < 0: a patch (live flag and generation
// untouched); `tail` (upserts and removals): where the batch's lists were appended, one per list of the table.
void scatter(ScatterArgs& a, Table& t, int n, int upsert, int live_col, const int32_t* tail, cudaStream_t st, int* nl) {
  if (!n) return;
  a.n = n; a.upsert = upsert;
  if (live_col >= 0) {
    a.live = static_cast<uint8_t*>(t.col[live_col]);
    a.gen = static_cast<uint32_t*>(t.col[live_col + 1]);
  }
  if (tail) {
    for (int l = 0; l < t.nlist; l++) {
      a.loff[l] = static_cast<int32_t*>(t.col[t.lcol[l]]);
      a.llen[l] = static_cast<int32_t*>(t.col[t.lcol[l] + 1]);
      a.tail[l] = tail[l];
    }
  }
  scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
  (*nl)++;
}

int32_t apply(cook_pool* pool, PoolState* S, const cook_state_delta* d) {
  const cook_jobs_soa& P = d->pending;
  const cook_tasks_soa& T = d->running;
  const int np = P.n, nr = T.n, npr = d->n_pending_rm, nrr = d->n_running_rm;
  if (np < 0 || nr < 0 || npr < 0 || nrr < 0) return set_err(pool, COOK_E_BADARG, "cook_state_apply: bad sizes");
  if (np && (!P.user || !P.cpus || !P.mem || !d->pending_priority || !d->pending_job_id))
    return set_err(pool, COOK_E_BADARG, "cook_state_apply: pending upserts need user, cpus, mem, priority and job id");
  if (nr && (!T.user || !T.priority || !T.start_time || !T.task_id || !T.job_id || !T.cpus || !T.mem))
    return set_err(pool, COOK_E_BADARG, "cook_state_apply: running upserts need every column but gpus");
  if ((npr && !d->pending_rm_job_id) || (nrr && !d->running_rm_task_id))
    return set_err(pool, COOK_E_BADARG, "cook_state_apply: null removal ids");
  if (!csr_ok(P.novel_off, np, P.novel_host, nullptr, false) || !csr_ok(P.attr_off, np, P.attr_col, P.attr_val, true) ||
      !csr_ok(P.group_off, np, P.group_idx, nullptr, false) ||
      !csr_ok(d->running_group_off, nr, d->running_group_idx, nullptr, false))
    return set_err(pool, COOK_E_BADARG, "cook_state_apply: malformed CSR offsets");
  // codes are checked where they enter
  if (!idx_in_range(P.user, np, 0, INT32_MAX) || !idx_in_range(T.user, nr, 0, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "cook_state_apply: negative user code");
  if ((P.attr_off && !idx_in_range(P.attr_col, P.attr_off[np], 0, INT32_MAX)) ||
      (P.group_off && !idx_in_range(P.group_idx, P.group_off[np], 0, INT32_MAX)) ||
      (d->running_group_off && !idx_in_range(d->running_group_idx, d->running_group_off[nr], 0, INT32_MAX)) ||
      (P.novel_off && !idx_in_range(P.novel_host, P.novel_off[np], 0, INT32_MAX)) ||
      !idx_in_range(P.reserved_host, np, -1, INT32_MAX) || !idx_in_range(d->running_hostname_id, nr, -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "cook_state_apply: bad attribute column, group or hostname code");
  const bool rs = d->reset != 0;
  {
    std::unordered_set<int64_t> seen;
    seen.reserve((size_t)np + npr);
    for (int i = 0; i < np; i++)
      if (!seen.insert(d->pending_job_id[i]).second) return set_err(pool, COOK_E_BADARG, "cook_state_apply: job id twice in one batch");
    for (int i = 0; i < npr; i++) {
      const int64_t id = d->pending_rm_job_id[i];
      if (!seen.insert(id).second) return set_err(pool, COOK_E_BADARG, "cook_state_apply: job id twice in one batch");
      if (rs || !S->pend.slot_of.count(id)) return set_err(pool, COOK_E_BADARG, "cook_state_apply: removal of an unknown job id");
    }
    seen.clear();
    for (int i = 0; i < nr; i++)
      if (!seen.insert(T.task_id[i]).second) return set_err(pool, COOK_E_BADARG, "cook_state_apply: task id twice in one batch");
    for (int i = 0; i < nrr; i++) {
      const int64_t id = d->running_rm_task_id[i];
      if (!seen.insert(id).second) return set_err(pool, COOK_E_BADARG, "cook_state_apply: task id twice in one batch");
      if (rs || !S->run.slot_of.count(id)) return set_err(pool, COOK_E_BADARG, "cook_state_apply: removal of an unknown task id");
    }
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  // ---- the batch is valid: the host side first (slots, counts), all O(delta)
  if (rs) {
    for (Table* t : {&S->pend, &S->run}) {
      if (t->hw) {
        const int lc = t == &S->pend ? (int)P_LIVE : (int)R_LIVE;
        CK(pool, cudaMemsetAsync(t->col[lc], 0, (size_t)t->hw, st));
      }
      t->slot_of.clear(); t->free.clear(); t->hw = 0;
    }
    S->users_p.clear(); S->users_r.clear(); S->attr_cols.clear(); S->groups.clear(); S->hosts_r.clear();
    S->groups_r.clear();
    S->cot_rows = S->cot_n = 0;
    S->reserved.clear();
    for (auto& f : S->nflag) f = 0;
    for (auto& l : S->lists) l.tail = l.live = 0;
  }
  std::vector<int32_t> prm_slot(npr), pup_slot(np), rrm_slot(nrr), rup_slot(nr);
  for (int i = 0; i < npr; i++) {
    auto it = S->pend.slot_of.find(d->pending_rm_job_id[i]);
    const int32_t s = it->second;
    S->pend.slot_of.erase(it);
    S->add_pending(s, S->pinfo[s], -1);
    S->pend.free.push_back(s);
    prm_slot[i] = s;
  }
  for (int i = 0; i < nrr; i++) {
    auto it = S->run.slot_of.find(d->running_rm_task_id[i]);
    const int32_t s = it->second;
    S->run.slot_of.erase(it);
    S->add_running(s, -1);
    S->run.free.push_back(s);
    rrm_slot[i] = s;
  }
  for (int i = 0; i < np; i++) {
    auto it = S->pend.slot_of.find(d->pending_job_id[i]);
    int32_t s;
    if (it != S->pend.slot_of.end()) { s = it->second; S->add_pending(s, S->pinfo[s], -1); }
    else { s = S->pend.take_slot(); S->pend.slot_of.emplace(d->pending_job_id[i], s); }
    if ((size_t)s >= S->pinfo.size()) S->pinfo.resize(std::max<size_t>(s + 1, 2 * S->pinfo.size()));
    PendingInfo& pi = S->pinfo[s];
    pi.user = P.user[i];
    pi.len[L_NOVEL] = P.novel_off ? P.novel_off[i + 1] - P.novel_off[i] : 0;
    pi.len[L_ATTR] = P.attr_off ? P.attr_off[i + 1] - P.attr_off[i] : 0;
    pi.len[L_GROUP] = P.group_off ? P.group_off[i + 1] - P.group_off[i] : 0;
    pi.attr_cols.assign(P.attr_off ? P.attr_col + P.attr_off[i] : nullptr, P.attr_off ? P.attr_col + P.attr_off[i + 1] : nullptr);
    pi.groups.assign(P.group_off ? P.group_idx + P.group_off[i] : nullptr, P.group_off ? P.group_idx + P.group_off[i + 1] : nullptr);
    const bool f[F_N] = {P.gpus && P.gpus[i] != 0.0, P.ports && P.ports[i] != 0, P.allowed && !P.allowed[i],
                         P.plugin_accept && !P.plugin_accept[i], P.gpu_model && P.gpu_model[i] != -1,
                         P.disk_request && P.disk_request[i] >= 0.0, P.est_end_ms && P.est_end_ms[i] != -1,
                         P.ckpt_location && P.ckpt_location[i] != -1, P.reserved_host && P.reserved_host[i] != -1};
    pi.flags = 0;
    for (int k = 0; k < F_N; k++) if (f[k]) pi.flags |= (uint16_t)(1u << k);
    S->add_pending(s, pi, +1);
    pup_slot[i] = s;
  }
  const int32_t* rgo = d->running_group_off;
  for (int i = 0; i < nr; i++) {
    auto it = S->run.slot_of.find(T.task_id[i]);
    int32_t s;
    if (it != S->run.slot_of.end()) {
      s = it->second;
      S->add_running(s, -1);
    } else {
      s = S->run.take_slot();
      S->run.slot_of.emplace(T.task_id[i], s);
    }
    S->running_room(s);
    S->ruser[s] = T.user[i];
    S->rhost[s] = d->running_hostname_id ? d->running_hostname_id[i] : -1;
    S->rgroups[s].assign(rgo ? d->running_group_idx + rgo[i] : nullptr, rgo ? d->running_group_idx + rgo[i + 1] : nullptr);
    S->add_running(s, +1);
    rup_slot[i] = s;
  }
  // ---- device: capacity, the upload, then the scatters (removals before upserts: a slot a removal
  // frees may be taken by an upsert of the same batch)
  CK(pool, S->pend.grow(S->pend.hw, st));
  CK(pool, S->run.grow(S->run.hw, st));
  const int32_t* lists_off[3] = {P.novel_off, P.attr_off, P.group_off};
  const int32_t* lists_v[3][2] = {{P.novel_host, nullptr}, {P.attr_col, P.attr_val}, {P.group_idx, nullptr}};
  int32_t tail0[3];
  for (int l = 0; l < 3; l++) {
    tail0[l] = (int32_t)S->lists[l].tail;
    const int64_t add = lists_off[l] ? lists_off[l][np] : 0;
    CK(pool, S->lists[l].grow(S->lists[l].tail + add, st));
    S->lists[l].tail += add;
  }
  ListArena& RG = S->lists[L_RGROUP];
  const int32_t rtail0 = (int32_t)RG.tail;
  const int64_t radd = rgo ? rgo[nr] : 0;
  CK(pool, RG.grow(RG.tail + radd, st));
  RG.tail += radd;
  ScatterArgs pu, pr, ru, rr;
  memset(&pu, 0, sizeof(pu)); memset(&pr, 0, sizeof(pr)); memset(&ru, 0, sizeof(ru)); memset(&rr, 0, sizeof(rr));
  int64_t h2d = 0;
  const cudaError_t carved = carve(S->stage, st, pool->ev[20], &h2d, [&](Carve& c) {
    if (np) {
      const void* src[P_NDATA] = {P.user, d->pending_priority, d->pending_job_id, P.cpus, P.mem, P.gpus, P.ports,
                                  P.allowed, P.plugin_accept, P.gpu_model, P.disk_request, P.disk_type, P.est_end_ms,
                                  P.ckpt_location, P.reserved_host};
      const long long dflt[P_NDATA] = {0, 0, 0, 0, 0, 0, 0, 1, 1, -1, bits_of(-1.0), -1, -1, -1, -1};
      for (int k = 0; k < P_NDATA; k++) {
        const char* up = nullptr;
        if (P_SZ[k] == 1) up = reinterpret_cast<const char*>(c.up(static_cast<const uint8_t*>(src[k]), np));
        else if (P_SZ[k] == 4) up = reinterpret_cast<const char*>(c.up(static_cast<const int32_t*>(src[k]), np));
        else up = reinterpret_cast<const char*>(c.up(static_cast<const int64_t*>(src[k]), np));
        pu.c[k] = ScatterCol{static_cast<char*>(S->pend.col[k]), up, dflt[k], P_SZ[k]};
      }
      pu.nc = P_NDATA;
      pu.slot = c.up(pup_slot.data(), np);
      for (int l = 0; l < 3; l++) {
        pu.doff[l] = c.up(lists_off[l], np + 1);
        const int64_t nv = lists_off[l] ? lists_off[l][np] : 0;
        for (int i = 0; i < S->lists[l].k; i++)
          if (c.base && nv) c.copy(S->lists[l].v[i] + tail0[l], lists_v[l][i], nv);
      }
    }
    if (npr) pr.slot = c.up(prm_slot.data(), npr);
    if (nr) {
      const void* src[R_NDATA] = {T.user, T.priority, T.start_time, T.task_id, T.job_id, T.cpus, T.mem, T.gpus,
                                  d->running_hostname_id};
      const long long dflt[R_NDATA] = {0, 0, 0, 0, 0, 0, 0, 0, -1};
      for (int k = 0; k < R_NDATA; k++) {
        const char* up = R_SZ[k] == 4 ? reinterpret_cast<const char*>(c.up(static_cast<const int32_t*>(src[k]), nr))
                                      : reinterpret_cast<const char*>(c.up(static_cast<const int64_t*>(src[k]), nr));
        ru.c[k] = ScatterCol{static_cast<char*>(S->run.col[k]), up, dflt[k], R_SZ[k]};
      }
      ru.nc = R_NDATA;
      ru.slot = c.up(rup_slot.data(), nr);
      ru.doff[0] = c.up(rgo, nr + 1);
      if (c.base && radd) c.copy(RG.v[0] + rtail0, d->running_group_idx, radd);
    }
    if (nrr) rr.slot = c.up(rrm_slot.data(), nrr);
  });
  CK(pool, carved);
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int nl = 0;
  scatter(pr, S->pend, npr, 0, P_LIVE, tail0, st, &nl);
  scatter(rr, S->run, nrr, 0, R_LIVE, &rtail0, st, &nl);
  scatter(pu, S->pend, np, 1, P_LIVE, tail0, st, &nl);
  scatter(ru, S->run, nr, 1, R_LIVE, &rtail0, st, &nl);
  CK(pool, cudaGetLastError());
  int32_t rc = compact_lists(pool, S, st, &nl);
  if (rc != COOK_OK) return rc;
  CK(pool, cudaEventRecord(pool->ev[22], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_STATE, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[22], h2d, 0, nl);
  return COOK_OK;
}

// the slots of n distinct live pending job ids, or why not
const char* pending_slots(const PoolState* S, int n, const int64_t* job_id, std::vector<int32_t>* slot) {
  std::unordered_set<int64_t> seen;
  seen.reserve((size_t)n);
  slot->resize(n);
  for (int i = 0; i < n; i++) {
    if (!seen.insert(job_id[i]).second) return "job id twice";
    auto it = S->pend.slot_of.find(job_id[i]);
    if (it == S->pend.slot_of.end()) return "unknown job id";
    (*slot)[i] = it->second;
  }
  return nullptr;
}

// pending_rm = job_id plus the running upserts built from the rows, without their columns crossing the bus
int32_t launch(cook_pool* pool, PoolState* S, int n, const int64_t* job_id, const int64_t* task_id,
               const int64_t* start_time, const int32_t* hostname_id) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "cook_state_launch: n < 0");
  if (n && (!job_id || !task_id || !start_time))
    return set_err(pool, COOK_E_BADARG, "cook_state_launch: null job_id, task_id or start_time");
  if (!idx_in_range(hostname_id, n, -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "cook_state_launch: a hostname code below -1");
  std::vector<int32_t> pslot, rslot(n);
  if (const char* why = pending_slots(S, n, job_id, &pslot)) return set_err(pool, COOK_E_BADARG, "cook_state_launch: %s", why);
  {
    std::unordered_set<int64_t> seen;
    seen.reserve((size_t)n);
    for (int i = 0; i < n; i++) {
      if (!seen.insert(task_id[i]).second) return set_err(pool, COOK_E_BADARG, "cook_state_launch: task id twice");
      if (S->run.slot_of.count(task_id[i])) return set_err(pool, COOK_E_BADARG, "cook_state_launch: task id already running");
    }
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  // ---- host side, in cook_state_apply's order: the removals free their slots, then the tasks take theirs
  for (int i = 0; i < n; i++) {
    const int32_t s = pslot[i];
    S->pend.slot_of.erase(job_id[i]);
    S->add_pending(s, S->pinfo[s], -1);
    S->pend.free.push_back(s);
  }
  int64_t ng = 0;   // group list entries that move with the jobs
  for (int i = 0; i < n; i++) {
    const int32_t r = S->run.take_slot();
    S->run.slot_of.emplace(task_id[i], r);
    S->running_room(r);
    S->ruser[r] = S->pinfo[pslot[i]].user;
    S->rhost[r] = hostname_id ? hostname_id[i] : -1;
    S->rgroups[r] = S->pinfo[pslot[i]].groups;
    S->add_running(r, +1);
    ng += (int64_t)S->rgroups[r].size();
    rslot[i] = r;
  }
  // ---- device: capacity, the upload, the move (rows, then group lists), the pending slots' removal, then the
  // arena rule
  CK(pool, S->run.grow(S->run.hw, st));
  ListArena& RG = S->lists[L_RGROUP];
  const int32_t rtail0 = (int32_t)RG.tail;
  CK(pool, RG.grow(RG.tail + ng, st));
  RG.tail += ng;
  const int32_t *d_pslot = nullptr, *d_rslot = nullptr, *d_host = nullptr;
  const int64_t *d_tid = nullptr, *d_start = nullptr;
  OrderScan<int, 1> os;
  int64_t h2d = 0;
  CK(pool, carve(S->stage, st, pool->ev[20], &h2d, [&](Carve& c) {
    if (!n) return;
    d_pslot = c.up(pslot.data(), n); d_rslot = c.up(rslot.data(), n);
    d_tid = c.up(task_id, n); d_start = c.up(start_time, n);
    d_host = c.up(hostname_id, n);
    if (ng) {   // device-only buffers: nothing uploaded
      os.part[0] = c.take<int32_t>(n);
      os.tile[0] = c.take<int32_t>((n + OS_TILE - 1) / OS_TILE + 1);
    }
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int nl = 0;
  if (n) {
    launch_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_pslot, d_rslot, d_tid, d_start, d_host, S->pend.d_col,
                                                   S->run.d_col, n, rtail0);
    nl++;
    if (ng) {
      const int32_t* plen = S->pend.at<int32_t>(P_GLEN);
      order_scan(os, RowLen{d_pslot, plen}, n, S->gf0, st, &nl);
      launch_lists_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, d_pslot, d_rslot, n, S->pend.at<int32_t>(P_GOFF), plen,
                                                       S->lists[L_GROUP].v[0], static_cast<int32_t*>(S->run.col[R_GOFF]),
                                                       static_cast<int32_t*>(S->run.col[R_GLEN]), RG.v[0], rtail0);
      nl++;
    }
    ScatterArgs rm;
    memset(&rm, 0, sizeof(rm));
    rm.slot = d_pslot;
    int32_t tail[3];
    for (int l = 0; l < 3; l++) tail[l] = (int32_t)S->lists[l].tail;
    scatter(rm, S->pend, n, 0, P_LIVE, tail, st, &nl);
  }
  CK(pool, cudaGetLastError());
  int32_t rc = compact_lists(pool, S, st, &nl);
  if (rc != COOK_OK) return rc;
  CK(pool, cudaEventRecord(pool->ev[22], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_STATE, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[22], h2d, 0, nl);
  return COOK_OK;
}

// the given match-time columns of live pending rows, in place; clear: every reservation is dropped first
int32_t patch(cook_pool* pool, PoolState* S, int n, const int64_t* job_id, const uint8_t* allowed,
              const uint8_t* plugin_accept, const int32_t* reserved_host, bool clear) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "cook_state_patch: n < 0");
  if (n && !job_id) return set_err(pool, COOK_E_BADARG, "cook_state_patch: null job_id");
  if (!idx_in_range(reserved_host, n, -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "cook_state_patch: a reserved_host below -1");
  std::vector<int32_t> slot;
  if (const char* why = pending_slots(S, n, job_id, &slot)) return set_err(pool, COOK_E_BADARG, "cook_state_patch: %s", why);
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  // ---- host side: the per-slot flags and their counts, O(n + reservations cleared)
  std::vector<int32_t> cleared;
  if (clear) {
    cleared.assign(S->reserved.begin(), S->reserved.end());
    for (int32_t s : cleared) S->set_flag(s, F_RESERVED, false);
  }
  for (int i = 0; i < n; i++) {
    const int32_t s = slot[i];
    if (allowed) S->set_flag(s, F_NOT_ALLOWED, !allowed[i]);
    if (plugin_accept) S->set_flag(s, F_NOT_PLUGIN, !plugin_accept[i]);
    if (reserved_host) S->set_flag(s, F_RESERVED, reserved_host[i] != -1);
  }
  // ---- device: the cleared slots get -1, then the batch's columns
  const int nc = (int)cleared.size();
  const bool cols = n && (allowed || plugin_accept || reserved_host);
  ScatterArgs cl, pa;
  memset(&cl, 0, sizeof(cl)); memset(&pa, 0, sizeof(pa));
  int64_t h2d = 0;
  CK(pool, carve(S->stage, st, pool->ev[20], &h2d, [&](Carve& c) {
    if (nc) {
      cl.c[0] = ScatterCol{static_cast<char*>(S->pend.col[P_RESERVED]), nullptr, -1, P_SZ[P_RESERVED]};
      cl.nc = 1;
      cl.slot = c.up(cleared.data(), nc);
    }
    if (cols) {
      pa.slot = c.up(slot.data(), n);
      if (allowed) pa.c[pa.nc++] = ScatterCol{static_cast<char*>(S->pend.col[P_ALLOWED]),
                                              reinterpret_cast<const char*>(c.up(allowed, n)), 1, 1};
      if (plugin_accept) pa.c[pa.nc++] = ScatterCol{static_cast<char*>(S->pend.col[P_PLUGIN]),
                                                    reinterpret_cast<const char*>(c.up(plugin_accept, n)), 1, 1};
      if (reserved_host) pa.c[pa.nc++] = ScatterCol{static_cast<char*>(S->pend.col[P_RESERVED]),
                                                    reinterpret_cast<const char*>(c.up(reserved_host, n)), -1, 4};
    }
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int nl = 0;
  scatter(cl, S->pend, nc, 0, -1, nullptr, st, &nl);
  scatter(pa, S->pend, cols ? n : 0, 0, -1, nullptr, st, &nl);
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_STATE, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[22], h2d, 0, nl);
  return COOK_OK;
}

// ---- the two running-side pipelines.  Each lists its scratch on a carve (take), writes into device
// destinations its caller sets (a standalone call's download buffers, or the columns a match or rebalance
// plan carved) and launches its kernels on the stream (run).  cook_state_usage and cook_state_cotasks are
// these plus their uploads and downloads; a derived match or rebalance runs the same kernels into its plan.

// hostname code -> index h of the code in d_codes[0, H), -1 for a code not listed (n_codes: one past the largest)
cudaError_t map_hosts(int32_t* host_of, int32_t n_codes, const int32_t* d_codes, int H, cudaStream_t st, int* nl) {
  const cudaError_t e = cudaMemsetAsync(host_of, 0xff, sizeof(int32_t) * (size_t)n_codes, st);
  if (e != cudaSuccess) return e;
  host_map_kernel<<<(H + 255) / 256, 256, 0, st>>>(d_codes, H, host_of);
  (*nl)++;
  return cudaGetLastError();
}

// The running usage of R live rows, each sum a left fold in ascending task id: per user (U > 0), per listed host
// (H > 0) and of the pool.  The caller sets rows.host_of / rows.n_codes (H > 0) and the destinations
// a.user_out [4][U], a.host_cpus / host_mem / host_count [H] and a.pool_out [4] of the sums it asked for.
struct UsageFold {
  int R = 0, U = 0, H = 0;
  bool pool = false;
  UsageRows rows = {};
  UsageArgs a = {};
  int32_t *blk = nullptr, *tmp = nullptr;
  GridFlag* gf = nullptr;

  void take(Carve& c, int hw) {
    rows.user = c.take<int32_t>(R); rows.tid = c.take<int64_t>(R);
    for (int k = 0; k < 3; k++) rows.amt[k] = c.take<double>(R);
    blk = c.take<int32_t>((size_t)hw / CP_BLOCK + 2);
    tmp = c.take<int32_t>(R);
    gf = c.take<GridFlag>(1);
    const auto segs = [&](UsageSegs& q, int n_seg, bool bounds) {
      q.n = n_seg;
      q.ord = c.take<int32_t>(R);
      if (!bounds) return;
      q.start = c.take<int32_t>(n_seg + 1); q.end = c.take<int32_t>(n_seg + 1);
      q.scan = 1;
      for (int k = 0; k < 3; k++) {
        q.os.part[k] = c.take<double>(R);
        q.os.tile[k] = c.take<double>(R / OS_TILE + 2);
      }
    };
    if (U > 0) segs(a.seg[US_USER], U, true);
    if (H > 0) {
      rows.host = c.take<int32_t>(R);
      segs(a.seg[US_HOST], H, true);
    }
    if (pool) segs(a.seg[US_POOL], 1, false);
  }

  // the live rows, the grid check, the orders with their segments and (on the grid) order-wide scans, the folds
  cudaError_t run(const PoolState* S, cudaStream_t st, int* nl) {
    rows.col = S->run.d_col; rows.H = H;
    cudaError_t e = cudaMemsetAsync(gf, 0, sizeof(GridFlag), st);
    if (e != cudaSuccess) return e;
    compact(rows, S->run.hw, nullptr, blk, S->counters, R, st, nl);
    grid_check_kernel<<<(R + 255) / 256, 256, 0, st>>>(rows.amt[0], rows.amt[1], rows.amt[2], R, gf);
    (*nl)++;
    const int32_t* key[US_N] = {rows.user, rows.host, nullptr};
    for (int k = 0; k < US_N; k++) {
      UsageSegs& q = a.seg[k];
      if (!q.n) continue;
      if ((e = csort::sort_indices(writable(q.ord), tmp, R, LessKeyTid{key[k], rows.tid}, st, nl)) != cudaSuccess) return e;
      if (!q.start) continue;
      // +1: the hosts' segment H holds the rows no listed host carries
      if ((e = cudaMemsetAsync(writable(q.start), 0, sizeof(int32_t) * (q.n + 1), st)) != cudaSuccess) return e;
      if ((e = cudaMemsetAsync(writable(q.end), 0, sizeof(int32_t) * (q.n + 1), st)) != cudaSuccess) return e;
      seg_bounds_kernel<<<(R + 255) / 256, 256, 0, st>>>(SortedKey{q.ord, nullptr, key[k]}, R, writable(q.start),
                                                         writable(q.end), nullptr);
      (*nl)++;
      order_scan(q.os, LoadSorted{q.ord, {rows.amt[0], rows.amt[1], rows.amt[2]}}, R, gf, st, nl);
    }
    // the pool's total from an order-wide scan when there is one (the sum is the same over any order there)
    if (a.seg[US_POOL].n) {
      for (int k : {US_USER, US_HOST})
        if (a.seg[k].scan && !a.seg[US_POOL].scan) { a.seg[US_POOL].os = a.seg[k].os; a.seg[US_POOL].scan = 1; }
    }
    for (int k = 0; k < 3; k++) a.amt[k] = rows.amt[k];
    a.gf = gf; a.R = R; a.U = U;
    const int nseg = a.seg[US_USER].n + a.seg[US_HOST].n + a.seg[US_POOL].n;
    usage_fold_kernel<<<(nseg + 3) / 4, 128, 0, st>>>(a);
    (*nl)++;
    return cudaGetLastError();
  }
};

// Each group's running cotasks: the K live running rows with a known host and a group list, expanded into their N
// entries and ordered by (group, task id).  The caller sets a.host_of / a.n_codes (null: no host listed), a.gcol
// [G] (a group's column of a.attr, or -1), a.attr [columns][a.H] and the destinations off [G + 1], o_host and
// o_attr [N].
struct CotaskList {
  int K = 0, N = 0, G = 0;
  CotaskArgs a = {};
  int32_t *blk = nullptr, *ord = nullptr, *tmp = nullptr;
  int32_t *off = nullptr, *o_host = nullptr, *o_attr = nullptr;

  void take(Carve& c, int hw) {
    a.slot = c.take<int32_t>(K);
    blk = c.take<int32_t>((size_t)hw / CP_BLOCK + 2);
    a.os.part[0] = c.take<int32_t>(K);
    a.os.tile[0] = c.take<int32_t>((K + OS_TILE - 1) / OS_TILE + 1);
    a.e_grp = c.take<int32_t>(N); a.e_tid = c.take<int64_t>(N); a.e_host = c.take<int32_t>(N);
    a.e_attr = c.take<int32_t>(N);
    ord = c.take<int32_t>(N); tmp = c.take<int32_t>(N);
  }

  // the rows, their entries, the (group, task id) order, the outputs
  cudaError_t run(const PoolState* S, cudaStream_t st, int* nl) {
    a.K = K;
    a.goff = S->run.at<int32_t>(R_GOFF); a.glen = S->run.at<int32_t>(R_GLEN); a.arena = S->lists[L_RGROUP].v[0];
    a.host = S->run.at<int32_t>(R_HOST); a.tid = S->run.at<int64_t>(R_TID);
    compact(CotaskRows{S->run.at<uint8_t>(R_LIVE), a.host, a.glen, writable(a.slot)}, S->run.hw, nullptr, blk,
            S->counters + 3, K, st, nl);
    order_scan(a.os, RowLen{a.slot, a.glen}, K, S->gf0, st, nl);
    cotask_expand_kernel<<<(K + 255) / 256, 256, 0, st>>>(a);
    (*nl)++;
    const cudaError_t e = csort::sort_indices(ord, tmp, N, LessKeyTid{a.e_grp, a.e_tid}, st, nl);
    if (e != cudaSuccess) return e;
    const int np = std::max(N, G + 1);
    cotask_out_kernel<<<(np + 255) / 256, 256, 0, st>>>(ord, a.e_grp, a.e_host, a.e_attr, N, G, off, o_host, o_attr);
    (*nl)++;
    return cudaGetLastError();
  }
};

// the running usage per user, of the pool and per listed host, each a left fold in ascending task id
int32_t usage(cook_pool* pool, PoolState* S, int U, double* out_user, double* out_pool, int H, const int32_t* hostname_id,
              double* out_run_cpus, double* out_run_mem, int32_t* out_run_count) {
  // ---- every check before any device work: the rows' codes from the host-side counts, the list itself
  if (out_user && count_max(S->users_r) >= U)
    return set_err(pool, COOK_E_BADARG, "cook_state_usage: a live running row's user code is >= n_users");
  if (H < 0) return set_err(pool, COOK_E_BADARG, "cook_state_usage: n_hosts < 0");
  if (H > 0 && !hostname_id) return set_err(pool, COOK_E_BADARG, "cook_state_usage: null hostname_id");
  int32_t n_codes = 0;
  if (!host_codes(hostname_id, H, &n_codes))
    return set_err(pool, COOK_E_BADARG, "cook_state_usage: a hostname_id is negative or twice in the list");
  const int R = (int)S->run.slot_of.size();
  const bool users = out_user && U > 0, hosts = H > 0 && (out_run_cpus || out_run_mem || out_run_count);
  if (R == 0) {   // nothing live: every sum is the empty fold
    if (users) memset(out_user, 0, sizeof(double) * 4 * (size_t)U);
    if (out_pool) memset(out_pool, 0, sizeof(double) * 4);
    if (out_run_cpus) memset(out_run_cpus, 0, sizeof(double) * (size_t)H);
    if (out_run_mem) memset(out_run_mem, 0, sizeof(double) * (size_t)H);
    if (out_run_count) memset(out_run_count, 0, sizeof(int32_t) * (size_t)H);
    pool->phase[COOK_PHASE_USAGE] = cook_phase_stats{};
    return COOK_OK;
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  UsageFold f;
  f.R = R; f.U = users ? U : 0; f.H = hosts ? H : 0; f.pool = out_pool != nullptr;
  UsageArgs& a = f.a;
  int32_t *d_codes = nullptr, *host_of = nullptr;
  int64_t h2d = 0, d2h = 0;
  CK(pool, carve(S->scratch, st, pool->ev[20], &h2d, [&](Carve& c) {
    f.take(c, S->run.hw);
    if (users) a.user_out = c.take<double>(4 * (size_t)U);
    if (hosts) {
      host_of = c.take<int32_t>(n_codes);
      a.host_cpus = c.take<double>(H); a.host_mem = c.take<double>(H); a.host_count = c.take<int32_t>(H);
    }
    if (out_pool) a.pool_out = c.take<double>(4);
    if (H > 0) d_codes = c.up(hostname_id, H);
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int nl = 0;
  if (hosts) {
    CK(pool, map_hosts(host_of, n_codes, d_codes, H, st, &nl));
    f.rows.host_of = host_of; f.rows.n_codes = n_codes;
  }
  CK(pool, f.run(S, st, &nl));
  CK(pool, cudaEventRecord(pool->ev[22], st));
  if (users) CK(pool, download(out_user, a.user_out, 4 * (size_t)U, st, &d2h));
  if (out_pool) CK(pool, download(out_pool, a.pool_out, 4, st, &d2h));
  if (hosts) {
    if (out_run_cpus) CK(pool, download(out_run_cpus, a.host_cpus, H, st, &d2h));
    if (out_run_mem) CK(pool, download(out_run_mem, a.host_mem, H, st, &d2h));
    if (out_run_count) CK(pool, download(out_run_count, a.host_count, H, st, &d2h));
  }
  CK(pool, cudaEventRecord(pool->ev[23], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_USAGE, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[23], h2d, d2h, nl);
  return COOK_OK;
}

// each group's running cotasks (cook_groups.cot_*): the live running rows with a known host, by (group, task id)
int32_t cotasks(cook_pool* pool, PoolState* S, int G, const int32_t* attr_col, const cook_host_table* hosts, int cap,
                int32_t* out_off, int32_t* out_host, int32_t* out_attr, int32_t* out_n) {
  // ---- every check before any device work or output: the rows' codes and the size from the host-side counts
  const bool query = !out_host;
  if (!out_n || (!query && (!out_off || !out_attr)))
    return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: null output");
  if (G < 0) return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: n_groups < 0");
  if (S && count_max(S->groups_r) >= G)
    return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: a live running row's group code is >= n_groups");
  const int H = hosts ? hosts->n : 0;
  if (H < 0) return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: hosts->n < 0");
  if (H > 0 && !hosts->hostname_id) return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: null hosts->hostname_id");
  int32_t n_codes = 0;
  if (!host_codes(H > 0 ? hosts->hostname_id : nullptr, H, &n_codes))
    return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: a hostname_id is negative or twice in `hosts`");
  // the distinct attribute columns the groups name, in first-named order; gcol[g]: the group's among them
  std::vector<int32_t> gcol(G, -1), cols;
  if (hosts && attr_col) {
    std::vector<int32_t> at(std::max(hosts->n_attr_cols, 0), -1);
    for (int g = 0; g < G; g++) {
      const int32_t c = attr_col[g];
      if (c < -1 || c >= hosts->n_attr_cols)
        return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: attr_col outside [-1, hosts->n_attr_cols)");
      if (c < 0 || H == 0) continue;
      if (at[c] < 0) { at[c] = (int32_t)cols.size(); cols.push_back(c); }
      gcol[g] = at[c];
    }
    if (!cols.empty() && !hosts->attr) return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: null hosts->attr");
  }
  const int64_t N = S ? S->cot_n : 0;
  if (N > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "cook_state_cotasks: more than 2^31 - 1 entries");
  if (!query && cap < N) return set_err(pool, COOK_E_BADARG, "cook_state_cotasks: cap < the required size");
  *out_n = (int32_t)N;
  if (query || N == 0) {   // no device work
    if (!query) memset(out_off, 0, sizeof(int32_t) * ((size_t)G + 1));
    pool->phase[COOK_PHASE_COTASKS] = cook_phase_stats{};
    return COOK_OK;
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  const int D = (int)cols.size();
  CotaskList l;
  l.K = (int)S->cot_rows; l.N = (int)N; l.G = G;
  l.a.H = H; l.a.n_codes = n_codes;
  int32_t *host_of = nullptr, *attr = nullptr;
  const int32_t* d_codes = nullptr;
  int64_t h2d = 0, d2h = 0;
  CK(pool, carve(S->scratch, st, pool->ev[20], &h2d, [&](Carve& c) {
    l.take(c, S->run.hw);
    l.off = c.take<int32_t>((size_t)G + 1); l.o_host = c.take<int32_t>(N); l.o_attr = c.take<int32_t>(N);
    if (H > 0) {
      d_codes = c.up(hosts->hostname_id, H);
      host_of = c.take<int32_t>(n_codes);
    }
    if (D) {
      attr = c.take<int32_t>((size_t)D * H);
      if (attr)
        for (int j = 0; j < D; j++) c.copy(attr + (size_t)j * H, hosts->attr + (size_t)cols[j] * H, H);
    }
    l.a.gcol = c.up(gcol.data(), G);
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  l.a.host_of = host_of; l.a.attr = attr;
  int nl = 0;
  if (H > 0) CK(pool, map_hosts(host_of, n_codes, d_codes, H, st, &nl));
  CK(pool, l.run(S, st, &nl));
  CK(pool, cudaEventRecord(pool->ev[22], st));
  CK(pool, download(out_off, l.off, (size_t)G + 1, st, &d2h));
  CK(pool, download(out_host, l.o_host, (size_t)N, st, &d2h));
  CK(pool, download(out_attr, l.o_attr, (size_t)N, st, &d2h));
  CK(pool, cudaEventRecord(pool->ev[23], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_COTASKS, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[23], h2d, d2h, nl);
  return COOK_OK;
}

// ---- a derived match or rebalance: the running-side columns its plan carved, filled on the device.  The scratch
// comes from the state's `derive` arena: `scratch` still holds the queue rows and maps the call carved before
// its build.

// A group's column of the plan's attribute matrix: the plan's copy of groups->attr_col, or (none given) a column
// of -1 in `derive_gcol`, which the caller carved.
cudaError_t group_cols(const int32_t* plan_gcol, int32_t* derive_gcol, int G, cudaStream_t st, const int32_t** gcol) {
  *gcol = plan_gcol;
  if (plan_gcol) return cudaSuccess;
  *gcol = derive_gcol;
  return cudaMemsetAsync(derive_gcol, 0xff, sizeof(int32_t) * (size_t)G, st);
}

// The users' usage [4][U], the offers' run_* [O] at their input index (n_codes: one past the largest offer
// hostname code) and, when the plan reads the lists (rows.cot_off), the groups' cot_* lists.  No live running
// row: zeros, without a kernel.
int32_t derive_match(cook_pool* pool, PoolState* S, const MatchRows& rows, int U, int O, int32_t n_codes, int G,
                     const int32_t* attr_col, int* nl) {
  cudaStream_t st = pool->stream;
  const int R = (int)S->run.slot_of.size();
  const bool lists = rows.cot_off != nullptr, entries = lists && S->cot_n > 0;
  if (R == 0 || !entries) {
    if (lists) CK(pool, cudaMemsetAsync(rows.cot_off, 0, sizeof(int32_t) * ((size_t)G + 1), st));
  }
  if (R == 0) {
    CK(pool, cudaMemsetAsync(rows.usage, 0, sizeof(double) * 4 * (size_t)U, st));
    if (O > 0) {
      CK(pool, cudaMemsetAsync(rows.run_cpus, 0, sizeof(double) * (size_t)O, st));
      CK(pool, cudaMemsetAsync(rows.run_mem, 0, sizeof(double) * (size_t)O, st));
      CK(pool, cudaMemsetAsync(rows.run_count, 0, sizeof(int32_t) * (size_t)O, st));
    }
    return COOK_OK;
  }
  UsageFold f;
  f.R = R; f.U = U; f.H = O;
  CotaskList l;
  l.K = (int)S->cot_rows; l.N = (int)S->cot_n; l.G = G;
  int32_t *host_of = nullptr, *gcol = nullptr;
  CK(pool, carve(S->derive, st, nullptr, nullptr, [&](Carve& c) {
    f.take(c, S->run.hw);
    if (O > 0) host_of = c.take<int32_t>(n_codes);
    if (entries) {
      l.take(c, S->run.hw);
      if (!attr_col) gcol = c.take<int32_t>(G);
    }
  }));
  if (O > 0) {
    CK(pool, map_hosts(host_of, n_codes, rows.hostname_id, O, st, nl));
    f.rows.host_of = host_of; f.rows.n_codes = n_codes;
  }
  f.a.user_out = rows.usage;
  f.a.host_cpus = rows.run_cpus; f.a.host_mem = rows.run_mem; f.a.host_count = rows.run_count;
  CK(pool, f.run(S, st, nl));
  if (!entries) return COOK_OK;
  l.a.host_of = O > 0 ? host_of : nullptr; l.a.n_codes = n_codes;
  l.a.attr = rows.attr; l.a.H = O;
  CK(pool, group_cols(rows.gcol, gcol, G, st, &l.a.gcol));
  l.off = rows.cot_off; l.o_host = rows.cot_host; l.o_attr = rows.cot_attr;
  CK(pool, l.run(S, st, nl));
  return COOK_OK;
}

// The groups' cot_* lists of a rebalance (rows.cot_off: the plan reads them) over its host table, through the
// host_of map the rebalance built from it (n_codes: one past the largest code of the table).
int32_t derive_rebalance(cook_pool* pool, PoolState* S, const RebRows& rows, const int32_t* host_of, int32_t n_codes,
                         int H, int G, const int32_t* attr_col, int* nl) {
  cudaStream_t st = pool->stream;
  if (!rows.cot_off) return COOK_OK;
  if (S->cot_n == 0) {
    CK(pool, cudaMemsetAsync(rows.cot_off, 0, sizeof(int32_t) * ((size_t)G + 1), st));
    return COOK_OK;
  }
  CotaskList l;
  l.K = (int)S->cot_rows; l.N = (int)S->cot_n; l.G = G;
  int32_t* gcol = nullptr;
  CK(pool, carve(S->derive, st, nullptr, nullptr, [&](Carve& c) {
    l.take(c, S->run.hw);
    if (!attr_col) gcol = c.take<int32_t>(G);
  }));
  l.a.host_of = host_of; l.a.n_codes = n_codes;
  l.a.attr = rows.attr; l.a.H = H;
  CK(pool, group_cols(rows.gcol, gcol, G, st, &l.a.gcol));
  l.off = rows.cot_off; l.o_host = rows.cot_host; l.o_attr = rows.cot_attr;
  CK(pool, l.run(S, st, nl));
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_apply(cook_pool* pool, const cook_state_delta* delta) {
  if (!pool) return COOK_E_BADARG;
  if (!delta) return set_err(pool, COOK_E_BADARG, "cook_state_apply: null argument");
  CK(pool, cudaSetDevice(pool->device));
  PoolState* S = state_of(pool, true);
  if (!S) return set_err(pool, COOK_E_OOM, "cook_state_apply: out of device memory");
  return apply(pool, S, delta);
}

extern "C" int32_t cook_state_launch(cook_pool* pool, int32_t n, const int64_t* job_id, const int64_t* task_id,
                                     const int64_t* start_time, const int32_t* hostname_id) {
  if (!pool) return COOK_E_BADARG;
  CK(pool, cudaSetDevice(pool->device));
  PoolState* S = state_of(pool, true);
  if (!S) return set_err(pool, COOK_E_OOM, "cook_state_launch: out of device memory");
  return launch(pool, S, n, job_id, task_id, start_time, hostname_id);
}

extern "C" int32_t cook_state_patch(cook_pool* pool, int32_t n, const int64_t* job_id, const uint8_t* allowed,
                                    const uint8_t* plugin_accept, const int32_t* reserved_host,
                                    int32_t clear_reservations) {
  if (!pool) return COOK_E_BADARG;
  CK(pool, cudaSetDevice(pool->device));
  PoolState* S = state_of(pool, true);
  if (!S) return set_err(pool, COOK_E_OOM, "cook_state_patch: out of device memory");
  return patch(pool, S, n, job_id, allowed, plugin_accept, reserved_host, clear_reservations != 0);
}

extern "C" int32_t cook_state_usage(cook_pool* pool, int32_t n_users, double* out_user_usage, double* out_pool_usage,
                                    int32_t n_hosts, const int32_t* hostname_id, double* out_run_cpus,
                                    double* out_run_mem, int32_t* out_run_count) {
  if (!pool) return COOK_E_BADARG;
  CK(pool, cudaSetDevice(pool->device));
  PoolState* S = state_of(pool, true);
  if (!S) return set_err(pool, COOK_E_OOM, "cook_state_usage: out of device memory");
  return usage(pool, S, n_users, out_user_usage, out_pool_usage, n_hosts, hostname_id, out_run_cpus, out_run_mem,
               out_run_count);
}

extern "C" int32_t cook_state_cotasks(cook_pool* pool, int32_t n_groups, const int32_t* attr_col,
                                      const cook_host_table* hosts, int32_t cap, int32_t* out_cot_off,
                                      int32_t* out_cot_hostname_id, int32_t* out_cot_attr_val, int32_t* out_n) {
  if (!pool) return COOK_E_BADARG;
  return cotasks(pool, static_cast<PoolState*>(pool->state), n_groups, attr_col, hosts, cap, out_cot_off,
                 out_cot_hostname_id, out_cot_attr_val, out_n);
}

namespace {

// cook_state_rank, and with `offensive` cook_state_rank_offensive: the jobs the rank drops as offensive, as job ids
int32_t state_rank(cook_pool* pool, const char* who, bool offensive, const cook_user_table* users,
                   const cook_pool_quota* pool_quota, const cook_pool_quota* group_quota, const double* group_usage,
                   const cook_rank_params* params, int64_t* out_ranked_job_id, int32_t* out_n, int64_t* out_off,
                   int32_t off_cap, int32_t* out_n_off) {
  if (!pool) return COOK_E_BADARG;
  if (!users || !params || !out_n || (offensive && (!out_off || !out_n_off)))
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  *out_n = 0;
  if (offensive) *out_n_off = 0;
  CK(pool, cudaSetDevice(pool->device));
  PoolState* S = state_of(pool, true);
  if (!S) return set_err(pool, COOK_E_OOM, "%s: out of device memory", who);
  const int U = users->n_users;
  if (U <= 0) return set_err(pool, COOK_E_BADARG, "%s: bad sizes", who);
  if (std::max(count_max(S->users_p), count_max(S->users_r)) >= U)
    return set_err(pool, COOK_E_BADARG, "%s: a resident row's user code is >= n_users", who);
  if (offensive && (int64_t)off_cap < (int64_t)S->pend.slot_of.size())
    return set_err(pool, COOK_E_BADARG, "%s: offensive_cap < the live pending rows", who);
  cudaStream_t st = pool->stream;
  const int R = (int)S->run.slot_of.size(), J = (int)S->pend.slot_of.size();
  const size_t N = (size_t)R + J;
  S->ranked = false;
  CK(pool, cudaEventRecord(pool->ev[7], st));
  int nl = 0;
  TaskCols dt = {};
  int32_t* pslot = nullptr;
  if (N > 0) {
    int32_t* blk = nullptr;
    CK(pool, carve(S->scratch, st, nullptr, nullptr, [&](Carve& c) {
      dt.user = c.take<int32_t>(N); dt.prio = c.take<int32_t>(N);
      dt.start = c.take<int64_t>(N); dt.tid = c.take<int64_t>(N); dt.jid = c.take<int64_t>(N);
      dt.cpus = c.take<double>(N); dt.mem = c.take<double>(N); dt.gpus = c.take<double>(N);
      pslot = c.take<int32_t>(J);
      blk = c.take<int32_t>((size_t)std::max(S->pend.hw, S->run.hw) / CP_BLOCK + 2);
    }));
    if (R) compact(RunningRows{S->run.d_col, dt}, S->run.hw, nullptr, blk, S->counters, R, st, &nl);
    if (J) compact(PendingRows{S->pend.d_col, dt, pslot, R}, S->pend.hw, nullptr, blk, S->counters + 1, J, st, &nl);
    CK(pool, cudaGetLastError());
    CK(pool, cudaEventRecord(pool->ev[23], st));
  }
  int32_t n = 0;
  RankQueue rq = {};
  const RankOffensive ro{pslot, S->pend.at<int64_t>(P_JID), out_off, out_n_off};
  const int32_t rc = rank_impl(pool, R, J, nullptr, nullptr, &dt, users, pool_quota, group_quota, group_usage, params,
                               nullptr, &n, nullptr, nullptr, nullptr, &rq, offensive ? &ro : nullptr);
  if (rc != COOK_OK) return rc;
  cook_phase_stats& ps = pool->phase[COOK_PHASE_RANK];
  if (N > 0) ps.ms_device += ev_ms(pool->ev[7], pool->ev[23]);   // the gathering of the live rows
  if (J > 0) {   // the ranked list as (slot, generation) pairs, while it is still in the pool's arena
    int32_t* q_slot = nullptr; uint32_t* q_gen = nullptr; int64_t* q_jid = nullptr;
    CK(pool, carve(S->queue, st, nullptr, nullptr, [&](Carve& c) {
      q_slot = c.take<int32_t>(J + 1); q_gen = c.take<uint32_t>(J + 1); q_jid = c.take<int64_t>(J + 1);
    }));
    S->q_slot = q_slot; S->q_gen = q_gen; S->q_jid = q_jid;
    CK(pool, cudaEventRecord(pool->ev[7], st));
    queue_kernel<<<(J + 255) / 256, 256, 0, st>>>(rq.ranked, rq.n, pslot, S->pend.at<uint32_t>(P_GEN),
                                                  S->pend.at<int64_t>(P_JID), q_slot, q_gen, q_jid);
    nl++;
    CK(pool, cudaGetLastError());
    CK(pool, cudaEventRecord(pool->ev[23], st));
    if (out_ranked_job_id && n > 0) {
      int64_t d2h = 0;
      CK(pool, download(out_ranked_job_id, S->q_jid, n, st, &d2h));
      ps.d2h_bytes += d2h;
    }
    CK(pool, cudaStreamSynchronize(st));
    ps.ms_device += ev_ms(pool->ev[7], pool->ev[23]);
  }
  ps.n_launches += nl;
  S->n_q = n;
  S->ranked = true;
  *out_n = n;
  return COOK_OK;
}

// cook_state_match, and with `derived` cook_state_match_derived: the users' usage, the offers' run_* and the
// groups' cot_* lists come from the live running rows, filled on the device into the columns the plan carved
int32_t state_match(cook_pool* pool, const char* who, bool derived, const cook_offers_soa* offers,
                    const cook_groups* groups, const cook_user_table* users, const cook_pool_quota* pool_quota,
                    const cook_match_params* params, int64_t* out_considerable_job_id, int32_t* out_assign,
                    int32_t* out_ports, int32_t max_ports, uint8_t* out_fail_reason, cook_match_stats* out_stats) {
  if (!pool) return COOK_E_BADARG;
  if (!offers || !users || !params || !out_considerable_job_id || !out_assign)
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (params->reuse_resident)
    return set_err(pool, COOK_E_BADARG, "%s: reuse_resident does not apply: the queue's rows are resident", who);
  PoolState* S = static_cast<PoolState*>(pool->state);
  const int NC = params->num_considerable;
  cudaStream_t st = pool->stream;
  // ---- the queue minus what left it since the rank.  This comes first: as in cook_match, the offer and
  // group tables are checked only when some row is left to match.
  int nl = 0;
  int32_t n = 0;
  int64_t d2h = 0;
  int32_t* m_slot = nullptr;
  OrderScan<int, 1> os;
  if (S && S->ranked && S->n_q > 0 && NC > 0) {
    CK(pool, cudaSetDevice(pool->device));
    const int nq = S->n_q;
    int32_t* blk = nullptr;
    CK(pool, carve(S->scratch, st, nullptr, nullptr, [&](Carve& c) {
      m_slot = c.take<int32_t>(nq);
      blk = c.take<int32_t>((size_t)nq / CP_BLOCK + 2);
      os.part[0] = c.take<int32_t>(nq);
      os.tile[0] = c.take<int32_t>((nq + OS_TILE - 1) / OS_TILE + 1);
    }));
    const QueueLive ql{S->q_slot, S->q_gen, S->pend.at<uint8_t>(P_LIVE), S->pend.at<uint32_t>(P_GEN), m_slot};
    compact(ql, nq, nullptr, blk, S->counters + 2, nq, st, &nl);
    CK(pool, cudaGetLastError());
    CK(pool, download(&n, S->counters + 2, 1, st, &d2h));
    CK(pool, cudaStreamSynchronize(st));
  }
  int32_t rc = check_match_inputs(pool, who, offers, groups, users, params, max_ports, n > 0,
                                  S && S->lists[L_NOVEL].live > 0, S && S->lists[L_GROUP].live > 0, derived);
  if (rc != COOK_OK) return rc;
  if (!S || !S->ranked) return set_err(pool, COOK_E_BADARG, "%s: no cook_state_rank on this handle yet", who);
  const int U = users->n_users;
  if (count_max(S->users_p) >= U) return set_err(pool, COOK_E_BADARG, "%s: a pending row's user code is >= n_users", who);
  if (count_max(S->attr_cols) >= std::max(1, offers->n_attr_cols))
    return set_err(pool, COOK_E_BADARG, "%s: a pending row's attribute column is >= n_attr_cols", who);
  const int G = groups ? groups->n_groups : 0;
  if (G > 0 && count_max(S->groups) >= G)
    return set_err(pool, COOK_E_BADARG, "%s: a pending row's group code is >= n_groups", who);
  // ---- what the derivation reads, checked from the host-side counts and the offer and group tables
  const int O = offers->n;
  int32_t n_codes = 0;
  if (derived) {
    if (count_max(S->users_r) >= U)
      return set_err(pool, COOK_E_BADARG, "%s: a live running row's user code is >= n_users", who);
    if (n > 0) {
      if (O > 0 && !offers->hostname_id) return set_err(pool, COOK_E_BADARG, "%s: null offers->hostname_id", who);
      if (!host_codes(offers->hostname_id, O, &n_codes))
        return set_err(pool, COOK_E_BADARG, "%s: an offers->hostname_id is negative or twice in the table", who);
      if (G > 0) {
        if (count_max(S->groups_r) >= G)
          return set_err(pool, COOK_E_BADARG, "%s: a live running row's group code is >= n_groups", who);
        bool named = false;
        for (int g = 0; groups->attr_col && g < G; g++) {
          const int32_t c = groups->attr_col[g];
          if (c < -1 || c >= offers->n_attr_cols)
            return set_err(pool, COOK_E_BADARG, "%s: groups->attr_col outside [-1, offers->n_attr_cols)", who);
          named = named || c >= 0;
        }
        if (named && O > 0 && !offers->attr) return set_err(pool, COOK_E_BADARG, "%s: null offers->attr", who);
        if (S->cot_n > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 cotask entries", who);
      }
    }
  }
  if (out_stats) memset(out_stats, 0, sizeof(*out_stats));
  if (n == 0) return COOK_OK;
  // ---- what the rows hold, from the host-side counts: the resident columns of the kinds some live row
  // holds a non-absent value of
  JobShape sh;
  sh.J = n;
  sh.job_ids = true;
  const Table& P = S->pend;
  const ListArena* L = S->lists;
  const auto has = [&](int f) { return S->nflag[f] > 0; };
  JobDev& c = sh.cols;
  c.user = P.at<int32_t>(P_USER); c.cpus = P.at<double>(P_CPUS); c.mem = P.at<double>(P_MEM);
  c.gpus = P.at<double>(P_GPUS);
  if (has(F_PORTS)) c.ports = P.at<int32_t>(P_PORTS);
  if (has(F_NOT_ALLOWED)) c.allowed = P.at<uint8_t>(P_ALLOWED);
  if (has(F_NOT_PLUGIN)) c.plugin = P.at<uint8_t>(P_PLUGIN);
  if (L[L_NOVEL].live) { c.novel_off = P.at<int32_t>(P_NOFF); c.novel_host = L[L_NOVEL].v[0]; }
  if (has(F_GPU_MODEL)) c.gpu_model = P.at<int32_t>(P_GPU_MODEL);
  if (has(F_DISK)) { c.disk_request = P.at<double>(P_DISK_REQ); c.disk_type = P.at<int32_t>(P_DISK_TYPE); }
  if (L[L_ATTR].live) { c.attr_off = P.at<int32_t>(P_AOFF); c.attr_col = L[L_ATTR].v[0]; c.attr_val = L[L_ATTR].v[1]; }
  if (has(F_EST)) c.est_end_ms = P.at<int64_t>(P_EST);
  if (has(F_CKPT)) c.ckpt_location = P.at<int32_t>(P_CKPT);
  if (has(F_RESERVED)) c.reserved_host = P.at<int32_t>(P_RESERVED);
  if (L[L_GROUP].live) { c.group_off = P.at<int32_t>(P_GOFF); c.group_idx = L[L_GROUP].v[0]; }
  sh.n_novel = L[L_NOVEL].live; sh.n_attr = L[L_ATTR].live; sh.n_group = L[L_GROUP].live;
  sh.gp_off.assign(G + 1, 0);
  for (const auto& kv : S->groups) if (kv.first < G) sh.gp_off[kv.first + 1] = (int32_t)kv.second;
  for (int g = 0; g < G; g++) sh.gp_off[g + 1] += sh.gp_off[g];
  sh.any_gpus_ports = has(F_GPUS) || has(F_PORTS);
  sh.dev.usage = sh.dev.run = sh.dev.cot = derived;
  sh.dev.n_cot = S->cot_n;
  // ---- the plan, the gathers into the job columns it carved, the derived columns, the run
  CK(pool, cudaEventRecord(pool->ev[0], st));
  MatchRows rows;
  rc = match_build(pool, nullptr, n, sh, offers, groups, users, pool_quota, params, max_ports, &rows);
  if (rc != COOK_OK) return rc;
  fill_rows_kernel<<<(n + 255) / 256, 256, 0, st>>>(rows, S->pend.d_col, m_slot, n);
  nl++;
  gather_lists(S, rows.jb, m_slot, n, os, st, &nl);
  CK(pool, cudaGetLastError());
  if (derived) {
    rc = derive_match(pool, S, rows, U, O, n_codes, G, groups ? groups->attr_col : nullptr, &nl);
    if (rc != COOK_OK) return rc;
  }
  rc = match_run(pool, nullptr, out_considerable_job_id, out_assign, out_ports, out_fail_reason, out_stats, true,
                 params->max_ctas);
  if (rc != COOK_OK) return rc;
  cook_phase_stats& ps = pool->phase[COOK_PHASE_MATCH];
  ps.n_launches += nl;
  ps.d2h_bytes += d2h;
  if (out_stats) { out_stats->n_launches += nl; out_stats->d2h_bytes += d2h; }
  return COOK_OK;
}

// cook_state_rebalance, and with `derived` cook_state_rebalance_derived: the groups' cot_* lists come from the live
// running rows over `hosts`, filled on the device into the lists the build carved
int32_t state_rebalance(cook_pool* pool, const char* who, bool derived, const cook_host_table* hosts,
                        const cook_groups* groups, const cook_user_table* users, const cook_rebalance_params* params,
                        cook_decision* out_decisions, int64_t* out_decision_job_id, int64_t* out_victim_task_id,
                        int32_t victim_cap, int32_t* out_n) {
  if (!pool) return COOK_E_BADARG;
  if (!hosts || !users || !params || !out_decisions || !out_decision_job_id || !out_victim_task_id || !out_n)
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (pool->dru_mode != 0)
    return set_err(pool, COOK_E_UNSUPPORTED_CONSTRAINT,
                   "%s: GPU DRU mode has no reference behaviour (rebalancer.clj:339-349 throws)", who);
  PoolState* S = static_cast<PoolState*>(pool->state);
  if (!S || !S->ranked) return set_err(pool, COOK_E_BADARG, "%s: no cook_state_rank on this handle yet", who);
  *out_n = 0;
  const int H = hosts->n, MP = params->max_preemption;
  if (MP <= 0 || H <= 0) return COOK_OK;
  // ---- every check before any device work, from the host-side counts
  const int R = (int)S->run.slot_of.size();
  if ((int64_t)victim_cap < (int64_t)R + MP)
    return set_err(pool, COOK_E_BADARG, "%s: victim_cap < live running rows + max_preemption", who);
  if (!hosts->hostname_id) return set_err(pool, COOK_E_BADARG, "%s: null hosts->hostname_id", who);
  std::unordered_set<int32_t> codes;
  codes.reserve((size_t)H);
  int32_t max_code = 0;
  for (int h = 0; h < H; h++) {
    const int32_t c = hosts->hostname_id[h];
    if (c < 0 || !codes.insert(c).second)
      return set_err(pool, COOK_E_BADARG, "%s: a hostname_id is negative or twice in the host table", who);
    max_code = std::max(max_code, c);
  }
  for (const auto& kv : S->hosts_r)
    if (!codes.count(kv.first))
      return set_err(pool, COOK_E_BADARG, "%s: a running row's host is unknown or not in the host table", who);
  if (std::max(count_max(S->users_p), count_max(S->users_r)) >= users->n_users)
    return set_err(pool, COOK_E_BADARG, "%s: a resident row's user code is >= n_users", who);
  const int G = groups ? groups->n_groups : 0;
  if (groups && count_max(S->groups) >= G)
    return set_err(pool, COOK_E_BADARG, "%s: a pending row's group code is >= n_groups", who);
  if (G && S->lists[L_GROUP].live && ((!derived && !groups->cot_off) || !groups->kind))
    return set_err(pool, COOK_E_BADARG, "%s: incomplete cook_groups", who);
  if (count_max(S->attr_cols) >= std::max(1, hosts->n_attr_cols))
    return set_err(pool, COOK_E_BADARG, "%s: a pending row's attribute column is >= n_attr_cols", who);
  if (derived && G > 0) {   // what the derivation of the lists reads
    if (count_max(S->groups_r) >= G)
      return set_err(pool, COOK_E_BADARG, "%s: a live running row's group code is >= n_groups", who);
    bool named = false;
    for (int g = 0; groups->attr_col && g < G; g++) {
      const int32_t c = groups->attr_col[g];
      if (c < -1 || c >= hosts->n_attr_cols)
        return set_err(pool, COOK_E_BADARG, "%s: groups->attr_col outside [-1, hosts->n_attr_cols)", who);
      named = named || c >= 0;
    }
    if (named && !hosts->attr) return set_err(pool, COOK_E_BADARG, "%s: null hosts->attr", who);
    if (S->cot_n > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 cotask entries", who);
  }
  const int nq = S->n_q;
  if (nq == 0) return COOK_OK;
  // ---- jobs-to-make-room-for: the first allowed jobs of the live queue, their count downloaded
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  const int PM = std::min(MP, nq);
  int nl = 0;
  int64_t d2h = 0;
  int32_t *m_slot = nullptr, *blk = nullptr, *host_of = nullptr;
  OrderScan<int, 1> os;
  CK(pool, carve(S->scratch, st, nullptr, nullptr, [&](Carve& c) {
    m_slot = c.take<int32_t>(PM);
    blk = c.take<int32_t>((size_t)std::max(nq, S->run.hw) / CP_BLOCK + 2);
    host_of = c.take<int32_t>((size_t)max_code + 1);
    os.part[0] = c.take<int32_t>(PM);
    os.tile[0] = c.take<int32_t>((PM + OS_TILE - 1) / OS_TILE + 1);
  }));
  CK(pool, cudaEventRecord(pool->ev[20], st));
  const QueueLive ql{S->q_slot, S->q_gen, S->pend.at<uint8_t>(P_LIVE), S->pend.at<uint32_t>(P_GEN), m_slot};
  compact(QueueAllowed{ql, S->pend.at<uint8_t>(P_ALLOWED)}, nq, nullptr, blk, S->counters + 2, PM, st, &nl);
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int32_t P = 0;
  CK(pool, download(&P, S->counters + 2, 1, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  if (P == 0) return COOK_OK;
  // ---- the build, the gathers into the rows it carved, the run
  RebShape sh;
  sh.R = R; sh.P = P;
  sh.n_novel = S->lists[L_NOVEL].live; sh.n_attr = S->lists[L_ATTR].live; sh.n_group = S->lists[L_GROUP].live;
  sh.dev.cot = derived;
  sh.dev.n_cot = S->cot_n;
  RebPlanPtr plan;
  RebRows rows;
  int32_t rc = rebalance_build(pool, sh, hosts, groups, users, params, &plan, &rows);
  if (rc != COOK_OK) return rc;
  CK(pool, cudaEventRecord(pool->ev[22], st));
  if (R > 0) {
    host_map_kernel<<<(H + 255) / 256, 256, 0, st>>>(rows.hostname_id, H, host_of);
    nl++;
    compact(RebRunningRows{RunningRows{S->run.d_col, rows.t}, writable(rows.host), host_of}, S->run.hw, nullptr, blk,
            S->counters, R, st, &nl);
  }
  reb_pending_kernel<<<(P + 255) / 256, 256, 0, st>>>(rows, S->pend.d_col, m_slot, P);
  nl++;
  gather_lists(S, rows.jb, m_slot, P, os, st, &nl);
  CK(pool, cudaGetLastError());
  if (derived) {
    rc = derive_rebalance(pool, S, rows, host_of, max_code + 1, H, G, groups ? groups->attr_col : nullptr, &nl);
    if (rc != COOK_OK) return rc;
  }
  CK(pool, cudaEventRecord(pool->ev[23], st));
  rc = rebalance_run(pool, *plan, out_decisions, out_victim_task_id, out_decision_job_id, out_n);
  if (rc != COOK_OK) return rc;
  cook_phase_stats& ps = pool->phase[COOK_PHASE_REBALANCE];
  ps.ms_device += ev_ms(pool->ev[20], pool->ev[21]) + ev_ms(pool->ev[22], pool->ev[23]);   // the gathers
  ps.n_launches += nl;
  ps.d2h_bytes += d2h;
  return COOK_OK;
}

// cook_state_considerable: M0 over the live queue, the considerable pass cook_match runs (match.cu), without a plan
int32_t considerable(cook_pool* pool, PoolState* S, const cook_user_table* users, const cook_pool_quota* pool_quota,
                     const cook_considerable_params* prm, int64_t* out_job_id, int32_t* out_n) {
  const char* who = "cook_state_considerable";
  // ---- every check before any device work or output
  if (!users || !prm || !out_job_id || !out_n) return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (!S || !S->ranked) return set_err(pool, COOK_E_BADARG, "%s: no cook_state_rank on this handle yet", who);
  const int U = users->n_users, src = prm->usage_source;
  if (U <= 0) return set_err(pool, COOK_E_BADARG, "%s: bad sizes", who);
  if (src != COOK_USAGE_GIVEN && src != COOK_USAGE_DERIVED && src != COOK_USAGE_LAST_MATCH)
    return set_err(pool, COOK_E_BADARG, "%s: unknown usage_source", who);
  const double* quota[4] = {users->quota_count, users->quota_cpus, users->quota_mem, users->quota_gpus};
  const double* given[4] = {users->usage_count, users->usage_cpus, users->usage_mem, users->usage_gpus};
  for (int k = 0; k < 4; k++)
    if (!quota[k] || (src == COOK_USAGE_GIVEN && !given[k]))
      return set_err(pool, COOK_E_BADARG, "%s: null quota or (given usage) usage column", who);
  if (count_max(S->users_p) >= U) return set_err(pool, COOK_E_BADARG, "%s: a pending row's user code is >= n_users", who);
  if (src == COOK_USAGE_DERIVED && count_max(S->users_r) >= U)
    return set_err(pool, COOK_E_BADARG, "%s: a live running row's user code is >= n_users", who);
  const double* last[4] = {};
  if (src == COOK_USAGE_LAST_MATCH && !match_last_usage(pool, U, last))
    return set_err(pool, COOK_E_BADARG, "%s: LAST_MATCH without a match on this handle for these n_users", who);
  *out_n = 0;
  const int nq = S->n_q;
  if (prm->num_considerable <= 0 || nq == 0) {
    pool->phase[COOK_PHASE_CONSIDERABLE] = cook_phase_stats{};
    return COOK_OK;
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  const bool masks = !prm->quota_only;
  const bool al = masks && S->nflag[F_NOT_ALLOWED] > 0, pl = masks && S->nflag[F_NOT_PLUGIN] > 0;
  const int R = (int)S->run.slot_of.size();
  const int NC = std::min(prm->num_considerable, nq);
  const int32_t* tokens = prm->enforce_rate_limit ? users->tokens : nullptr;
  // ---- one carve, sized by the queue: the rows, M0's scratch, the user columns (uploaded), the derived usage
  ConsRows r;
  r.n_users = U;
  int32_t *m_slot = nullptr, *qpos = nullptr, *blk = nullptr;
  int64_t* d_jid = nullptr;
  double* usage = nullptr;
  UsageFold f;
  f.R = R; f.U = U;
  const bool fold = src == COOK_USAGE_DERIVED && R > 0;
  int64_t h2d = 0, d2h = 0;
  CK(pool, carve(S->scratch, st, pool->ev[20], &h2d, [&](Carve& c) {
    m_slot = c.take<int32_t>(nq); qpos = c.take<int32_t>(nq);
    blk = c.take<int32_t>((size_t)nq / CP_BLOCK + 2);
    r.ranked = c.take<int32_t>(nq); r.user = c.take<int32_t>(nq);
    r.cpus = c.take<double>(nq); r.mem = c.take<double>(nq); r.gpus = c.take<double>(nq);
    r.allowed = al ? c.take<uint8_t>(nq) : nullptr;
    r.plugin = pl ? c.take<uint8_t>(nq) : nullptr;
    r.pos = c.take<int32_t>(nq + 1); r.tmp = c.take<int32_t>(nq + 1);
    r.seg_s = c.take<int32_t>(U + 1); r.seg_e = c.take<int32_t>(U + 1);
    r.keep = c.take<uint8_t>(nq + 1);
    r.gf = c.take<GridFlag>(1);
    r.out_row = c.take<int32_t>(NC);
    d_jid = c.take<int64_t>(NC);
    for (int k = 0; k < 4; k++) r.quota[k] = c.up(quota[k], U);
    if (tokens) r.tokens = c.up(tokens, U);
    if (src == COOK_USAGE_GIVEN) {
      for (int k = 0; k < 4; k++) r.usage[k] = c.up(given[k], U);
    } else if (src == COOK_USAGE_DERIVED) {
      usage = c.take<double>(4 * (size_t)U);
      if (fold) f.take(c, S->run.hw);
    }
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int nl = 0;
  // ---- the live queue with its positions, its length downloaded
  const QueueLive ql{S->q_slot, S->q_gen, S->pend.at<uint8_t>(P_LIVE), S->pend.at<uint32_t>(P_GEN), m_slot};
  compact(QueueLivePos{ql, qpos}, nq, nullptr, blk, S->counters + 2, nq, st, &nl);
  CK(pool, cudaGetLastError());
  int32_t n = 0;
  CK(pool, download(&n, S->counters + 2, 1, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  int32_t n_out = 0;
  if (n > 0) {
    // ---- the rows' columns, the usage, M0, the ids (and the consumption)
    cons_rows_kernel<<<(n + 255) / 256, 256, 0, st>>>(S->pend.d_col, m_slot, n, writable(r.ranked), writable(r.user),
                                                      writable(r.cpus), writable(r.mem), writable(r.gpus),
                                                      writable(r.allowed), writable(r.plugin));
    nl++;
    if (src == COOK_USAGE_DERIVED) {
      if (fold) {
        f.a.user_out = usage;
        CK(pool, f.run(S, st, &nl));
      } else {
        CK(pool, cudaMemsetAsync(usage, 0, sizeof(double) * 4 * (size_t)U, st));
      }
      for (int k = 0; k < 4; k++) r.usage[k] = usage + (size_t)k * U;
    } else if (src == COOK_USAGE_LAST_MATCH) {
      for (int k = 0; k < 4; k++) r.usage[k] = last[k];
    }
    r.n = n;
    r.enforce_rate_limit = prm->enforce_rate_limit;
    r.pool_q = pool_quota ? *pool_quota : cook_pool_quota{0, 0, 0, 0, 0};
    r.num_considerable = NC;
    r.out_n = S->counters + 4;
    CK(pool, considerable_rows(r, st, &nl));
    cons_take_kernel<<<(NC + 255) / 256, 256, 0, st>>>(r.out_row, r.out_n, qpos, S->q_jid, writable(S->q_gen),
                                                       prm->consume ? 1 : 0, d_jid);
    nl++;
    CK(pool, cudaGetLastError());
    CK(pool, cudaEventRecord(pool->ev[22], st));
    CK(pool, download(&n_out, r.out_n, 1, st, &d2h));
    CK(pool, cudaStreamSynchronize(st));
    if (n_out > 0) CK(pool, download(out_job_id, d_jid, n_out, st, &d2h));
  } else {
    CK(pool, cudaEventRecord(pool->ev[22], st));
  }
  CK(pool, cudaEventRecord(pool->ev[23], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_CONSIDERABLE, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[23], h2d, d2h, nl);
  *out_n = n_out;
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_rank(cook_pool* pool, const cook_user_table* users, const cook_pool_quota* pool_quota,
                                   const cook_pool_quota* group_quota, const double* group_usage,
                                   const cook_rank_params* params, int64_t* out_ranked_job_id, int32_t* out_n) {
  return state_rank(pool, "cook_state_rank", false, users, pool_quota, group_quota, group_usage, params,
                    out_ranked_job_id, out_n, nullptr, 0, nullptr);
}

extern "C" int32_t cook_state_rank_offensive(cook_pool* pool, const cook_user_table* users,
                                             const cook_pool_quota* pool_quota, const cook_pool_quota* group_quota,
                                             const double* group_usage, const cook_rank_params* params,
                                             int64_t* out_ranked_job_id, int32_t* out_n, int64_t* out_offensive_job_id,
                                             int32_t offensive_cap, int32_t* out_n_offensive) {
  return state_rank(pool, "cook_state_rank_offensive", true, users, pool_quota, group_quota, group_usage, params,
                    out_ranked_job_id, out_n, out_offensive_job_id, offensive_cap, out_n_offensive);
}

extern "C" int32_t cook_state_considerable(cook_pool* pool, const cook_user_table* users,
                                           const cook_pool_quota* pool_quota, const cook_considerable_params* params,
                                           int64_t* out_job_id, int32_t* out_n) {
  if (!pool) return COOK_E_BADARG;
  return considerable(pool, static_cast<PoolState*>(pool->state), users, pool_quota, params, out_job_id, out_n);
}

extern "C" int32_t cook_state_match(cook_pool* pool, const cook_offers_soa* offers, const cook_groups* groups,
                                    const cook_user_table* users, const cook_pool_quota* pool_quota,
                                    const cook_match_params* params, int64_t* out_considerable_job_id,
                                    int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                                    uint8_t* out_fail_reason, cook_match_stats* out_stats) {
  return state_match(pool, "cook_state_match", false, offers, groups, users, pool_quota, params,
                     out_considerable_job_id, out_assign, out_ports, max_ports, out_fail_reason, out_stats);
}

extern "C" int32_t cook_state_match_derived(cook_pool* pool, const cook_offers_soa* offers, const cook_groups* groups,
                                            const cook_user_table* users, const cook_pool_quota* pool_quota,
                                            const cook_match_params* params, int64_t* out_considerable_job_id,
                                            int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                                            uint8_t* out_fail_reason, cook_match_stats* out_stats) {
  return state_match(pool, "cook_state_match_derived", true, offers, groups, users, pool_quota, params,
                     out_considerable_job_id, out_assign, out_ports, max_ports, out_fail_reason, out_stats);
}

extern "C" int32_t cook_state_rebalance(cook_pool* pool, const cook_host_table* hosts, const cook_groups* groups,
                                        const cook_user_table* users, const cook_rebalance_params* params,
                                        cook_decision* out_decisions, int64_t* out_decision_job_id,
                                        int64_t* out_victim_task_id, int32_t victim_cap, int32_t* out_n) {
  return state_rebalance(pool, "cook_state_rebalance", false, hosts, groups, users, params, out_decisions,
                         out_decision_job_id, out_victim_task_id, victim_cap, out_n);
}

extern "C" int32_t cook_state_rebalance_derived(cook_pool* pool, const cook_host_table* hosts, const cook_groups* groups,
                                                const cook_user_table* users, const cook_rebalance_params* params,
                                                cook_decision* out_decisions, int64_t* out_decision_job_id,
                                                int64_t* out_victim_task_id, int32_t victim_cap, int32_t* out_n) {
  return state_rebalance(pool, "cook_state_rebalance_derived", true, hosts, groups, users, params, out_decisions,
                         out_decision_job_id, out_victim_task_id, victim_cap, out_n);
}
