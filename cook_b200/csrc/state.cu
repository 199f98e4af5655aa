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
#include <cassert>
#include <cmath>
#include <cstdlib>
#include <map>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>

#include "fold.cuh"
#include "sort.cuh"

namespace {

// ---- device tables: column k of a table is cols[k] (sz bytes per slot)
enum PCol {
  P_USER, P_PRIO, P_JID, P_CPUS, P_MEM, P_GPUS, P_PORTS, P_ALLOWED, P_PLUGIN, P_GPU_MODEL, P_DISK_REQ, P_DISK_TYPE,
  P_EST, P_CKPT, P_RESERVED, P_NDATA,   // the columns a delta row carries
  P_LIVE = P_NDATA, P_GEN, P_NOFF, P_NLEN, P_AOFF, P_ALEN, P_GOFF, P_GLEN,
  P_JF, P_JF_GPU, P_JF_DREQ, P_JF_DLIM, P_JF_DTYPE, P_LF_SUBMIT, P_LF_POOL, P_LF_EXEC, P_NCOL
};
constexpr int P_SZ[P_NCOL] = {4, 4, 8, 8, 8, 8, 4, 1, 1, 4, 8, 4, 8, 4, 4, 1, 4, 4, 4, 4, 4, 4, 4, 1, 4, 8, 8, 4, 8, 4, 1};
// P_JF .. P_JF_DTYPE are the job facts cook_state_job_facts writes (the stats keys of jobs->resource-maps): the
// COOK_JF_* bits, then the gpu model, disk request, disk limit and disk type, each read only under its bit.  Every
// pending upsert writes P_JF = 0, so the others need no reset.
// P_LF_* / R_LF_* are the list facts cook_state_list_facts writes (what /list and /jobs filter on): the submit time
// in ms, the submit pool's code (-1: none) and LF_EXEC, 0 for no facts, else 2 + :job/custom-executor (-1 nil, 0
// false, 1 true).  Every upsert writes LF_EXEC 0, so the others are read only once written; a launch copies them.
// R_MAXRT and R_FACTS are the facts cook_state_task_facts writes: the job's max-runtime (-1: none) and the
// RF_* bits; R_REASON the fact cook_state_task_reason writes: the instance's reason code (-1: none).  Every upsert
// and launch writes their absent values.
enum RCol { R_USER, R_PRIO, R_START, R_TID, R_JID, R_CPUS, R_MEM, R_GPUS, R_HOST, R_NDATA, R_LIVE = R_NDATA, R_GEN,
            R_GOFF, R_GLEN, R_MAXRT, R_FACTS, R_REASON, R_LF_SUBMIT, R_LF_POOL, R_LF_EXEC, R_NCOL };
constexpr int R_SZ[R_NCOL] = {4, 4, 8, 8, 8, 8, 8, 8, 4, 1, 4, 4, 4, 8, 1, 4, 8, 4, 1};
enum { RF_CANCELLED = 1, RF_UNKNOWN = 2 };

// The live offers (leases): one row per offer as it arrived, before any merge.  Data columns first, then the live
// flag and generation, then the (off, len) pairs of the offer's four lists.
enum OCol {
  O_CODE, O_CPUS, O_MEM, O_GPUS, O_K8S, O_LOC, O_MAXT, O_NUMT, O_START, O_SEQ, O_NDATA,
  O_LIVE = O_NDATA, O_GEN, O_POFF, O_PLEN, O_GOFF, O_GLEN, O_DOFF, O_DLEN, O_AOFF, O_ALEN, O_NCOL
};
constexpr int O_SZ[O_NCOL] = {4, 8, 8, 8, 1, 4, 4, 4, 8, 8, 1, 4, 4, 4, 4, 4, 4, 4, 4, 4};

// the pending rows' three lists, then the running rows' group list
enum { L_NOVEL = 0, L_ATTR = 1, L_GROUP = 2, L_RGROUP = 3, L_N };
// the offers' port ranges (begin, end), gpu map (model, count), disk map (type, MiB) and attribute values (one per
// column of the offer's row)
enum { OL_PORT = 0, OL_GPU = 1, OL_DISK = 2, OL_ATTR = 3, OL_N };

// ---- scatter: row i of a batch to slot[i].  Upserts write the columns (a null source writes the
// column's absent value) and the rows' list ranges; removals clear the live flag.  Both bump the
// generation, which is what retires a queue entry.  A patch (live null) writes its columns only: the
// slot keeps its live flag and generation, so its queue entry stays.
constexpr int MAXC = 16;
constexpr int SCATTER_MAXC = MAXC + 1;   // a pending upsert: its data columns, then the job and list facts' resets
// The columns an upsert resets after the delta's own, with the absent value each gets.  The scatters write exactly these
// lists, so a further reset column is one more entry here, and the column count that bounds ScatterArgs::c follows.
struct ResetCol { int col; long long dflt; };
constexpr ResetCol PENDING_UPSERT_RESETS[] = {{P_JF, 0},        // no job facts
                                              {P_LF_EXEC, 0}};  // no list facts
constexpr ResetCol RUNNING_UPSERT_RESETS[] = {{R_MAXRT, -1}, {R_FACTS, 0}, {R_REASON, -1},   // the absent task facts
                                              {R_LF_EXEC, 0}};                              // no list facts
constexpr int N_PENDING_UPSERT_RESETS = sizeof(PENDING_UPSERT_RESETS) / sizeof(ResetCol);
constexpr int N_RUNNING_UPSERT_RESETS = sizeof(RUNNING_UPSERT_RESETS) / sizeof(ResetCol);
static_assert(P_NDATA + N_PENDING_UPSERT_RESETS <= SCATTER_MAXC, "a pending upsert's columns do not fit ScatterArgs");
static_assert(R_NDATA + N_RUNNING_UPSERT_RESETS <= SCATTER_MAXC, "a running upsert's columns do not fit ScatterArgs");
static_assert(O_NDATA <= SCATTER_MAXC, "an offer's columns do not fit ScatterArgs");
struct ScatterCol { char* dst; const char* src; long long dflt; int sz; };
struct ScatterArgs {
  ScatterCol c[SCATTER_MAXC];
  int nc, n, upsert;
  const int32_t* slot;
  uint8_t* live;           // null: a patch
  uint32_t* gen;
  int32_t* loff[4];        // per-slot list range; null: the table has no lists
  int32_t* llen[4];
  const int32_t* doff[4];  // the batch's CSR offsets (null: empty lists)
  int32_t tail[4];         // where the batch's lists were appended
};

__global__ void scatter_kernel(ScatterArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int s = a.slot[i];
#pragma unroll
  for (int k = 0; k < SCATTER_MAXC; k++) {
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
  for (int l = 0; l < 4; l++)
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
  static_cast<int64_t*>(rc[R_MAXRT])[r] = -1;
  static_cast<uint8_t*>(rc[R_FACTS])[r] = 0;
  static_cast<int32_t*>(rc[R_REASON])[r] = -1;
  static_cast<int64_t*>(rc[R_LF_SUBMIT])[r] = static_cast<const int64_t*>(pc[P_LF_SUBMIT])[s];
  static_cast<int32_t*>(rc[R_LF_POOL])[r] = static_cast<const int32_t*>(pc[P_LF_POOL])[s];
  static_cast<uint8_t*>(rc[R_LF_EXEC])[r] = static_cast<const uint8_t*>(pc[P_LF_EXEC])[s];
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
template <class T1>
__global__ void list_compact_kernel(OrderScan<int, 1> os, const uint8_t* live, int32_t* off, const int32_t* len, int n,
                                    const int32_t* src0, const T1* src1, int32_t* dst0, T1* dst1) {
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

// a pending slot's list entries survive a compaction while it is live or parked
__global__ void park_keep_kernel(const uint8_t* live, const uint8_t* park, int n, uint8_t* keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keep[i] = live[i] | park[i];
}

// warp per requeued row whose novel-host list gains the entry code[w]: pending slot slot[w]'s list moves to the
// arena's tail + the exclusive scan of the rows' new lengths, the entry after it, where an upsert's CSR would put it
struct NovelLen {
  const int32_t* slot; const int32_t* len;
  __device__ void operator()(int p, int (&x)[1]) const { x[0] = len[slot[p]] + 1; }
};
__global__ void requeue_novel_kernel(OrderScan<int, 1> os, const int32_t* slot, const int32_t* code, int n,
                                     int32_t* off, int32_t* len, int32_t* v, int32_t tail) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n) return;
  const int s = slot[w], l = len[s], start = tail + os.at(0, w) - (l + 1), o = off[s];
  for (int i = lane; i < l; i += 32) v[start + i] = v[o + i];
  __syncwarp();
  if (lane == 0) {
    v[start + l] = code[w];
    off[s] = start;
    len[s] = l + 1;
  }
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
template <class T1>
__global__ void csr_gather_kernel(OrderScan<int, 1> os, const int32_t* m_slot, int n, const int32_t* off,
                                  const int32_t* len, const int32_t* src0, const T1* src1, int32_t* doff,
                                  int32_t* dst0, T1* dst1) {
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

// ---- usage folds: a table's live rows, dense in slot order, each handle's after those of the handles before it
// (base).  The table's columns by index: the running rows (user, task id, amounts, hostname code) or the pending
// rows (user, job id, amounts; no host).  host = the index of the row's hostname code in the caller's list, or H
// when the row's host is -1 or not listed (a segment no output reads)
struct TableCols { int live, user, id, amt[3], host; };
constexpr TableCols RUN_COLS = {R_LIVE, R_USER, R_TID, {R_CPUS, R_MEM, R_GPUS}, R_HOST};
constexpr TableCols PEND_COLS = {P_LIVE, P_USER, P_JID, {P_CPUS, P_MEM, P_GPUS}, -1};
struct UsageRows {
  void* const* col; TableCols c; int base;
  int32_t* user; int64_t* id; int32_t* host; double* amt[3];   // host null: no host list
  const int32_t* host_of; int32_t n_codes, H;
  __device__ bool keep(int i) const { return static_cast<const uint8_t*>(col[c.live])[i]; }
  template <class V> void outs(V&& v) { v(user); v(id); v(amt[0]); v(amt[1]); v(amt[2]); v(host); }
  __device__ void emit(int i, int d) const {
    d += base;
    user[d] = static_cast<const int32_t*>(col[c.user])[i];
    id[d] = static_cast<const int64_t*>(col[c.id])[i];
#pragma unroll
    for (int k = 0; k < 3; k++) amt[k][d] = static_cast<const double*>(col[c.amt[k]])[i];
    if (host) {
      const int32_t code = static_cast<const int32_t*>(col[c.host])[i];
      const int32_t h = code >= 0 && code < n_codes ? host_of[code] : -1;
      host[d] = h < 0 ? H : h;
    }
  }
};
// (key, task id, dense index); key null: task id alone.  Task ids are unique among one handle's live rows; an id
// that several handles hold goes in handle order, which the dense index keeps.
struct LessKeyTid {
  const int32_t* key; const int64_t* tid;
  __device__ bool operator()(int32_t a, int32_t b) const {
    if (key && key[a] != key[b]) return key[a] < key[b];
    if (tid[a] != tid[b]) return tid[a] < tid[b];
    return a < b;
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

// Warp per segment (users, then hosts, then the pool; a user or host without rows has an empty one): the left
// fold of cpus, mem and gpus in the segment's order (ascending task id within it), by segment_fold.
__global__ void __launch_bounds__(128) usage_fold_kernel(UsageArgs a) {
  __shared__ double stage[4][3][32];
  int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, kind = 0;
  while (kind < US_N && g >= a.seg[kind].n) g -= a.seg[kind++].n;
  if (kind == US_N) return;
  const UsageSegs& q = a.seg[kind];
  const int s = q.start ? q.start[g] : 0, e = q.start ? q.end[g] : a.R;
  double acc[3];
  // The load reads q.ord through the kernel parameter: a LoadSorted copy of the pointers compiled to a different load
  // schedule and made the off-grid folds about 3 % slower on an H100.
  segment_fold(acc, s, e, q.scan && grid_exact(a.gf, a.R), q.os, a.gf, [&](int p, double (&x)[3]) {
    const int i = q.ord[p];
    x[0] = a.amt[0][i]; x[1] = a.amt[1][i]; x[2] = a.amt[2][i];
  }, stage[threadIdx.x >> 5]);
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

// ---- the monitor's user stats (set-stats-counters!, monitor.clj:177-207) from the running and waiting folds
struct StatsArgs {
  const double* run; const double* wait;   // [4][U] count, cpus, mem, gpus: the two usage folds
  const double *div_cpus, *div_mem, *q_count, *q_cpus, *q_mem;
  const uint8_t* rest_ok;                  // null: every user's other quota keys are > 0
  int U;
  int64_t* jobs; double* cpus; double* mem;   // [4][U] by COOK_STATS_*
  uint8_t* member;                            // [U] bit s: the user is in state s
};
// Thread per user.  Starved (get-starved-job-stats :69-90): every share key above the running amount; values
// (merge-with min waiting (merge-with - share running)), where :jobs is only in the running map and passes the
// subtraction.  Waiting under quota (:92-116): every quota key above the running amount; values min(max(quota -
// running, 0), waiting).  An absent running map reads 0.0, which leaves every subtraction exact.
__global__ void user_stats_kernel(StatsArgs a) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= a.U) return;
  const int U = a.U;
  const double rj = a.run[u], rc = a.run[U + u], rm = a.run[2 * U + u];
  const double wj = a.wait[u], wc = a.wait[U + u], wm = a.wait[2 * U + u];
  const bool running = rj > 0.0, waiting = wj > 0.0;
  int64_t j[4] = {(int64_t)rj, (int64_t)wj, 0, 0};
  double c[4] = {rc, wc, 0.0, 0.0}, m[4] = {rm, wm, 0.0, 0.0};
  int bits = (running ? 1 << COOK_STATS_RUNNING : 0) | (waiting ? 1 << COOK_STATS_WAITING : 0);
  if (waiting) {
    const double sc = a.div_cpus[u], sm = a.div_mem[u];
    if (rc < sc && rm < sm) {
      bits |= 1 << COOK_STATS_STARVED;
      j[COOK_STATS_STARVED] = running ? min(j[0], j[1]) : j[1];
      c[COOK_STATS_STARVED] = fmin(wc, sc - rc);
      m[COOK_STATS_STARVED] = fmin(wm, sm - rm);
    }
    const double qj = a.q_count[u], qc = a.q_cpus[u], qm = a.q_mem[u];
    if (rj < qj && rc < qc && rm < qm && (!a.rest_ok || a.rest_ok[u])) {
      bits |= 1 << COOK_STATS_WUQ;
      j[COOK_STATS_WUQ] = (int64_t)fmin(wj, fmax(qj - rj, 0.0));
      c[COOK_STATS_WUQ] = fmin(wc, fmax(qc - rc, 0.0));
      m[COOK_STATS_WUQ] = fmin(wm, fmax(qm - rm, 0.0));
    }
  }
#pragma unroll
  for (int s = 0; s < 4; s++) {
    a.jobs[(size_t)s * U + u] = j[s]; a.cpus[(size_t)s * U + u] = c[s]; a.mem[(size_t)s * U + u] = m[s];
  }
  a.member[u] = (uint8_t)bits;
}

struct StatsTotals { int64_t jobs[4]; double cpus[4]; double mem[4]; int64_t users[COOK_USERS_N]; };
__device__ __forceinline__ long long warp_sum_ll(long long x) {
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(FULL_MASK, x, o);
  return x;
}
// One block, warp s per state: the "all" entry (add-aggregated-stats :59-67), a left fold of cpus and mem over the
// state's users in ascending user code (association-free when all 4 * U values are on the grid), jobs an integer sum;
// then the five user counts.
__global__ void __launch_bounds__(128) user_stats_totals_kernel(const int64_t* jobs, const double* cpus,
                                                                const double* mem, const uint8_t* member, int U,
                                                                const GridFlag* gf, StatsTotals* out) {
  __shared__ double stage[4][2][32];
  __shared__ long long n_in[4];
  const int s = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t o = (size_t)s * U;
  double acc[2] = {0.0, 0.0};
  warp_fold_sum<2, 4>(acc, U, grid_exact(gf, U), [&](int u, double (&x)[2]) {
    if (!((member[u] >> s) & 1)) return false;
    x[0] = cpus[o + u]; x[1] = mem[o + u];
    return true;
  }, stage[s]);
  long long nj = 0, nm = 0, nt = 0, nsat = 0;
  for (int u = lane; u < U; u += 32) {
    const int b = member[u];
    if ((b >> s) & 1) { nj += jobs[o + u]; nm++; }
    nt += (b & 3) != 0;   // running or waiting
    nsat += (b & 3) == 1; // running, not waiting
  }
  nj = warp_sum_ll(nj); nm = warp_sum_ll(nm); nt = warp_sum_ll(nt); nsat = warp_sum_ll(nsat);
  if (lane == 0) { out->jobs[s] = nj; out->cpus[s] = acc[0]; out->mem[s] = acc[1]; n_in[s] = nm; }
  __syncthreads();
  if (threadIdx.x == 0) {
    out->users[COOK_USERS_TOTAL] = nt;
    out->users[COOK_USERS_STARVED] = n_in[COOK_STATS_STARVED];
    out->users[COOK_USERS_WUQ] = n_in[COOK_STATS_WUQ];
    out->users[COOK_USERS_HUNGRY] = n_in[COOK_STATS_WAITING] - n_in[COOK_STATS_STARVED];
    out->users[COOK_USERS_SATISFIED] = nsat;
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
  uint8_t jf = 0;            // the COOK_JF_* bits of the row's job facts
  int64_t touched = 0;       // PoolState::pend_epoch when the slot was last upserted or removed
  std::vector<int32_t> groups, attr_cols;
  std::vector<int32_t> novel;   // the novel-host list: a requeue appends to it only what it does not hold
};

// A job's retry facts (cook_state_retry_facts): its max-retries, COOK_RF_* bits and its done instances' reason codes
// counted per code (-1: none), as reasons->attempts-consumed reads them (frequencies).
struct RetryFacts {
  int32_t max_retries = 0;
  uint8_t flags = 0;
  std::map<int32_t, int32_t> done;
};
struct RetryReason { bool mea_culpa = false; int32_t limit = -2; };   // limit -2: the global one

// Up to MAXC device columns of `cap` rows each, column k w[k] bytes per row (1, 4 or 8): the storage of every growing
// store of a handle.  A store fixes its widths, its capacity floor and whether new rows are zeroed when it is built.
struct Columns {
  static constexpr int MAXC = std::max({(int)P_NCOL, (int)R_NCOL, (int)O_NCOL});   // the widest slot table
  int n = 0, w[MAXC] = {};
  int64_t floor = 0;
  bool zero = false;
  void* p[MAXC] = {};
  int64_t cap = 0;

  Columns() = default;
  Columns(const int* widths, int nc, int64_t fl, bool z) : n(nc), floor(fl), zero(z) {
    assert(nc >= 0 && nc <= MAXC);
    std::copy(widths, widths + nc, w);
    for (int k = 0; k < nc; k++) assert(w[k] == 1 || w[k] == 4 || w[k] == 8);
  }
  Columns(std::initializer_list<int> widths, int64_t fl, bool z) : Columns(widths.begin(), (int)widths.size(), fl, z) {}

  Columns shape() const { return Columns(w, n, floor, zero); }   // no rows
  void* operator[](int k) const { return p[k]; }
  template <class T>
  T* at(int k) const { return static_cast<T*>(p[k]); }
  // *out: a set of this shape with capacity max(want, 2 cap, floor) holding this set's first keep rows (device to
  // device), the stream synchronized when rows were copied or zeroed.  On failure nothing is left allocated and *out
  // is untouched.
  cudaError_t grown(int64_t want, int64_t keep, cudaStream_t st, Columns* out) const {
    Columns nc = shape();
    nc.cap = std::max({want, 2 * cap, floor});
    cudaError_t e = cudaSuccess;
    for (int k = 0; k < n && e == cudaSuccess; k++) {
      char* q = nullptr;
      e = cudaMalloc(&q, (size_t)nc.cap * w[k]);
      if (e != cudaSuccess) break;
      nc.p[k] = q;
      if (keep) e = cudaMemcpyAsync(q, p[k], (size_t)keep * w[k], cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess && zero) e = cudaMemsetAsync(q + keep * w[k], 0, (size_t)(nc.cap - keep) * w[k], st);
    }
    if (e == cudaSuccess && (keep || zero)) e = cudaStreamSynchronize(st);   // the copies and fills done
    if (e != cudaSuccess) {
      nc.release();
      return e;
    }
    *out = nc;
    return cudaSuccess;
  }
  // capacity >= want, the first keep rows kept; all or nothing: on failure the set is as it was
  cudaError_t grow(int64_t want, int64_t keep, cudaStream_t st) {
    if (want <= cap) return cudaSuccess;
    Columns nc;
    if (cudaError_t e = grown(want, keep, st, &nc)) return e;
    release();
    *this = nc;
    return cudaSuccess;
  }
  void release() {
    for (int k = 0; k < n; k++) if (p[k]) cudaFree(p[k]);
    std::fill(p, p + n, nullptr);
    cap = 0;
  }
  // inside a carve: host rows srcs[k][0, m) to rows [row, row + m) of column k, for the first srcs.size() columns.  A
  // source past the set's columns must be null (the second array of a one-array list arena).
  void copy(Carve& c, int64_t row, int64_t m, std::initializer_list<const void*> srcs) const {
    for (int k = 0; k < (int)srcs.size(); k++) {
      const void* s = srcs.begin()[k];
      if (k >= n) {
        assert(!s);
        continue;
      }
      c.copy(static_cast<char*>(p[k]) + row * w[k], static_cast<const char*>(s), (size_t)m * w[k]);
    }
  }
};

struct Table {
  Columns col;                   // zeroed on growth: the live flag and generation of unused slots are read
  Columns ptrs;                  // MAXC rows: the column pointers on the device (for the gather kernels)
  void** d_col = nullptr;        // ptrs' column
  int32_t hw = 0;                // slots ever used
  int nlist = 0, lcol[4] = {};   // the per-slot (off, len) column pairs of the table's lists: off at lcol[l]
  int live_col = 0;
  std::unordered_map<int64_t, int32_t> slot_of;
  std::vector<int32_t> free;

  Table(const int* sz, int ncol) : col(sz, ncol, 1024, true), ptrs({(int)sizeof(void*)}, 0, false) {}
  template <class T>
  const T* at(int k) const { return col.at<const T>(k); }
  // capacity >= n: the columns grown, and a fresh pointer array naming them, so that col and d_col change together
  cudaError_t grow(int32_t n, cudaStream_t st) {
    if (n <= col.cap) return cudaSuccess;
    Columns nc, np = ptrs.shape();
    cudaError_t e = col.grown(n, col.cap, st, &nc);
    if (e == cudaSuccess) e = np.grow(Columns::MAXC, 0, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(np[0], nc.p, sizeof(nc.p), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
      nc.release();
      np.release();
      return e;
    }
    release();
    col = nc;
    ptrs = np;
    d_col = ptrs.at<void*>(0);
    return cudaSuccess;
  }
  int32_t take_slot() {
    if (!free.empty()) { const int32_t s = free.back(); free.pop_back(); return s; }
    return hw++;
  }
  void release() { col.release(); ptrs.release(); }
};

// A CSR arena: one value array, or two for (attribute column, value) pairs, whose second one holds doubles in an
// offer's gpu or disk map; and its compaction target, freed when the arena grows and made again at the next compaction.
struct ListArena {
  Columns v, alt;
  int64_t tail = 0, live = 0;
  explicit ListArena(std::initializer_list<int> widths = {4}) : v(widths, 4096, false), alt(v.shape()) {}
  int32_t* at(int i) const { return v.at<int32_t>(i); }   // value array i, as int32
  cudaError_t grow(int64_t n, cudaStream_t st) {
    if (n <= v.cap) return cudaSuccess;
    if (cudaError_t e = v.grow(n, tail, st)) return e;
    alt.release();
    return cudaSuccess;
  }
  void release() { v.release(); alt.release(); }
};

// A handle's append-only device table (the history, the completed-job log, the straggler records): rows in arrival
// order, dense in [0, tail), in one column set; rows leave only by a stable compaction (LogKeep).  Off until seeded;
// `since` is the horizon.
struct Log {
  Columns c;
  int64_t tail = 0, since = 0;
  bool on = false;
  explicit Log(std::initializer_list<int> widths) : c(widths, 4096, false) {}
  cudaError_t grow(int64_t n, cudaStream_t st) { return c.grow(n, tail, st); }
  void release() { c.release(); tail = since = 0; on = false; }
};

// The successful runtimes the straggler sweep measures against: (group code, whole seconds) with a live flag,
// compacted (compact_records) into its own target once its dead records outnumber the live ones.
enum { RC_GRP, RC_RT, RC_LIVE };
struct Records : Log {
  Columns alt;   // compaction target: freed when the table grows, made again at the next compaction
  int64_t n_live = 0;
  Records() : Log({4, 4, 1}), alt(c.shape()) {}
  cudaError_t grow(int64_t n, cudaStream_t st) {
    if (n <= c.cap) return cudaSuccess;
    if (cudaError_t e = Log::grow(n, st)) return e;
    alt.release();
    return cudaSuccess;
  }
  void release() { Log::release(); alt.release(); n_live = 0; }
};

// The finished instances (cook_state_history_*): 49 B per row; the horizon is on start time.  HistCols: the typed
// columns, as the readers take them.
enum { H_TID, H_START, H_END, H_CPUS, H_MEM, H_USER, H_REASON, H_OK };
struct HistCols {
  int64_t* tid = nullptr; int64_t* start = nullptr; int64_t* end = nullptr; double* cpus = nullptr; double* mem = nullptr;
  int32_t* user = nullptr; int32_t* reason = nullptr; uint8_t* ok = nullptr;
};
struct History : Log {
  History() : Log({8, 8, 8, 8, 8, 4, 4, 1}) {}
  HistCols cols() const {
    return {c.at<int64_t>(H_TID), c.at<int64_t>(H_START), c.at<int64_t>(H_END), c.at<double>(H_CPUS),
            c.at<double>(H_MEM), c.at<int32_t>(H_USER), c.at<int32_t>(H_REASON), c.at<uint8_t>(H_OK)};
  }
};

// The completed-job log (cook_state_completed_*): 34 B per row, a job-state record each; the horizon is on submit time.
// The device log and, by row on the host, each row's user and submit time: the listing sizes its buffers by the
// user's rows, and the advance knows whose rows it drops, without a transfer.
enum { CJ_JID, CJ_STAMP, CJ_SUBMIT, CJ_USER, CJ_SPOOL, CJ_EXEC, CJ_KIND };
struct CJCols {
  int64_t* jid = nullptr; int64_t* stamp = nullptr; int64_t* submit = nullptr; int32_t* user = nullptr;
  int32_t* spool = nullptr; int8_t* exec = nullptr; uint8_t* kind = nullptr;
};
struct Completed : Log {
  std::vector<int32_t> h_user;
  std::vector<int64_t> h_submit;
  std::unordered_map<int32_t, int64_t> users;   // user -> rows
  Completed() : Log({8, 8, 8, 4, 4, 1, 1}) {}
  CJCols cols() const {
    return {c.at<int64_t>(CJ_JID), c.at<int64_t>(CJ_STAMP), c.at<int64_t>(CJ_SUBMIT), c.at<int32_t>(CJ_USER),
            c.at<int32_t>(CJ_SPOOL), c.at<int8_t>(CJ_EXEC), c.at<uint8_t>(CJ_KIND)};
  }
  void clear_rows() { tail = 0; h_user.clear(); h_submit.clear(); users.clear(); }
  void release() { Log::release(); clear_rows(); }
};

void count_add(std::map<int32_t, int64_t>& m, int32_t code, int64_t d) {
  auto it = m.emplace(code, 0).first;
  if ((it->second += d) == 0) m.erase(it);
}
int32_t count_max(const std::map<int32_t, int64_t>& m) { return m.empty() ? -1 : m.rbegin()->first; }

// What the host keeps of one live offer, by offer slot.
struct OfferInfo {
  int64_t id = 0, seq = 0, received = 0;
  int32_t code = 0;
  int32_t len[4] = {0, 0, 0, 0};   // ports, gpu map, disk map, attribute columns
  bool single_shot = false, k8s = false, max_tasks = false;
};
// A hostname code: its name, and its live offers in arrival order (seq, slot).  A code with a live offer is a VM.
struct OfferHost {
  std::string name;
  std::map<int64_t, int32_t> live;
};

// The last resident match round, as cook_state_match_metrics reads it: the match's rows as pending slots (its m_slot,
// copied on the device), the pending epoch at the match and the plan run (match_runs) that holds the considerable jobs
// and their assignments; and the unmatched counters, the last counted round's unmatched jobs as (job id ascending,
// cycles), double-buffered.
struct MetricsRound {
  bool on = false, counted = false;
  int32_t n_rows = 0;
  int64_t epoch = 0;
  uint64_t run = 0;
  Columns slot{{4}, 0, false};
  Columns u[2] = {Columns({8, 4}, 0, false), Columns({8, 4}, 0, false)};   // (job id, cycles) each
  int cur = 0; int32_t u_n = 0;
  void release() {
    slot.release(); u[0].release(); u[1].release();
    *this = MetricsRound{};
  }
};

struct PoolState {
  Table pend{P_SZ, P_NCOL}, run{R_SZ, R_NCOL};
  // ---- the live offers (cook_state_offers_add, cook_state_match_offers)
  Table offer{O_SZ, O_NCOL};
  std::vector<OfferInfo> oinfo;                  // by offer slot
  std::unordered_map<int32_t, OfferHost> ohost;  // by hostname code, every code the handle has a name for
  std::map<std::string, int32_t> code_of_name;   // every name the handle knows (byte order)
  std::map<std::string, int32_t> vm_names;       // the names of the VMs (hosts with a live offer), in byte order
  std::map<std::pair<int64_t, int64_t>, int32_t> by_time;   // (received, seq) -> slot: expiry walks this
  std::map<int64_t, int32_t> single_shot;        // seq -> slot of the live single-shot offers
  std::map<int32_t, int64_t> owidth;             // attribute-row width -> live offers
  int64_t next_seq = 0;
  int64_t o_ports = 0;                           // port ranges over the live offers
  int64_t vm_gpu = 0, vm_disk = 0, vm_k8s = 0, vm_maxt = 0;   // over the VMs' newest offers: map entries, flags
  std::vector<PendingInfo> pinfo;    // by pending slot
  std::vector<int32_t> ruser, rhost; // by running slot
  std::vector<std::vector<int32_t>> rgroups;   // by running slot: its group list
  std::vector<int64_t> rstart;                 // by running slot: its start time (cook_state_finish's checks)
  std::vector<uint8_t> rfacts;                 // by running slot: its RF_* bits
  std::vector<int64_t> rjid, rtid;             // by running slot: its job id and task id
  std::vector<int32_t> rreason;                // by running slot: its reason fact (cook_state_task_reason)
  std::unordered_map<int64_t, std::vector<int32_t>> jobs_r;   // job id -> its live running slots (cook_state_unscheduled)
  int64_t grp_rows = 0;                        // live running rows with a group list
  Records rec;                                 // the successful runtimes per group
  std::map<int32_t, int64_t> rec_groups;       // group code -> live records
  History hist;                                // the finished instances
  Completed cj;                                // the completed-job log
  ListArena lists[L_N];
  ListArena olists[OL_N];
  std::map<int32_t, int64_t> users_p, users_r, attr_cols, groups;   // code -> live uses
  std::map<int32_t, int64_t> hosts_r;                               // running rows' hostname codes (-1 too)
  std::map<int32_t, int64_t> groups_r;                              // running rows' group codes
  int64_t cot_rows = 0, cot_n = 0;   // live running rows with a known host and a group list, and their entries
  int64_t nflag[F_N] = {};
  int64_t jf_keyed = 0;               // live pending rows whose job facts hold a gpus or disk resource
  int64_t pend_epoch = 0;             // counts the calls that upserted or removed a pending row
  MetricsRound mm;
  std::unordered_set<int32_t> reserved;   // the live pending slots whose reserved_host is not -1
  // ---- retries (cook_state_retry_config / _facts, cook_state_status).  A launched job with facts keeps its pending
  // slot parked: not live, not on the free list, its columns and lists kept for a requeue.
  int32_t mc_limit = 5;                              // the global mea-culpa failure limit
  std::unordered_map<int32_t, RetryReason> reasons;  // reason code -> mea-culpa and failure limit
  std::unordered_map<int64_t, RetryFacts> retry;     // job id -> its facts
  std::unordered_map<int64_t, int32_t> parked;       // job id -> its parked pending slot
  int64_t park_len[3] = {};                          // list entries the parked slots hold (kept by the compaction)
  Columns park{{1}, 0, true};                        // per pending slot: 1 while parked; allocated at the first park
  Arena stage;                        // one batch's uploads
  Arena scratch;                      // one call's device buffers
  Arena derive;                       // a derived match's or rebalance's running-side scratch (scratch is live then)
  Arena omerge;                       // a match's merge of the live offers
  Arena queue;                        // the ranked queue, carved by rank only: it lives until the match
  int32_t* counters = nullptr;        // [0] running rows, [1] pending rows, [2] live queue entries
  GridFlag* gf0 = nullptr;            // stays zero: integer scans are always exact
  const int32_t* q_slot = nullptr; const uint32_t* q_gen = nullptr; const int64_t* q_jid = nullptr;
  int32_t n_q = 0;
  bool ranked = false;

  PoolState() {
    pend.nlist = 3; pend.lcol[L_NOVEL] = P_NOFF; pend.lcol[L_ATTR] = P_AOFF; pend.lcol[L_GROUP] = P_GOFF;
    run.nlist = 1; run.lcol[0] = R_GOFF;
    pend.live_col = P_LIVE; run.live_col = R_LIVE;
    offer.live_col = O_LIVE;
    offer.nlist = 4;
    for (int l = 0; l < 4; l++) offer.lcol[l] = O_POFF + 2 * l;
    lists[L_ATTR] = olists[OL_PORT] = ListArena({4, 4});
    olists[OL_GPU] = olists[OL_DISK] = ListArena({4, 8});
  }
  void release() {
    pend.release(); run.release(); offer.release(); rec.release(); hist.release(); cj.release();
    for (auto& l : lists) l.release();
    for (auto& l : olists) l.release();
    stage.release(); scratch.release(); derive.release(); queue.release(); omerge.release();
    mm.release();
    park.release();
    if (counters) cudaFree(counters);
    if (gf0) cudaFree(gf0);
  }
  void add_pending(int32_t slot, const PendingInfo& pi, int64_t sign) {
    count_add(users_p, pi.user, sign);
    for (int32_t g : pi.groups) count_add(groups, g, sign);
    for (int32_t c : pi.attr_cols) count_add(attr_cols, c, sign);
    for (int l = 0; l < 3; l++) lists[l].live += sign * pi.len[l];
    for (int f = 0; f < F_N; f++) if ((pi.flags >> f) & 1) nflag[f] += sign;
    if (pi.jf & (COOK_JF_GPUS | COOK_JF_DISK)) jf_keyed += sign;
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
    if (!g.empty()) grp_rows += sign;
    if (rhost[slot] != -1 && !g.empty()) {
      cot_rows += sign;
      cot_n += sign * (int64_t)g.size();
    }
    if (sign > 0) {
      jobs_r[rjid[slot]].push_back(slot);
    } else {
      auto it = jobs_r.find(rjid[slot]);
      std::vector<int32_t>& v = it->second;
      v.erase(std::find(v.begin(), v.end(), slot));
      if (v.empty()) jobs_r.erase(it);
    }
  }
  void running_room(int32_t slot) {
    if ((size_t)slot < ruser.size()) return;
    const size_t n = std::max<size_t>(slot + 1, 2 * ruser.size());
    ruser.resize(n); rhost.resize(n); rgroups.resize(n); rstart.resize(n); rfacts.resize(n); rjid.resize(n); rtid.resize(n);
    rreason.resize(n);
  }
  // the park flags cover every pending slot, new ones zeroed: their capacity is exactly pend's, since each growth of
  // pend at least doubles it and the flags' capacity is one pend had before
  cudaError_t park_room(cudaStream_t st) { return park.grow(pend.col.cap, park.cap, st); }
  // job jid's parked copy, if any, is freed: its slot back on the free list (appended to *freed), its entries dead
  void unpark(int64_t jid, std::vector<int32_t>* freed) {
    auto it = parked.find(jid);
    if (it == parked.end()) return;
    const int32_t s = it->second;
    parked.erase(it);
    for (int l = 0; l < 3; l++) park_len[l] -= pinfo[s].len[l];
    pend.free.push_back(s);
    freed->push_back(s);
  }
  // reasons->attempts-consumed (schema.clj:1154-1172) over a job's done instances
  int32_t attempts(const RetryFacts& f) const {
    int64_t a = 0;
    for (const auto& kv : f.done) {
      auto r = reasons.find(kv.first);
      if (kv.first < 0 || r == reasons.end() || !r->second.mea_culpa) { a += kv.second; continue; }
      const int32_t lim = (f.flags & COOK_RF_DISABLE_MEA_CULPA) ? 0 : r->second.limit != -2 ? r->second.limit : mc_limit;
      if (lim != -1) a += std::max(0, kv.second - lim);
    }
    return (int32_t)std::min<int64_t>(a, INT32_MAX);
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
    csr_gather_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, m_slot, n, S->pend.at<int32_t>(loff[l]), len, S->lists[l].at(0),
                                                   S->lists[l].at(1), writable(doff[l]), writable(dst[l][0]),
                                                   writable(dst[l][1]));
    (*nl)++;
  }
}

// compaction of every list arena whose dead entries outnumber its live ones
int32_t compact_lists(cook_pool* pool, PoolState* S, cudaStream_t st, int* nl) {
  for (int l = 0; l < L_N + OL_N; l++) {
    ListArena& A = l < L_N ? S->lists[l] : S->olists[l - L_N];
    const bool parked = l < 3 && !S->parked.empty();   // parked slots' entries are kept, not dead
    const int64_t kept = A.live + (l < 3 ? S->park_len[l] : 0);
    if (A.tail - kept <= kept) continue;
    const Table& t = l == L_RGROUP ? S->run : l >= L_N ? S->offer : S->pend;
    const int n = t.hw, oc = t.lcol[l == L_RGROUP ? 0 : l >= L_N ? l - L_N : l];
    if (kept > 0 && n > 0) {
      CK(pool, A.alt.grow(A.v.cap, 0, st));
      if (parked) CK(pool, S->park_room(st));
      OrderScan<int, 1> os;
      uint8_t* keep = nullptr;
      CK(pool, carve(S->scratch, st, nullptr, nullptr, [&](Carve& c) {
        os.part[0] = c.take<int32_t>(n);
        os.tile[0] = c.take<int32_t>((n + OS_TILE - 1) / OS_TILE + 1);
        if (parked) keep = c.take<uint8_t>(n);
      }));
      const uint8_t* live = static_cast<const uint8_t*>(t.col[t.live_col]);
      if (parked) {
        park_keep_kernel<<<(n + 255) / 256, 256, 0, st>>>(live, S->park.at<uint8_t>(0), n, keep);
        (*nl)++;
        live = keep;
      }
      int32_t* off = static_cast<int32_t*>(t.col[oc]);
      const int32_t* len = static_cast<const int32_t*>(t.col[oc + 1]);
      order_scan(os, SlotLen{live, len}, n, S->gf0, st, nl);
      if (A.v.w[1] == 8)
        list_compact_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, live, off, len, n, A.at(0), A.v.at<double>(1),
                                                         A.alt.at<int32_t>(0), A.alt.at<double>(1));
      else
        list_compact_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, live, off, len, n, A.at(0), A.at(1),
                                                         A.alt.at<int32_t>(0), A.alt.at<int32_t>(1));
      (*nl)++;
      CK(pool, cudaGetLastError());
      std::swap(A.v, A.alt);
    }
    A.tail = kept;
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

// One column of a patch scatter: table column `col` from the host source `src` (n values; null: the column is not
// written), with its absent value.
struct PatchCol { int col; const void* src; long long dflt; };
// Fills a patch scatter of table t's n rows at `slot` inside a carve: the slots, then each given column uploaded at the
// table's own width.  The columns start from none on each pass of the carve.
void patch_args(Carve& c, ScatterArgs& a, const Table& t, const int32_t* slot, int n, std::initializer_list<PatchCol> cols) {
  a.slot = c.up(slot, n);
  a.nc = 0;
  for (const PatchCol& p : cols) {
    if (!p.src) continue;
    const int sz = t.col.w[p.col];
    const char* up = sz == 1   ? reinterpret_cast<const char*>(c.up(static_cast<const uint8_t*>(p.src), n))
                     : sz == 4 ? reinterpret_cast<const char*>(c.up(static_cast<const int32_t*>(p.src), n))
                               : reinterpret_cast<const char*>(c.up(static_cast<const int64_t*>(p.src), n));
    a.c[a.nc++] = ScatterCol{static_cast<char*>(t.col[p.col]), up, p.dflt, sz};
  }
}

// the slots of n distinct ids live in table t (`kind`: "job" or "task"), or the call's refusal
int32_t live_slots(cook_pool* pool, const char* who, const Table& t, const char* kind, int n, const int64_t* id,
                   std::vector<int32_t>* slot) {
  std::unordered_set<int64_t> seen;
  seen.reserve((size_t)n);
  slot->resize(n);
  for (int i = 0; i < n; i++) {
    if (!seen.insert(id[i]).second) return set_err(pool, COOK_E_BADARG, "%s: %s id twice", who, kind);
    auto it = t.slot_of.find(id[i]);
    if (it == t.slot_of.end()) return set_err(pool, COOK_E_BADARG, "%s: unknown %s id", who, kind);
    (*slot)[i] = it->second;
  }
  return COOK_OK;
}

// A single-handle call's entry: a NULL handle is a bare COOK_E_BADARG (no handle to hold the message); then the
// handle's device is made current and body(S) runs on its state, created at the first call.
template <class Body>
int32_t on_state(cook_pool* pool, const char* who, const Body& body) {
  if (!pool) return COOK_E_BADARG;
  CK(pool, cudaSetDevice(pool->device));
  PoolState* S = state_of(pool, true);
  if (!S) return set_err(pool, COOK_E_OOM, "%s: out of device memory", who);
  return body(S);
}

// A state write on the handle's stream: up() carves its uploads (from `stage` unless another arena is given) between
// ev[20] and ev[21]; the call counts its launches in nl; end() checks the launches, records ev[22], synchronizes and
// records the COOK_PHASE_STATE statistics of the bytes and launches counted here.
struct StateWrite {
  cook_pool* pool;
  PoolState* S;
  cudaStream_t st;
  int64_t h2d = 0, d2h = 0;
  int nl = 0;
  StateWrite(cook_pool* p, PoolState* s) : pool(p), S(s), st(p->stream) {}
  template <class Body>
  int32_t up(const Body& body) { return up(S->stage, body); }
  template <class Body>
  int32_t up(Arena& a, const Body& body) {
    CK(pool, carve(a, st, pool->ev[20], &h2d, body));
    CK(pool, cudaEventRecord(pool->ev[21], st));
    return COOK_OK;
  }
  // copies straight into device columns, nothing staged: body(Carve&) runs once, with only Carve::copy, between ev[20]
  // and ev[21]
  template <class Body>
  int32_t direct(const Body& body) {
    CK(pool, cudaEventRecord(pool->ev[20], st));
    Carve c;
    c.st = st;
    body(c);
    CK(pool, c.err);
    h2d += c.h2d;
    CK(pool, cudaEventRecord(pool->ev[21], st));
    return COOK_OK;
  }
  int32_t end() {
    CK(pool, cudaGetLastError());
    CK(pool, cudaEventRecord(pool->ev[22], st));
    CK(pool, cudaStreamSynchronize(st));
    record_phase(pool, COOK_PHASE_STATE, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[22], h2d, d2h, nl);
    return COOK_OK;
  }
};

void offers_drop(PoolState* S);

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
    S->jobs_r.clear();
    S->cot_rows = S->cot_n = S->grp_rows = 0;
    S->rec.tail = S->rec.n_live = 0;
    S->rec_groups.clear();
    S->hist.tail = S->hist.since = 0;
    S->hist.on = false;
    S->cj.clear_rows();
    S->cj.since = 0;
    S->cj.on = false;
    S->reserved.clear();
    for (auto& f : S->nflag) f = 0;
    for (auto& l : S->lists) l.tail = l.live = 0;
    if (S->offer.hw) CK(pool, cudaMemsetAsync(S->offer.col[O_LIVE], 0, (size_t)S->offer.hw, st));
    offers_drop(S);
    S->jf_keyed = 0;
    S->mm.on = false;
    S->mm.u_n = 0;
    if (!S->parked.empty()) CK(pool, cudaMemsetAsync(S->park[0], 0, (size_t)S->park.cap, st));
    S->parked.clear();
    S->retry.clear();
    for (auto& l : S->park_len) l = 0;
  }
  if (rs || np || npr) S->pend_epoch++;
  // a pending upsert or removal drops the job's retry facts; an upsert frees its parked copy (the caller's row wins)
  std::vector<int32_t> unparked;
  if (!S->retry.empty()) {
    for (int i = 0; i < npr; i++) S->retry.erase(d->pending_rm_job_id[i]);
    for (int i = 0; i < np; i++) {
      S->retry.erase(d->pending_job_id[i]);
      S->unpark(d->pending_job_id[i], &unparked);
    }
  }
  std::vector<int32_t> prm_slot(npr), pup_slot(np), rrm_slot(nrr), rup_slot(nr);
  for (int i = 0; i < npr; i++) {
    auto it = S->pend.slot_of.find(d->pending_rm_job_id[i]);
    const int32_t s = it->second;
    S->pend.slot_of.erase(it);
    S->add_pending(s, S->pinfo[s], -1);
    S->pinfo[s].touched = S->pend_epoch;
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
    pi.novel.assign(P.novel_off ? P.novel_host + P.novel_off[i] : nullptr, P.novel_off ? P.novel_host + P.novel_off[i + 1] : nullptr);
    const bool f[F_N] = {P.gpus && P.gpus[i] != 0.0, P.ports && P.ports[i] != 0, P.allowed && !P.allowed[i],
                         P.plugin_accept && !P.plugin_accept[i], P.gpu_model && P.gpu_model[i] != -1,
                         P.disk_request && P.disk_request[i] >= 0.0, P.est_end_ms && P.est_end_ms[i] != -1,
                         P.ckpt_location && P.ckpt_location[i] != -1, P.reserved_host && P.reserved_host[i] != -1};
    pi.flags = 0;
    for (int k = 0; k < F_N; k++) if (f[k]) pi.flags |= (uint16_t)(1u << k);
    pi.jf = 0;
    pi.touched = S->pend_epoch;
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
    S->rstart[s] = T.start_time[i];
    S->rfacts[s] = 0;
    S->rreason[s] = -1;
    S->rjid[s] = T.job_id[i]; S->rtid[s] = T.task_id[i];
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
  ScatterArgs pu, pr, ru, rr, uk;
  memset(&pu, 0, sizeof(pu)); memset(&pr, 0, sizeof(pr)); memset(&ru, 0, sizeof(ru)); memset(&rr, 0, sizeof(rr));
  memset(&uk, 0, sizeof(uk));
  const int nuk = (int)unparked.size();
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (nuk) {
      uk.c[0] = ScatterCol{S->park.at<char>(0), nullptr, 0, 1};
      uk.nc = 1;
      uk.slot = c.up(unparked.data(), nuk);
    }
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
      for (const ResetCol& r : PENDING_UPSERT_RESETS)
        pu.c[pu.nc++] = ScatterCol{static_cast<char*>(S->pend.col[r.col]), nullptr, r.dflt, P_SZ[r.col]};
      pu.slot = c.up(pup_slot.data(), np);
      for (int l = 0; l < 3; l++) {
        pu.doff[l] = c.up(lists_off[l], np + 1);
        const int64_t nv = lists_off[l] ? lists_off[l][np] : 0;
        if (c.base && nv) S->lists[l].v.copy(c, tail0[l], nv, {lists_v[l][0], lists_v[l][1]});
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
      for (const ResetCol& r : RUNNING_UPSERT_RESETS)
        ru.c[ru.nc++] = ScatterCol{static_cast<char*>(S->run.col[r.col]), nullptr, r.dflt, R_SZ[r.col]};
      ru.slot = c.up(rup_slot.data(), nr);
      ru.doff[0] = c.up(rgo, nr + 1);
      if (c.base && radd) RG.v.copy(c, rtail0, radd, {d->running_group_idx});
    }
    if (nrr) rr.slot = c.up(rrm_slot.data(), nrr);
  }))
    return rc;
  scatter(pr, S->pend, npr, 0, P_LIVE, tail0, st, &w.nl);
  scatter(rr, S->run, nrr, 0, R_LIVE, &rtail0, st, &w.nl);
  scatter(pu, S->pend, np, 1, P_LIVE, tail0, st, &w.nl);
  scatter(ru, S->run, nr, 1, R_LIVE, &rtail0, st, &w.nl);
  scatter(uk, S->pend, nuk, 0, -1, nullptr, st, &w.nl);
  if (int32_t rc = compact_lists(pool, S, st, &w.nl)) return rc;
  return w.end();
}

// pending_rm = job_id plus the running upserts built from the rows, without their columns crossing the bus
int32_t launch(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* job_id, const int64_t* task_id,
               const int64_t* start_time, const int32_t* hostname_id) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && (!job_id || !task_id || !start_time))
    return set_err(pool, COOK_E_BADARG, "%s: null job_id, task_id or start_time", who);
  if (!idx_in_range(hostname_id, n, -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "%s: a hostname code below -1", who);
  std::vector<int32_t> pslot, rslot(n);
  if (int32_t rc = live_slots(pool, who, S->pend, "job", n, job_id, &pslot)) return rc;
  {
    std::unordered_set<int64_t> seen;
    seen.reserve((size_t)n);
    for (int i = 0; i < n; i++) {
      if (!seen.insert(task_id[i]).second) return set_err(pool, COOK_E_BADARG, "%s: task id twice", who);
      if (S->run.slot_of.count(task_id[i])) return set_err(pool, COOK_E_BADARG, "%s: task id already running", who);
    }
  }
  cudaStream_t st = pool->stream;
  // ---- host side, in cook_state_apply's order: the removals free their slots, then the tasks take theirs.  A job
  // with retry facts parks its slot instead of freeing it.
  if (n) S->pend_epoch++;
  std::vector<int32_t> kslot, fslot;   // parked and freed slots, when some job parks
  for (int i = 0; i < n; i++) {
    const int32_t s = pslot[i];
    S->pend.slot_of.erase(job_id[i]);
    S->add_pending(s, S->pinfo[s], -1);
    S->pinfo[s].touched = S->pend_epoch;
    if (!S->retry.empty() && S->retry.count(job_id[i])) {
      S->parked.emplace(job_id[i], s);
      for (int l = 0; l < 3; l++) S->park_len[l] += S->pinfo[s].len[l];
      kslot.push_back(s);
    } else {
      S->pend.free.push_back(s);
      fslot.push_back(s);
    }
  }
  const int nk = (int)kslot.size();
  if (!nk) fslot.clear();   // the removal takes every row
  int64_t ng = 0;   // group list entries that move with the jobs
  for (int i = 0; i < n; i++) {
    const int32_t r = S->run.take_slot();
    S->run.slot_of.emplace(task_id[i], r);
    S->running_room(r);
    S->ruser[r] = S->pinfo[pslot[i]].user;
    S->rhost[r] = hostname_id ? hostname_id[i] : -1;
    S->rgroups[r] = S->pinfo[pslot[i]].groups;
    S->rstart[r] = start_time[i];
    S->rfacts[r] = 0;
    S->rreason[r] = -1;
    S->rjid[r] = job_id[i]; S->rtid[r] = task_id[i];
    S->add_running(r, +1);
    ng += (int64_t)S->rgroups[r].size();
    rslot[i] = r;
  }
  // ---- device: capacity, the upload, the move (rows, then group lists), the pending slots' removal, then the
  // arena rule
  CK(pool, S->run.grow(S->run.hw, st));
  if (nk) CK(pool, S->park_room(st));
  ListArena& RG = S->lists[L_RGROUP];
  const int32_t rtail0 = (int32_t)RG.tail;
  CK(pool, RG.grow(RG.tail + ng, st));
  RG.tail += ng;
  const int32_t *d_pslot = nullptr, *d_rslot = nullptr, *d_host = nullptr, *d_kslot = nullptr, *d_fslot = nullptr;
  const int64_t *d_tid = nullptr, *d_start = nullptr;
  OrderScan<int, 1> os;
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (!n) return;
    d_pslot = c.up(pslot.data(), n); d_rslot = c.up(rslot.data(), n);
    d_tid = c.up(task_id, n); d_start = c.up(start_time, n);
    d_host = c.up(hostname_id, n);
    if (nk) { d_kslot = c.up(kslot.data(), nk); d_fslot = c.up(fslot.data(), fslot.size()); }
    if (ng) {   // device-only buffers: nothing uploaded
      os.part[0] = c.take<int32_t>(n);
      os.tile[0] = c.take<int32_t>((n + OS_TILE - 1) / OS_TILE + 1);
    }
  }))
    return rc;
  if (n) {
    launch_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_pslot, d_rslot, d_tid, d_start, d_host, S->pend.d_col,
                                                   S->run.d_col, n, rtail0);
    w.nl++;
    if (ng) {
      const int32_t* plen = S->pend.at<int32_t>(P_GLEN);
      order_scan(os, RowLen{d_pslot, plen}, n, S->gf0, st, &w.nl);
      launch_lists_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, d_pslot, d_rslot, n, S->pend.at<int32_t>(P_GOFF), plen,
                                                       S->lists[L_GROUP].at(0), static_cast<int32_t*>(S->run.col[R_GOFF]),
                                                       static_cast<int32_t*>(S->run.col[R_GLEN]), RG.at(0), rtail0);
      w.nl++;
    }
    ScatterArgs rm;
    memset(&rm, 0, sizeof(rm));
    rm.slot = nk ? d_fslot : d_pslot;
    int32_t tail[3];
    for (int l = 0; l < 3; l++) tail[l] = (int32_t)S->lists[l].tail;
    scatter(rm, S->pend, n - nk, 0, P_LIVE, tail, st, &w.nl);
    if (nk) {   // parking: the live flag cleared and the generation bumped as a removal's, the lists kept
      ScatterArgs pk;
      memset(&pk, 0, sizeof(pk));
      pk.c[0] = ScatterCol{S->park.at<char>(0), nullptr, 1, 1};
      pk.nc = 1;
      pk.slot = d_kslot;
      scatter(pk, S->pend, nk, 0, P_LIVE, nullptr, st, &w.nl);
    }
  }
  if (int32_t rc = compact_lists(pool, S, st, &w.nl)) return rc;
  return w.end();
}

// the given match-time columns of live pending rows, in place; clear: every reservation is dropped first
int32_t patch(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* job_id, const uint8_t* allowed,
              const uint8_t* plugin_accept, const int32_t* reserved_host, bool clear) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && !job_id) return set_err(pool, COOK_E_BADARG, "%s: null job_id", who);
  if (!idx_in_range(reserved_host, n, -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "%s: a reserved_host below -1", who);
  std::vector<int32_t> slot;
  if (int32_t rc = live_slots(pool, who, S->pend, "job", n, job_id, &slot)) return rc;
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
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (nc) {
      cl.c[0] = ScatterCol{static_cast<char*>(S->pend.col[P_RESERVED]), nullptr, -1, P_SZ[P_RESERVED]};
      cl.nc = 1;
      cl.slot = c.up(cleared.data(), nc);
    }
    if (cols)
      patch_args(c, pa, S->pend, slot.data(), n,
                 {{P_ALLOWED, allowed, 1}, {P_PLUGIN, plugin_accept, 1}, {P_RESERVED, reserved_host, -1}});
  }))
    return rc;
  scatter(cl, S->pend, nc, 0, -1, nullptr, w.st, &w.nl);
  scatter(pa, S->pend, cols ? n : 0, 0, -1, nullptr, w.st, &w.nl);
  return w.end();
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

// ---- the gather step of the reads whose handles may span devices (DESIGN.md §9a): cook_state_user_stats,
// cook_state_instance_stats, cook_state_history_stats and cook_state_list_completed compact each handle's rows into
// one dense range carved from pools[0]'s scratch, a handle's rows at `base`, after those of the handles before it.
// A handle on pools[0]'s device compacts straight into that range on pools[0]'s stream.  A handle on another device
// runs the same functor on its own device and stream into staging columns, a count and blk carved from its own
// scratch; pools[0]'s stream waits on an event recorded there and copies each packed column to `base` with
// cudaMemcpyPeerAsync (peer access is not enabled; no device or context setting changes).  Only the rows the
// compaction keeps cross, rows x the functor's bytes per row.  Handle order and base are those of one device, so the
// leader's pipeline reads the same rows in the same places.  COOK_STAGE_HANDLES=1 in the environment (read per call)
// sends every handle after pools[0] through the staging even on pools[0]'s device, so that one GPU runs the path.
// A gathered functor lists its output columns with outs(visitor) (a null column is not carved) and reads only its own
// handle's tables, so no call-wide array has to exist on the handle's device.
bool stage_handles() {
  const char* e = getenv("COOK_STAGE_HANDLES");
  return e && strcmp(e, "1") == 0;
}

struct Gather {
  static constexpr int MAXO = 8;   // the most output columns a gathered functor has
  cook_pool* lead;
  bool all = stage_handles();
  std::vector<const cook_pool*> used;   // the handles whose staging this call has filled

  explicit Gather(cook_pool* p) : lead(p) {}
  bool staged(const cook_pool* h) const { return h != lead && (all || h->device != lead->device); }

  // body() with handle h's device current; pools[0]'s device current again afterwards
  template <class Body>
  cudaError_t on(const cook_pool* h, const Body& body) const {
    cudaError_t e = cudaSetDevice(h->device);
    if (e == cudaSuccess) e = body();
    const cudaError_t back = cudaSetDevice(lead->device);
    return e != cudaSuccess ? e : back;
  }

  // Handle h's compaction f (its base and output columns those of pools[0]'s range) over n_max items, `rows` of them
  // kept.  Not staged: on pools[0]'s stream with blk and cnt (the call's own).  Counts its launches in *nl.
  template <class F>
  cudaError_t rows(cook_pool* h, const F& f, int n_max, int rows, int32_t* blk, int32_t* cnt, int* nl) {
    if (!staged(h)) {
      compact(f, n_max, nullptr, blk, cnt, rows, lead->stream, nl);
      return cudaGetLastError();
    }
    F g = f;
    char *dst[MAXO], *src[MAXO];
    size_t sz[MAXO];
    int nc = 0;
    g.outs([&](auto* p) {
      if (p) { dst[nc] = reinterpret_cast<char*>(p); sz[nc++] = sizeof(*p); }
    });
    // staging a second time in one call: its columns are free once pools[0]'s copies of the first have run
    const bool again = std::find(used.begin(), used.end(), h) != used.end();
    if (again) {
      cudaError_t e = cudaEventRecord(lead->ev[19], lead->stream);
      if (e != cudaSuccess) return e;
    } else {
      used.push_back(h);
    }
    cudaError_t e = on(h, [&]() -> cudaError_t {
      if (again) {
        const cudaError_t w = cudaStreamWaitEvent(h->stream, lead->ev[19], 0);
        if (w != cudaSuccess) return w;
      }
      PoolState* R = state_of(const_cast<cook_pool*>(h), false);   // h holds the rows
      int32_t *s_blk = nullptr, *s_cnt = nullptr;
      const cudaError_t c = carve(R->scratch, h->stream, nullptr, nullptr, [&](Carve& cv) {
        s_cnt = cv.take<int32_t>(1);
        s_blk = cv.take<int32_t>((size_t)n_max / CP_BLOCK + 2);
        for (int k = 0; k < nc; k++) src[k] = cv.take<char>(sz[k] * (size_t)rows);
      });
      if (c != cudaSuccess) return c;
      int k = 0;
      g.outs([&](auto*& p) {
        if (p) p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(src[k++]);
      });
      g.base = 0;
      compact(g, n_max, nullptr, s_blk, s_cnt, rows, h->stream, nl);
      const cudaError_t l = cudaGetLastError();
      return l != cudaSuccess ? l : cudaEventRecord(h->ev[20], h->stream);
    });
    if (e != cudaSuccess) return e;
    if ((e = cudaStreamWaitEvent(lead->stream, h->ev[20], 0)) != cudaSuccess) return e;
    for (int k = 0; k < nc; k++)
      if ((e = cudaMemcpyPeerAsync(dst[k] + sz[k] * (size_t)f.base, lead->device, src[k], h->device,
                                   sz[k] * (size_t)rows, lead->stream)) != cudaSuccess)
        return e;
    return cudaSuccess;
  }
};

// The usage of R live rows of one or more handles, each sum a left fold in ascending id: per user (U > 0), per
// listed host (H > 0, running rows only) and of the pool.  The running rows by task id, or (pending) the pending rows
// by job id; an id several handles hold, in handle order.  The caller sets rows.host_of / rows.n_codes (H > 0) and
// the destinations a.user_out [4][U], a.host_cpus / host_mem / host_count [H] and a.pool_out [4] of the sums it
// asked for.  take's hw: the largest slot high-water mark of the table among the handles.
struct UsageFold {
  int R = 0, U = 0, H = 0;
  bool pool = false, pending = false;
  UsageRows rows = {};
  UsageArgs a = {};
  int32_t *blk = nullptr, *tmp = nullptr;
  GridFlag* gf = nullptr;

  void take(Carve& c, int hw) {
    rows.user = c.take<int32_t>(R); rows.id = c.take<int64_t>(R);
    for (int k = 0; k < 3; k++) rows.amt[k] = c.take<double>(R);
    blk = c.take<int32_t>((size_t)hw / CP_BLOCK + 2);
    tmp = c.take<int32_t>(R);
    gf = c.take<GridFlag>(1);
    if (U > 0) take_segs(c, US_USER, U, true);
    if (H > 0) {
      rows.host = c.take<int32_t>(R);
      take_segs(c, US_HOST, H, true);
    }
    if (pool) take_segs(c, US_POOL, 1, false);
  }
  // kind k's order of the R rows; with bounds, its n_seg segments' bounds and the order-wide scan
  void take_segs(Carve& c, int k, int n_seg, bool bounds) {
    UsageSegs& q = a.seg[k];
    q.n = n_seg;
    q.ord = c.take<int32_t>(R);
    if (!bounds) return;
    q.start = c.take<int32_t>(n_seg + 1); q.end = c.take<int32_t>(n_seg + 1);
    q.scan = 1;
    for (int j = 0; j < 3; j++) {
      q.os.part[j] = c.take<double>(R);
      q.os.tile[j] = c.take<double>(R / OS_TILE + 2);
    }
  }

  // the live rows of handles S[0, n) (their counts in S[0]'s counters), then fold().  With a gather g, hp[k] is S[k]'s
  // handle and g->lead S[0]'s (cook_state_user_stats: the handles may span devices; no host is listed then).
  cudaError_t run(const PoolState* const* S, int n, cudaStream_t st, int* nl, Gather* g = nullptr,
                  cook_pool* const* hp = nullptr) {
    rows.c = pending ? PEND_COLS : RUN_COLS; rows.H = H;
    rows.base = 0;
    for (int k = 0; k < n; k++) {
      const Table& t = pending ? S[k]->pend : S[k]->run;
      const int live = (int)t.slot_of.size();
      if (!live) continue;
      rows.col = t.d_col;
      int32_t* cnt = S[0]->counters + (pending ? 1 : 0);
      if (g) {
        const cudaError_t e = g->rows(hp[k], rows, t.hw, live, blk, cnt, nl);
        if (e != cudaSuccess) return e;
      } else {
        compact(rows, t.hw, nullptr, blk, cnt, live, st, nl);
      }
      rows.base += live;
    }
    return fold(st, nl);
  }

  // Over rows.user / id / amt (and host) [0, R): the grid check, each kind's order by (key, id) with its segments
  // and (on the grid) order-wide scan, the folds.  Needs tmp, gf, a.user_out and the kinds take_segs carved.
  cudaError_t fold(cudaStream_t st, int* nl) {
    cudaError_t e = cudaMemsetAsync(gf, 0, sizeof(GridFlag), st);
    if (e != cudaSuccess) return e;
    grid_check_kernel<<<(R + 255) / 256, 256, 0, st>>>(rows.amt[0], rows.amt[1], rows.amt[2], R, gf);
    (*nl)++;
    const int32_t* key[US_N] = {rows.user, rows.host, nullptr};
    for (int k = 0; k < US_N; k++) {
      UsageSegs& q = a.seg[k];
      if (!q.n) continue;
      if ((e = csort::sort_indices(writable(q.ord), tmp, R, LessKeyTid{key[k], rows.id}, st, nl)) != cudaSuccess) return e;
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
    a.goff = S->run.at<int32_t>(R_GOFF); a.glen = S->run.at<int32_t>(R_GLEN); a.arena = S->lists[L_RGROUP].at(0);
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
  CK(pool, f.run(&S, 1, st, &nl));
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
  CK(pool, f.run(&S, 1, st, nl));
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

// ---- the live offers (Fenzo's leases): added once as they arrive, expired, merged per hostname and consumed here
// the live offers, dense, with their VM (host_of their hostname code) and arrival sequence
struct OfferRows {
  void* const* col; const int32_t* host_of; int32_t* vm; int64_t* seq; int32_t* slot;
  __device__ bool keep(int i) const { return static_cast<const uint8_t*>(col[O_LIVE])[i]; }
  __device__ void emit(int i, int d) const {
    slot[d] = i;
    vm[d] = host_of[static_cast<const int32_t*>(col[O_CODE])[i]];
    seq[d] = static_cast<const int64_t*>(col[O_SEQ])[i];
  }
};
// position p of the (VM, sequence) order: its slot, and the VMs' segments [start, end)
__global__ void offer_order_kernel(const int32_t* ord, const int32_t* vm, const int32_t* slot, int n, int32_t* ss,
                                   int32_t* start, int32_t* end) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  ss[p] = slot[ord[p]];
  mark_segment(p, n, SortedKey{ord, nullptr, vm}, start, end);
}
struct MergeArgs {
  void* const* col; const int32_t* ss; const int32_t* start; const int32_t* end; int O;
  OrderScan<int, 1> ports;   // the port ranges' scan over the order (when the plan has ports)
  const int32_t* attr_arena; // the offers' attribute rows
  OfferCols oc; int n_attr_cols;
  int32_t* newest;           // [O] the slot of each VM's newest offer
};
// thread per VM: cpus and mem as left folds over its offers in arrival order, every other column from its newest
__global__ void offer_merge_kernel(MergeArgs a) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.O) return;
  const double* oc = static_cast<const double*>(a.col[O_CPUS]);
  const double* om = static_cast<const double*>(a.col[O_MEM]);
  const int s = a.start[v], e = a.end[v];
  double cpus = 0.0, mem = 0.0;
  for (int p = s; p < e; p++) {
    const int i = a.ss[p];
    cpus = cpus + oc[i];
    mem = mem + om[i];
  }
  const int i = a.ss[e - 1];
  a.oc.perm[v] = v;
  a.oc.cpus[v] = cpus;
  a.oc.mem[v] = mem;
  a.newest[v] = i;
  if (a.oc.port_off) {
    a.oc.port_off[v + 1] = a.ports.at(0, e - 1);
    if (v == 0) a.oc.port_off[0] = 0;
  }
  if (a.oc.is_k8s) a.oc.is_k8s[v] = static_cast<const uint8_t*>(a.col[O_K8S])[i];
  if (a.oc.location) a.oc.location[v] = static_cast<const int32_t*>(a.col[O_LOC])[i];
  if (a.oc.max_tasks) a.oc.max_tasks[v] = static_cast<const int32_t*>(a.col[O_MAXT])[i];
  if (a.oc.num_tasks) a.oc.num_tasks[v] = static_cast<const int32_t*>(a.col[O_NUMT])[i];
  if (a.oc.host_start) a.oc.host_start[v] = static_cast<const int64_t*>(a.col[O_START])[i];
  if (a.oc.reserved) a.oc.reserved[v] = 0;
  const int ao = static_cast<const int32_t*>(a.col[O_AOFF])[i], al = static_cast<const int32_t*>(a.col[O_ALEN])[i];
  for (int c = 0; c < a.n_attr_cols; c++) a.oc.attr[(size_t)c * a.O + v] = c < al ? a.attr_arena[ao + c] : 0;
}
// thread per host of a rebalance's table: the spare resources of its live offers (view-incubating-offers), cpus, mem
// and the offers' "gpus" as left folds in arrival order; a host without a live offer keeps has_spare 0
__global__ void offer_spare_kernel(void* const* col, const int32_t* ss, const int32_t* start, const int32_t* end, int H,
                                   uint8_t* has, double* sc, double* sm, double* sg) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H || start[h] >= end[h]) return;
  const double* oc = static_cast<const double*>(col[O_CPUS]);
  const double* om = static_cast<const double*>(col[O_MEM]);
  const double* og = static_cast<const double*>(col[O_GPUS]);
  double c = 0.0, m = 0.0, g = 0.0;
  for (int p = start[h]; p < end[h]; p++) {
    const int i = ss[p];
    c = c + oc[i];
    m = m + om[i];
    g = g + og[i];
  }
  has[h] = 1; sc[h] = c; sm[h] = m; sg[h] = g;
}

// the hosts some live pending row has as reserved_host: pending slots pslot[0, n)
__global__ void offer_reserved_kernel(const int32_t* pslot, int n, const int32_t* reserved_host, const int32_t* host_of,
                                      int32_t n_codes, uint8_t* reserved) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int32_t c = reserved_host[pslot[k]];
  if (c >= 0 && c < n_codes && host_of[c] >= 0) reserved[host_of[c]] = 1;
}

// One cook_state_match_offers: the check table it starts from, the VMs and the plan's offer shape after the expiry,
// the offers that left (slot, fate, sequence), the uploads and launches of the expiry and the consumption.
struct OfferPass {
  int64_t now_ms = 0, incubate_ms = 0;
  int32_t dummy = 0;
  cook_offers_soa check = {};   // what the checks read before the expiry: no column is uploaded from it
  std::vector<int32_t> codes;   // the VMs' hostname codes in name order
  int32_t n_codes = 0;
  OfferShape osh;
  std::vector<std::pair<int64_t, std::pair<int64_t, uint8_t>>> gone;   // (seq, (id, fate))
  int64_t h2d = 0;
  int nl = 0;
};

// a hostname code's newest live offer enters (+1) or leaves (-1) the VM counts
void vm_touch(PoolState* S, OfferHost& h, int64_t sign) {
  if (h.live.empty()) return;
  const OfferInfo& oi = S->oinfo[h.live.rbegin()->second];
  S->vm_gpu += sign * oi.len[OL_GPU];
  S->vm_disk += sign * oi.len[OL_DISK];
  S->vm_k8s += sign * (oi.k8s ? 1 : 0);
  S->vm_maxt += sign * (oi.max_tasks ? 1 : 0);
}

// offer slot s enters (+1) or leaves (-1) the host-side bookkeeping
void offer_count(PoolState* S, int32_t s, int64_t sign) {
  const OfferInfo& oi = S->oinfo[s];
  OfferHost& h = S->ohost[oi.code];
  vm_touch(S, h, -1);
  if (sign > 0) {
    if (h.live.empty()) S->vm_names.emplace(h.name, oi.code);
    h.live.emplace(oi.seq, s);
    S->by_time.emplace(std::make_pair(oi.received, oi.seq), s);
    if (oi.single_shot) S->single_shot.emplace(oi.seq, s);
  } else {
    h.live.erase(oi.seq);
    if (h.live.empty()) S->vm_names.erase(h.name);
    S->by_time.erase(std::make_pair(oi.received, oi.seq));
    S->single_shot.erase(oi.seq);
  }
  vm_touch(S, h, +1);
  S->o_ports += sign * oi.len[OL_PORT];
  for (int l = 0; l < OL_N; l++) S->olists[l].live += sign * oi.len[l];
  count_add(S->owidth, oi.len[OL_ATTR], sign);
}

// slots leave: the host side, then one removal scatter (its upload and launch into *h2d, *nl)
int32_t offers_remove(cook_pool* pool, PoolState* S, const std::vector<int32_t>& slots, int64_t* h2d, int* nl) {
  if (slots.empty()) return COOK_OK;
  for (int32_t s : slots) {
    offer_count(S, s, -1);
    S->offer.slot_of.erase(S->oinfo[s].id);
    S->offer.free.push_back(s);
  }
  cudaStream_t st = pool->stream;
  ScatterArgs a;
  memset(&a, 0, sizeof(a));
  CK(pool, carve(S->stage, st, nullptr, h2d, [&](Carve& c) { a.slot = c.up(slots.data(), slots.size()); }));
  scatter(a, S->offer, (int)slots.size(), 0, O_LIVE, nullptr, st, nl);
  CK(pool, cudaGetLastError());
  return COOK_OK;
}

// drop every live offer (a reset); the names stay known
void offers_drop(PoolState* S) {
  for (auto& kv : S->ohost) kv.second.live.clear();
  S->offer.slot_of.clear(); S->offer.free.clear(); S->offer.hw = 0;
  S->vm_names.clear(); S->by_time.clear(); S->single_shot.clear(); S->owidth.clear();
  S->o_ports = S->vm_gpu = S->vm_disk = S->vm_k8s = S->vm_maxt = 0;
  for (auto& l : S->olists) l.tail = l.live = 0;
}

int32_t offers_add(cook_pool* pool, PoolState* S, const char* who, const cook_offers_soa* o, const int64_t* id,
                   const uint8_t* single, const double* gpus, const char* name, const int32_t* name_off, int64_t now_ms) {
  if (!o) return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  const int n = o->n;
  if (n < 0 || o->n_attr_cols < 0) return set_err(pool, COOK_E_BADARG, "%s: bad sizes", who);
  if (n == 0) {
    pool->phase[COOK_PHASE_STATE] = {};
    return COOK_OK;
  }
  if (!id || !o->hostname_id || !o->cpus || !o->mem || (o->n_attr_cols > 0 && !o->attr))
    return set_err(pool, COOK_E_BADARG, "%s: offers need offer_id, hostname_id, cpus and mem", who);
  const int32_t* gpu_cnt = reinterpret_cast<const int32_t*>(o->gpu_count);
  const int32_t* disk_sp = reinterpret_cast<const int32_t*>(o->disk_space);
  if (!csr_ok(o->port_off, n, o->port_begin, o->port_end, true) || !csr_ok(o->gpu_off, n, o->gpu_model, gpu_cnt, true) ||
      !csr_ok(o->disk_off, n, o->disk_type, disk_sp, true) ||
      (name_off && !csr_ok(name_off, n, reinterpret_cast<const int32_t*>(name), nullptr, false)))
    return set_err(pool, COOK_E_BADARG, "%s: malformed CSR offsets", who);
  // ids, codes and names, all before any change
  std::unordered_set<int64_t> seen;
  seen.reserve((size_t)n);
  std::unordered_map<int32_t, std::string> batch_name;   // code -> name given in this batch
  std::unordered_map<std::string, int32_t> batch_code;   // name -> code given in this batch
  for (int i = 0; i < n; i++) {
    if (!seen.insert(id[i]).second || S->offer.slot_of.count(id[i]))
      return set_err(pool, COOK_E_BADARG, "%s: an offer id is live already or twice in the batch", who);
    const int32_t code = o->hostname_id[i];
    if (code < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative hostname code", who);
    const int len = name_off ? name_off[i + 1] - name_off[i] : 0;
    if (!len) continue;
    const std::string nm(name + name_off[i], (size_t)len);
    auto h = S->ohost.find(code);
    auto k = S->code_of_name.find(nm);
    auto bn = batch_name.find(code);
    auto bc = batch_code.find(nm);
    if ((h != S->ohost.end() && h->second.name != nm) || (k != S->code_of_name.end() && k->second != code) ||
        (bn != batch_name.end() && bn->second != nm) || (bc != batch_code.end() && bc->second != code))
      return set_err(pool, COOK_E_BADARG, "%s: a hostname code with two names or a name with two codes", who);
    batch_name.emplace(code, nm);
    batch_code.emplace(nm, code);
  }
  for (int i = 0; i < n; i++) {
    const int32_t code = o->hostname_id[i];
    if (!S->ohost.count(code) && !batch_name.count(code))
      return set_err(pool, COOK_E_BADARG, "%s: a new hostname code without a name", who);
  }
  cudaStream_t st = pool->stream;
  // ---- the host side, O(batch)
  for (const auto& kv : batch_name) {
    if (S->ohost.count(kv.first)) continue;
    S->ohost[kv.first].name = kv.second;
    S->code_of_name.emplace(kv.second, kv.first);
  }
  const int W = o->n_attr_cols;
  std::vector<int32_t> slot(n);
  std::vector<int64_t> seq(n);
  for (int i = 0; i < n; i++) {
    const int32_t s = S->offer.take_slot();
    S->offer.slot_of.emplace(id[i], s);
    if ((size_t)s >= S->oinfo.size()) S->oinfo.resize(std::max<size_t>(s + 1, 2 * S->oinfo.size()));
    OfferInfo& oi = S->oinfo[s];
    oi.id = id[i]; oi.seq = seq[i] = S->next_seq++; oi.received = now_ms; oi.code = o->hostname_id[i];
    oi.len[OL_PORT] = o->port_off ? o->port_off[i + 1] - o->port_off[i] : 0;
    oi.len[OL_GPU] = o->gpu_off ? o->gpu_off[i + 1] - o->gpu_off[i] : 0;
    oi.len[OL_DISK] = o->disk_off ? o->disk_off[i + 1] - o->disk_off[i] : 0;
    oi.len[OL_ATTR] = W;
    oi.single_shot = single && single[i];
    oi.k8s = o->is_k8s && o->is_k8s[i];
    oi.max_tasks = o->max_tasks && o->max_tasks[i] != -1;
    offer_count(S, s, +1);
    slot[i] = s;
  }
  // the attribute rows, row-major: row i's W values at i * W
  std::vector<int32_t> attr_rows((size_t)n * W), attr_off(W ? n + 1 : 0);
  for (int i = 0; i < n && W; i++) {
    for (int c = 0; c < W; c++) attr_rows[(size_t)i * W + c] = o->attr[(size_t)c * n + i];
    attr_off[i] = i * W;
  }
  if (W) attr_off[n] = n * W;
  // ---- device: capacity, the upload, the scatter
  CK(pool, S->offer.grow(S->offer.hw, st));
  const int32_t* loff[OL_N] = {o->port_off, o->gpu_off, o->disk_off, W ? attr_off.data() : nullptr};
  const int32_t* lv0[OL_N] = {o->port_begin, o->gpu_model, o->disk_type, attr_rows.data()};
  const void* lv1[OL_N] = {o->port_end, o->gpu_count, o->disk_space, nullptr};
  int32_t tail0[OL_N];
  int64_t nv[OL_N];
  for (int l = 0; l < OL_N; l++) {
    ListArena& A = S->olists[l];
    tail0[l] = (int32_t)A.tail;
    nv[l] = loff[l] ? loff[l][n] : 0;
    CK(pool, A.grow(A.tail + nv[l], st));
    A.tail += nv[l];
  }
  ScatterArgs a;
  memset(&a, 0, sizeof(a));
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    const void* src[O_NDATA] = {o->hostname_id, o->cpus, o->mem, gpus, o->is_k8s, o->location, o->max_tasks,
                                o->num_tasks, o->host_start_time, seq.data()};
    const long long dflt[O_NDATA] = {0, 0, 0, 0, 0, -1, -1, 0, -1, 0};
    for (int k = 0; k < O_NDATA; k++) {
      const char* up = nullptr;
      if (O_SZ[k] == 1) up = reinterpret_cast<const char*>(c.up(static_cast<const uint8_t*>(src[k]), n));
      else if (O_SZ[k] == 4) up = reinterpret_cast<const char*>(c.up(static_cast<const int32_t*>(src[k]), n));
      else up = reinterpret_cast<const char*>(c.up(static_cast<const int64_t*>(src[k]), n));
      a.c[k] = ScatterCol{static_cast<char*>(S->offer.col[k]), up, dflt[k], O_SZ[k]};
    }
    a.nc = O_NDATA;
    a.slot = c.up(slot.data(), n);
    for (int l = 0; l < OL_N; l++) {
      a.doff[l] = c.up(loff[l], n + 1);
      if (c.base && nv[l]) S->olists[l].v.copy(c, tail0[l], nv[l], {lv0[l], lv1[l]});
    }
  }))
    return rc;
  scatter(a, S->offer, n, 1, O_LIVE, tail0, st, &w.nl);
  if (int32_t rc = compact_lists(pool, S, st, &w.nl)) return rc;
  return w.end();
}

// step (a) and the plan's offer shape: the offers received incubate_ms or more before now_ms leave, then the VMs are
// the hostname codes with a live offer, in name order.  Runs after every check of the match.
int32_t offers_expire(cook_pool* pool, PoolState* S, OfferPass* op, const cook_groups* groups) {
  std::vector<int32_t> old;
  for (auto it = S->by_time.begin(); it != S->by_time.end() && op->now_ms - it->first.first >= op->incubate_ms; ++it) {
    old.push_back(it->second);
    const OfferInfo& oi = S->oinfo[it->second];
    op->gone.push_back({oi.seq, {oi.id, (uint8_t)COOK_OFFER_EXPIRED}});
  }
  const int32_t rc = offers_remove(pool, S, old, &op->h2d, &op->nl);
  if (rc != COOK_OK) return rc;
  op->codes.clear();
  op->codes.reserve(S->vm_names.size());
  op->n_codes = 0;
  for (const auto& kv : S->vm_names) {
    op->codes.push_back(kv.second);
    op->n_codes = std::max(op->n_codes, kv.second + 1);
  }
  OfferShape& sh = op->osh;
  sh = OfferShape();
  sh.O = (int)op->codes.size();
  sh.hostname_id = op->codes.data();
  sh.ports = S->o_ports > 0; sh.n_ports = S->o_ports;
  sh.gpu = S->vm_gpu > 0; sh.n_gpu = S->vm_gpu;
  sh.disk = S->vm_disk > 0; sh.n_disk = S->vm_disk;
  sh.is_k8s = S->vm_k8s > 0;
  sh.max_tasks = S->vm_maxt > 0;
  sh.location = sh.num_tasks = sh.host_start = true;
  sh.reserved = S->nflag[F_RESERVED] > 0;
  int w = std::max<int>(count_max(S->owidth), count_max(S->attr_cols) + 1);
  for (int g = 0; groups && groups->attr_col && g < groups->n_groups; g++) w = std::max(w, groups->attr_col[g] + 1);
  sh.n_attr_cols = std::max(w, 0);
  return COOK_OK;
}

// step (b): the VMs' columns into the plan's, from the live offers
int32_t offers_merge(cook_pool* pool, PoolState* S, OfferPass& op, const MatchRows& rows, int* nl) {
  const int O = op.osh.O, L = (int)S->offer.slot_of.size();
  if (O == 0) return COOK_OK;
  cudaStream_t st = pool->stream;
  const OfferCols& oc = rows.oc;
  std::vector<int32_t> rslots(S->reserved.begin(), S->reserved.end());
  int32_t *host_of = nullptr, *vm = nullptr, *slot = nullptr, *ord = nullptr, *tmp = nullptr, *ss = nullptr;
  int32_t *start = nullptr, *end = nullptr, *blk = nullptr, *ldoff = nullptr, *newest = nullptr, *d_rslots = nullptr;
  int64_t* seq = nullptr;
  OrderScan<int, 1> osp, osg, osd;
  int64_t h2d = 0;
  CK(pool, carve(S->omerge, st, nullptr, &h2d, [&](Carve& c) {
    host_of = c.take<int32_t>(op.n_codes);
    vm = c.take<int32_t>(L); seq = c.take<int64_t>(L); slot = c.take<int32_t>(L);
    ord = c.take<int32_t>(L); tmp = c.take<int32_t>(L); ss = c.take<int32_t>(L);
    start = c.take<int32_t>(O); end = c.take<int32_t>(O); newest = c.take<int32_t>(O);
    blk = c.take<int32_t>((size_t)S->offer.hw / CP_BLOCK + 2);
    const auto scan = [&](OrderScan<int, 1>& os, int n) {
      os.part[0] = c.take<int32_t>(n);
      os.tile[0] = c.take<int32_t>((n + OS_TILE - 1) / OS_TILE + 1);
    };
    if (oc.port_off) { scan(osp, L); ldoff = c.take<int32_t>(L + 1); }
    if (oc.gpu_off) scan(osg, O);
    if (oc.disk_off) scan(osd, O);
    if (oc.reserved && !rslots.empty()) d_rslots = c.up(rslots.data(), rslots.size());
  }));
  CK(pool, map_hosts(host_of, op.n_codes, rows.hostname_id, O, st, nl));
  compact(OfferRows{S->offer.d_col, host_of, vm, seq, slot}, S->offer.hw, nullptr, blk, S->counters + 4, L, st, nl);
  CK(pool, csort::sort_indices(ord, tmp, L, LessKeyTid{vm, seq}, st, nl));
  offer_order_kernel<<<(L + 255) / 256, 256, 0, st>>>(ord, vm, slot, L, ss, start, end);
  (*nl)++;
  const ListArena* A = S->olists;
  if (oc.port_off) {
    const int32_t* plen = S->offer.at<int32_t>(O_PLEN);
    order_scan(osp, RowLen{ss, plen}, L, S->gf0, st, nl);
    csr_gather_kernel<<<(L + 7) / 8, 256, 0, st>>>(osp, ss, L, S->offer.at<int32_t>(O_POFF), plen, A[OL_PORT].at(0),
                                                   A[OL_PORT].at(1), ldoff, oc.port_begin, oc.port_end);
    (*nl)++;
  }
  MergeArgs ma = {S->offer.d_col, ss, start, end, O, osp, A[OL_ATTR].at(0), oc, op.osh.n_attr_cols, newest};
  offer_merge_kernel<<<(O + 127) / 128, 128, 0, st>>>(ma);
  (*nl)++;
  const int lists[2] = {OL_GPU, OL_DISK};
  for (int l : lists) {
    int32_t* doff = l == OL_GPU ? oc.gpu_off : oc.disk_off;
    if (!doff) continue;
    OrderScan<int, 1>& os = l == OL_GPU ? osg : osd;
    const int32_t* len = S->offer.at<int32_t>(O_POFF + 2 * l + 1);
    order_scan(os, RowLen{newest, len}, O, S->gf0, st, nl);
    csr_gather_kernel<<<(O + 7) / 8, 256, 0, st>>>(os, newest, O, S->offer.at<int32_t>(O_POFF + 2 * l), len, A[l].at(0),
                                                   A[l].v.at<double>(1), doff,
                                                   l == OL_GPU ? oc.gpu_model : oc.disk_type,
                                                   l == OL_GPU ? oc.gpu_count : oc.disk_space);
    (*nl)++;
  }
  if (d_rslots) {
    const int nr = (int)rslots.size();
    offer_reserved_kernel<<<(nr + 255) / 256, 256, 0, st>>>(d_rslots, nr, S->pend.at<int32_t>(P_RESERVED), host_of,
                                                            op.n_codes, oc.reserved);
    (*nl)++;
  }
  CK(pool, cudaGetLastError());
  op.h2d += h2d;
  return COOK_OK;
}

// a rebalance's has_spare / spare_* (rows carved them zeroed) from the live offers, at each host's table index through
// host_of (every live offer's code is in the table: checked by the caller)
int32_t offers_spare(cook_pool* pool, PoolState* S, const RebRows& rows, const int32_t* host_of, int H, int* nl) {
  const int L = (int)S->offer.slot_of.size();
  if (L == 0) return COOK_OK;
  cudaStream_t st = pool->stream;
  int32_t *vm = nullptr, *slot = nullptr, *ord = nullptr, *tmp = nullptr, *ss = nullptr, *start = nullptr;
  int32_t *end = nullptr, *blk = nullptr;
  int64_t* seq = nullptr;
  CK(pool, carve(S->omerge, st, nullptr, nullptr, [&](Carve& c) {
    vm = c.take<int32_t>(L); seq = c.take<int64_t>(L); slot = c.take<int32_t>(L);
    ord = c.take<int32_t>(L); tmp = c.take<int32_t>(L); ss = c.take<int32_t>(L);
    start = c.take<int32_t>(H); end = c.take<int32_t>(H);
    blk = c.take<int32_t>((size_t)S->offer.hw / CP_BLOCK + 2);
  }));
  CK(pool, cudaMemsetAsync(start, 0, sizeof(int32_t) * (size_t)H, st));
  CK(pool, cudaMemsetAsync(end, 0, sizeof(int32_t) * (size_t)H, st));
  compact(OfferRows{S->offer.d_col, host_of, vm, seq, slot}, S->offer.hw, nullptr, blk, S->counters + 4, L, st, nl);
  CK(pool, csort::sort_indices(ord, tmp, L, LessKeyTid{vm, seq}, st, nl));
  offer_order_kernel<<<(L + 255) / 256, 256, 0, st>>>(ord, vm, slot, L, ss, start, end);
  offer_spare_kernel<<<(H + 127) / 128, 128, 0, st>>>(S->offer.d_col, ss, start, end, H, rows.has_spare, rows.spare_cpus,
                                                      rows.spare_mem, rows.spare_gpus);
  *nl += 2;
  CK(pool, cudaGetLastError());
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_apply(cook_pool* pool, const cook_state_delta* delta) {
  const char* who = "cook_state_apply";
  if (pool && !delta) return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  return on_state(pool, who, [&](PoolState* S) { return apply(pool, S, delta); });
}

extern "C" int32_t cook_state_launch(cook_pool* pool, int32_t n, const int64_t* job_id, const int64_t* task_id,
                                     const int64_t* start_time, const int32_t* hostname_id) {
  const char* who = "cook_state_launch";
  return on_state(pool, who, [&](PoolState* S) { return launch(pool, S, who, n, job_id, task_id, start_time, hostname_id); });
}

extern "C" int32_t cook_state_patch(cook_pool* pool, int32_t n, const int64_t* job_id, const uint8_t* allowed,
                                    const uint8_t* plugin_accept, const int32_t* reserved_host,
                                    int32_t clear_reservations) {
  const char* who = "cook_state_patch";
  return on_state(pool, who, [&](PoolState* S) {
    return patch(pool, S, who, n, job_id, allowed, plugin_accept, reserved_host, clear_reservations != 0);
  });
}

extern "C" int32_t cook_state_usage(cook_pool* pool, int32_t n_users, double* out_user_usage, double* out_pool_usage,
                                    int32_t n_hosts, const int32_t* hostname_id, double* out_run_cpus,
                                    double* out_run_mem, int32_t* out_run_count) {
  return on_state(pool, "cook_state_usage", [&](PoolState* S) {
    return usage(pool, S, n_users, out_user_usage, out_pool_usage, n_hosts, hostname_id, out_run_cpus, out_run_mem,
                 out_run_count);
  });
}

extern "C" int32_t cook_state_cotasks(cook_pool* pool, int32_t n_groups, const int32_t* attr_col,
                                      const cook_host_table* hosts, int32_t cap, int32_t* out_cot_off,
                                      int32_t* out_cot_hostname_id, int32_t* out_cot_attr_val, int32_t* out_n) {
  if (!pool) return COOK_E_BADARG;
  return cotasks(pool, static_cast<PoolState*>(pool->state), n_groups, attr_col, hosts, cap, out_cot_off,
                 out_cot_hostname_id, out_cot_attr_val, out_n);
}

namespace {

// The round a match leaves for cook_state_match_metrics: its n rows' slots, copied device to device (no launch and no
// transfer between host and device), the pending epoch and the plan's run.
int32_t mm_record(cook_pool* pool, PoolState* S, const int32_t* m_slot, int n) {
  MetricsRound& R = S->mm;
  CK(pool, R.slot.grow(n, 0, pool->stream));
  if (n) CK(pool, cudaMemcpyAsync(R.slot[0], m_slot, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, pool->stream));
  R.n_rows = n;
  R.epoch = S->pend_epoch;
  R.run = match_runs(pool);
  R.on = true;
  R.counted = false;
  return COOK_OK;
}

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
  // the pool quota's start: the live running rows folded in ascending task id, cook_state_usage's pool total, not
  // the dense columns' slot order
  UsageFold pf;
  const bool pool_fold = pool_quota && pool_quota->enabled && R > 0;
  if (N > 0) {
    int32_t* blk = nullptr;
    CK(pool, carve(S->scratch, st, nullptr, nullptr, [&](Carve& c) {
      dt.user = c.take<int32_t>(N); dt.prio = c.take<int32_t>(N);
      dt.start = c.take<int64_t>(N); dt.tid = c.take<int64_t>(N); dt.jid = c.take<int64_t>(N);
      dt.cpus = c.take<double>(N); dt.mem = c.take<double>(N); dt.gpus = c.take<double>(N);
      pslot = c.take<int32_t>(J);
      blk = c.take<int32_t>((size_t)std::max(S->pend.hw, S->run.hw) / CP_BLOCK + 2);
      if (pool_fold) {
        pf.R = R; pf.pool = true;
        pf.take(c, S->run.hw);
        pf.a.pool_out = c.take<double>(4);
      }
    }));
    if (R) compact(RunningRows{S->run.d_col, dt}, S->run.hw, nullptr, blk, S->counters, R, st, &nl);
    if (J) compact(PendingRows{S->pend.d_col, dt, pslot, R}, S->pend.hw, nullptr, blk, S->counters + 1, J, st, &nl);
    if (pool_fold) CK(pool, pf.run(&S, 1, st, &nl));
    CK(pool, cudaGetLastError());
    CK(pool, cudaEventRecord(pool->ev[23], st));
  }
  int32_t n = 0;
  RankQueue rq = {};
  const RankOffensive ro{pslot, S->pend.at<int64_t>(P_JID), out_off, out_n_off};
  const int32_t rc = rank_impl(pool, R, J, nullptr, nullptr, &dt, users, pool_quota, group_quota, group_usage, params,
                               nullptr, &n, nullptr, nullptr, nullptr, &rq, offensive ? &ro : nullptr,
                               pool_fold ? pf.a.pool_out : nullptr);
  if (rc != COOK_OK) return rc;
  cook_phase_stats& ps = pool->phase[COOK_PHASE_RANK];
  if (N > 0) ps.ms_device += ev_ms(pool->ev[7], pool->ev[23]);   // the gathering of the live rows and the pool fold
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
// With `op` (cook_state_match_offers, derived): the offer table is the live offers merged per hostname after the
// expiry, which runs once every check has passed; offers is op->check until then.
int32_t state_match(cook_pool* pool, const char* who, bool derived, const cook_offers_soa* offers,
                    const cook_groups* groups, const cook_user_table* users, const cook_pool_quota* pool_quota,
                    const cook_match_params* params, int64_t* out_considerable_job_id, int32_t* out_assign,
                    int32_t* out_ports, int32_t max_ports, uint8_t* out_fail_reason, cook_match_stats* out_stats,
                    OfferPass* op = nullptr) {
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
  int O = offers->n;
  int32_t n_codes = 0;
  if (derived) {
    if (count_max(S->users_r) >= U)
      return set_err(pool, COOK_E_BADARG, "%s: a live running row's user code is >= n_users", who);
    if (n > 0) {
      if (O > 0 && !offers->hostname_id) return set_err(pool, COOK_E_BADARG, "%s: null offers->hostname_id", who);
      if (!op && !host_codes(offers->hostname_id, O, &n_codes))
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
  if (op) {
    CK(pool, cudaSetDevice(pool->device));
    rc = offers_expire(pool, S, op, groups);
    if (rc != COOK_OK) return rc;
    O = op->osh.O;
    n_codes = op->n_codes;
    if (n == 0) pool->phase[COOK_PHASE_MATCH] = {};   // this call's own removals are all it reports
  }
  S->mm.on = false;
  if (n == 0) return mm_record(pool, S, nullptr, 0);
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
  if (L[L_NOVEL].live) { c.novel_off = P.at<int32_t>(P_NOFF); c.novel_host = L[L_NOVEL].at(0); }
  if (has(F_GPU_MODEL)) c.gpu_model = P.at<int32_t>(P_GPU_MODEL);
  if (has(F_DISK)) { c.disk_request = P.at<double>(P_DISK_REQ); c.disk_type = P.at<int32_t>(P_DISK_TYPE); }
  if (L[L_ATTR].live) { c.attr_off = P.at<int32_t>(P_AOFF); c.attr_col = L[L_ATTR].at(0); c.attr_val = L[L_ATTR].at(1); }
  if (has(F_EST)) c.est_end_ms = P.at<int64_t>(P_EST);
  if (has(F_CKPT)) c.ckpt_location = P.at<int32_t>(P_CKPT);
  if (has(F_RESERVED)) c.reserved_host = P.at<int32_t>(P_RESERVED);
  if (L[L_GROUP].live) { c.group_off = P.at<int32_t>(P_GOFF); c.group_idx = L[L_GROUP].at(0); }
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
  rc = match_build(pool, nullptr, n, sh, op ? op->osh : host_offer_shape(offers), groups, users, pool_quota, params,
                   max_ports, &rows);
  if (rc != COOK_OK) return rc;
  fill_rows_kernel<<<(n + 255) / 256, 256, 0, st>>>(rows, S->pend.d_col, m_slot, n);
  nl++;
  gather_lists(S, rows.jb, m_slot, n, os, st, &nl);
  CK(pool, cudaGetLastError());
  if (op) {
    rc = offers_merge(pool, S, *op, rows, &nl);
    if (rc != COOK_OK) return rc;
  }
  if (derived) {
    rc = derive_match(pool, S, rows, U, O, n_codes, G, groups ? groups->attr_col : nullptr, &nl);
    if (rc != COOK_OK) return rc;
  }
  rc = match_run(pool, nullptr, out_considerable_job_id, out_assign, out_ports, out_fail_reason, out_stats, true,
                 params->max_ctas);
  if (rc != COOK_OK) return rc;
  rc = mm_record(pool, S, m_slot, n);
  if (rc != COOK_OK) return rc;
  cook_phase_stats& ps = pool->phase[COOK_PHASE_MATCH];
  ps.n_launches += nl;
  ps.d2h_bytes += d2h;
  if (out_stats) { out_stats->n_launches += nl; out_stats->d2h_bytes += d2h; }
  return COOK_OK;
}

// cook_state_match_offers: (a) expiry and (b) the merge inside state_match, (c) its match, (d) the consumption
int32_t match_offers(cook_pool* pool, int64_t now_ms, int64_t incubate_ms, const cook_groups* groups,
                     const cook_user_table* users, const cook_pool_quota* pool_quota, const cook_match_params* params,
                     int64_t* out_job_id, int32_t* out_assign, int32_t* out_ports, int32_t max_ports,
                     uint8_t* out_fail_reason, int64_t* out_gone_id, uint8_t* out_gone_fate, int32_t gone_cap,
                     int32_t* out_n_gone, cook_match_stats* out_stats) {
  const char* who = "cook_state_match_offers";
  if (!pool) return COOK_E_BADARG;
  if (!users || !params || !out_job_id || !out_assign || !out_gone_id || !out_gone_fate || !out_n_gone)
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (incubate_ms <= 0) return set_err(pool, COOK_E_BADARG, "%s: incubate_ms <= 0", who);
  PoolState* S = static_cast<PoolState*>(pool->state);
  if ((int64_t)gone_cap < (S ? (int64_t)S->offer.slot_of.size() : 0))
    return set_err(pool, COOK_E_BADARG, "%s: gone_cap < the live offers", who);
  if (groups && groups->attr_col)
    for (int g = 0; g < groups->n_groups; g++)
      if (groups->attr_col[g] < -1) return set_err(pool, COOK_E_BADARG, "%s: groups->attr_col < -1", who);
  *out_n_gone = 0;
  OfferPass op;
  op.now_ms = now_ms; op.incubate_ms = incubate_ms;
  // the checks read a table as wide as every column a pending row or group names, with a code for every VM
  op.check.n = S ? (int)S->vm_names.size() : 0;
  op.check.hostname_id = op.check.name_rank = op.check.attr = &op.dummy;
  int w = S ? count_max(S->attr_cols) + 1 : 0;
  for (int g = 0; groups && groups->attr_col && g < groups->n_groups; g++) w = std::max(w, groups->attr_col[g] + 1);
  op.check.n_attr_cols = w;
  // the offers that left, in arrival order; also after a failure past the expiry, so no removed offer goes unreported
  const auto report = [&]() {
    std::sort(op.gone.begin(), op.gone.end());
    for (size_t i = 0; i < op.gone.size(); i++) {
      out_gone_id[i] = op.gone[i].second.first;
      out_gone_fate[i] = op.gone[i].second.second;
    }
    *out_n_gone = (int32_t)op.gone.size();
  };
  cook_match_stats ms;
  int32_t rc = state_match(pool, who, true, &op.check, groups, users, pool_quota, params, out_job_id, out_assign,
                           out_ports, max_ports, out_fail_reason, &ms, &op);
  if (rc != COOK_OK) {
    report();
    return rc;
  }
  // (d) every offer of a host with an assignment, then every remaining single-shot offer
  std::vector<int32_t> used;
  std::unordered_set<int32_t> hit;
  for (int k = 0; k < ms.n_considerable; k++) {
    if (out_assign[k] < 0) continue;
    const int32_t code = op.codes[out_assign[k]];
    out_assign[k] = code;
    if (!hit.insert(code).second) continue;
    for (const auto& kv : S->ohost[code].live) {
      used.push_back(kv.second);
      op.gone.push_back({kv.first, {S->oinfo[kv.second].id, (uint8_t)COOK_OFFER_USED}});
    }
  }
  for (const auto& kv : S->single_shot) {
    if (hit.count(S->oinfo[kv.second].code)) continue;
    used.push_back(kv.second);
    op.gone.push_back({kv.first, {S->oinfo[kv.second].id, (uint8_t)COOK_OFFER_SINGLE_SHOT}});
  }
  cudaStream_t st = pool->stream;
  rc = offers_remove(pool, S, used, &op.h2d, &op.nl);
  if (rc == COOK_OK) rc = compact_lists(pool, S, st, &op.nl);
  if (rc == COOK_OK && cudaStreamSynchronize(st) != cudaSuccess)
    rc = set_err(pool, COOK_E_CUDA, "%s: %s", who, cudaGetErrorString(cudaGetLastError()));
  report();
  if (rc != COOK_OK) return rc;
  ms.h2d_bytes += op.h2d;
  ms.n_launches += op.nl;
  cook_phase_stats& ps = pool->phase[COOK_PHASE_MATCH];
  ps.h2d_bytes += op.h2d;
  ps.n_launches += op.nl;
  if (out_stats) *out_stats = ms;
  return COOK_OK;
}

// cook_state_rebalance, and with `derived` cook_state_rebalance_derived: the groups' cot_* lists come from the live
// running rows over `hosts`, filled on the device into the lists the build carved
int32_t state_rebalance(cook_pool* pool, const char* who, bool derived, const cook_host_table* hosts,
                        const cook_groups* groups, const cook_user_table* users, const cook_rebalance_params* params,
                        cook_decision* out_decisions, int64_t* out_decision_job_id, int64_t* out_victim_task_id,
                        int32_t victim_cap, int32_t* out_n, bool offers = false) {
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
  if (offers)
    for (const auto& kv : S->vm_names)
      if (!codes.count(kv.second))
        return set_err(pool, COOK_E_BADARG, "%s: a host with a live offer is not in the host table", who);
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
  sh.dev.spare = offers;
  RebPlanPtr plan;
  RebRows rows;
  int32_t rc = rebalance_build(pool, sh, hosts, groups, users, params, &plan, &rows);
  if (rc != COOK_OK) return rc;
  CK(pool, cudaEventRecord(pool->ev[22], st));
  const bool spare = offers && !S->offer.slot_of.empty();
  if (R > 0 || spare) {
    host_map_kernel<<<(H + 255) / 256, 256, 0, st>>>(rows.hostname_id, H, host_of);
    nl++;
  }
  if (spare) {
    rc = offers_spare(pool, S, rows, host_of, H, &nl);
    if (rc != COOK_OK) return rc;
  }
  if (R > 0) {
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
        CK(pool, f.run(&S, 1, st, &nl));
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

// The handle set of a call over several pools: a NULL pools, n <= 0 or a NULL pools[0] is a bare COOK_E_BADARG (no
// handle to hold the message); then every handle non-NULL, listed once and, unless any_device (the calls with a
// gather step), on pools[0]'s device.
int32_t check_handle_set(cook_pool* const* pools, int n, const char* who, bool any_device = false) {
  if (!pools || n <= 0 || !pools[0]) return COOK_E_BADARG;
  cook_pool* pool = pools[0];
  for (int k = 0; k < n; k++) {
    if (!pools[k]) return set_err(pool, COOK_E_BADARG, "%s: a NULL handle", who);
    if (std::find(pools, pools + k, pools[k]) != pools + k)
      return set_err(pool, COOK_E_BADARG, "%s: a handle listed twice", who);
    if (!any_device && pools[k]->device != pool->device)
      return set_err(pool, COOK_E_BADARG, "%s: handles on different devices", who);
  }
  return COOK_OK;
}

// A read-side call's own statistics, from its events ev[20 .. 23] (upload, device, download); no cook_last_stats
// slot is written
cook_phase_stats call_stats(const cook_pool* pool, int64_t h2d, int64_t d2h, int nl) {
  return {ev_ms(pool->ev[20], pool->ev[21]), ev_ms(pool->ev[21], pool->ev[22]), ev_ms(pool->ev[22], pool->ev[23]), h2d,
          d2h, nl, 0};
}

// A read-side call on pools[0]'s stream: open() makes its device current and finds its state (created at the first
// call: the scratch and counters, even when it holds no row); scratch() carves from that scratch between ev[20] and
// ev[21]; the call counts its bytes and launches here and records ev[22] after its kernels, before its first
// download; close() records ev[23], synchronizes and returns the call's own statistics.
struct ReadCall {
  cook_pool* pool;
  PoolState* S = nullptr;
  cudaStream_t st;
  int64_t h2d = 0, d2h = 0;
  int nl = 0;
  explicit ReadCall(cook_pool* p) : pool(p), st(p->stream) {}
  int32_t open(const char* who) {
    CK(pool, cudaSetDevice(pool->device));
    S = state_of(pool, true);
    return S ? COOK_OK : set_err(pool, COOK_E_OOM, "%s: out of device memory", who);
  }
  template <class Body>
  int32_t scratch(const Body& body) {
    CK(pool, carve(S->scratch, st, pool->ev[20], &h2d, body));
    CK(pool, cudaEventRecord(pool->ev[21], st));
    return COOK_OK;
  }
  int32_t close(cook_phase_stats* out) {
    CK(pool, cudaEventRecord(pool->ev[23], st));
    CK(pool, cudaStreamSynchronize(st));
    if (out) *out = call_stats(pool, h2d, d2h, nl);
    return COOK_OK;
  }
};

// a read-side call with no row to read, its empty outputs written: zeroed statistics, no device work
int32_t no_rows(cook_phase_stats* out) {
  if (out) *out = cook_phase_stats{};
  return COOK_OK;
}

// cook_state_user_stats: the running and waiting folds per user over the union of the handles' live rows, classified
int32_t user_stats(cook_pool* const* pools, int n, const cook_user_table* users, const uint8_t* rest_ok,
                   int64_t* out_jobs, double* out_cpus, double* out_mem, uint8_t* out_member, int64_t* out_all_jobs,
                   double* out_all_cpus, double* out_all_mem, int64_t* out_users, cook_phase_stats* out_stats) {
  const char* who = "cook_state_user_stats";
  // ---- every check before any device work or output
  if (int32_t rc = check_handle_set(pools, n, who, true)) return rc;
  cook_pool* pool = pools[0];
  std::vector<const PoolState*> S;
  std::vector<cook_pool*> P;   // S[k]'s handle
  int R = 0, J = 0, hw_r = 0, hw_p = 0;
  if (!users || !out_jobs || !out_cpus || !out_mem || !out_member || !out_all_jobs || !out_all_cpus || !out_all_mem ||
      !out_users)
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  const double* ucol[5] = {users->div_cpus, users->div_mem, users->quota_count, users->quota_cpus, users->quota_mem};
  for (const double* c : ucol)
    if (!c) return set_err(pool, COOK_E_BADARG, "%s: null div_cpus, div_mem, quota_count, quota_cpus or quota_mem", who);
  const int U = users->n_users;
  if (U <= 0) return set_err(pool, COOK_E_BADARG, "%s: n_users <= 0", who);
  for (int k = 0; k < n; k++) {
    const PoolState* s = static_cast<const PoolState*>(pools[k]->state);
    if (!s) continue;
    if (std::max(count_max(s->users_p), count_max(s->users_r)) >= U)
      return set_err(pool, COOK_E_BADARG, "%s: a live row's user code is >= n_users", who);
    S.push_back(s);
    P.push_back(pools[k]);
    R += (int)s->run.slot_of.size(); J += (int)s->pend.slot_of.size();
    hw_r = std::max(hw_r, s->run.hw); hw_p = std::max(hw_p, s->pend.hw);
  }
  if (R + J == 0) {   // no live row: every state is empty, without device work
    memset(out_jobs, 0, sizeof(int64_t) * 4 * (size_t)U);
    memset(out_cpus, 0, sizeof(double) * 4 * (size_t)U);
    memset(out_mem, 0, sizeof(double) * 4 * (size_t)U);
    memset(out_member, 0, (size_t)U);
    memset(out_all_jobs, 0, sizeof(int64_t) * 4);
    memset(out_all_cpus, 0, sizeof(double) * 4);
    memset(out_all_mem, 0, sizeof(double) * 4);
    memset(out_users, 0, sizeof(int64_t) * COOK_USERS_N);
    return no_rows(out_stats);
  }
  ReadCall r(pool);
  if (int32_t rc = r.open(who)) return rc;
  if (S.empty() || S[0] != r.S) {   // S[0] owns the counters the compactions write
    S.insert(S.begin(), r.S);
    P.insert(P.begin(), pool);
  }
  cudaStream_t st = r.st;
  Gather g(pool);
  // ---- one carve: the two folds, the user columns (uploaded), the per-state columns and the totals
  UsageFold fr, fw;
  fr.R = R; fr.U = U;
  fw.R = J; fw.U = U; fw.pending = true;
  StatsArgs a = {};
  a.U = U;
  GridFlag* gf = nullptr;
  StatsTotals* tot = nullptr;
  double *run = nullptr, *wait = nullptr;
  if (int32_t rc = r.scratch([&](Carve& c) {
    if (R) fr.take(c, hw_r);
    if (J) fw.take(c, hw_p);
    run = c.take<double>(4 * (size_t)U); wait = c.take<double>(4 * (size_t)U);
    a.jobs = c.take<int64_t>(4 * (size_t)U); a.cpus = c.take<double>(4 * (size_t)U);
    a.mem = c.take<double>(4 * (size_t)U); a.member = c.take<uint8_t>(U);
    gf = c.take<GridFlag>(1);
    tot = c.take<StatsTotals>(1);
    a.div_cpus = c.up(ucol[0], U); a.div_mem = c.up(ucol[1], U);
    a.q_count = c.up(ucol[2], U); a.q_cpus = c.up(ucol[3], U); a.q_mem = c.up(ucol[4], U);
    a.rest_ok = c.up(rest_ok, U);
  }))
    return rc;
  int& nl = r.nl;
  int64_t& d2h = r.d2h;
  const PoolState* const* list = S.data();
  const int ns = (int)S.size();
  fr.a.user_out = run; fw.a.user_out = wait;
  if (R) CK(pool, fr.run(list, ns, st, &nl, &g, P.data()));
  else CK(pool, cudaMemsetAsync(run, 0, sizeof(double) * 4 * (size_t)U, st));
  if (J) CK(pool, fw.run(list, ns, st, &nl, &g, P.data()));
  else CK(pool, cudaMemsetAsync(wait, 0, sizeof(double) * 4 * (size_t)U, st));
  a.run = run; a.wait = wait;
  user_stats_kernel<<<(U + 255) / 256, 256, 0, st>>>(a);
  CK(pool, cudaMemsetAsync(gf, 0, sizeof(GridFlag), st));
  grid_check_kernel<<<(4 * U + 255) / 256, 256, 0, st>>>(a.cpus, a.mem, nullptr, 4 * U, gf);
  user_stats_totals_kernel<<<1, 128, 0, st>>>(a.jobs, a.cpus, a.mem, a.member, U, gf, tot);
  nl += 3;
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  StatsTotals t;
  CK(pool, download(out_jobs, a.jobs, 4 * (size_t)U, st, &d2h));
  CK(pool, download(out_cpus, a.cpus, 4 * (size_t)U, st, &d2h));
  CK(pool, download(out_mem, a.mem, 4 * (size_t)U, st, &d2h));
  CK(pool, download(out_member, a.member, U, st, &d2h));
  CK(pool, download(&t, tot, 1, st, &d2h));
  if (int32_t rc = r.close(out_stats)) return rc;
  memcpy(out_all_jobs, t.jobs, sizeof t.jobs);
  memcpy(out_all_cpus, t.cpus, sizeof t.cpus);
  memcpy(out_all_mem, t.mem, sizeof t.mem);
  memcpy(out_users, t.users, sizeof t.users);
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_user_stats(cook_pool* const* pools, int32_t n_pools, const cook_user_table* users,
                                         const uint8_t* quota_rest_ok, int64_t* out_jobs, double* out_cpus,
                                         double* out_mem, uint8_t* out_member, int64_t* out_all_jobs,
                                         double* out_all_cpus, double* out_all_mem, int64_t* out_users,
                                         cook_phase_stats* out_stats) {
  return user_stats(pools, n_pools, users, quota_rest_ok, out_jobs, out_cpus, out_mem, out_member, out_all_jobs,
                    out_all_cpus, out_all_mem, out_users, out_stats);
}

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

extern "C" int32_t cook_state_offers_add(cook_pool* pool, const cook_offers_soa* offers, const int64_t* offer_id,
                                         const uint8_t* single_shot, const double* offer_gpus, const char* hostname,
                                         const int32_t* hostname_off, int64_t now_ms) {
  const char* who = "cook_state_offers_add";
  return on_state(pool, who, [&](PoolState* S) {
    return offers_add(pool, S, who, offers, offer_id, single_shot, offer_gpus, hostname, hostname_off, now_ms);
  });
}

extern "C" int32_t cook_state_match_offers(cook_pool* pool, int64_t now_ms, int64_t incubate_ms,
                                           const cook_groups* groups, const cook_user_table* users,
                                           const cook_pool_quota* pool_quota, const cook_match_params* params,
                                           int64_t* out_considerable_job_id, int32_t* out_assign_hostname_id,
                                           int32_t* out_ports, int32_t max_ports, uint8_t* out_fail_reason,
                                           int64_t* out_gone_offer_id, uint8_t* out_gone_fate, int32_t gone_cap,
                                           int32_t* out_n_gone, cook_match_stats* out_stats) {
  return match_offers(pool, now_ms, incubate_ms, groups, users, pool_quota, params, out_considerable_job_id,
                      out_assign_hostname_id, out_ports, max_ports, out_fail_reason, out_gone_offer_id, out_gone_fate,
                      gone_cap, out_n_gone, out_stats);
}

extern "C" int32_t cook_state_rebalance_offers(cook_pool* pool, const cook_host_table* hosts, const cook_groups* groups,
                                               const cook_user_table* users, const cook_rebalance_params* params,
                                               cook_decision* out_decisions, int64_t* out_decision_job_id,
                                               int64_t* out_victim_task_id, int32_t victim_cap, int32_t* out_n) {
  return state_rebalance(pool, "cook_state_rebalance_offers", true, hosts, groups, users, params, out_decisions,
                         out_decision_job_id, out_victim_task_id, victim_cap, out_n, true);
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

// ---- the periodic killers (cook_state_task_facts, cook_state_finish, cook_state_group_runtimes, cook_state_sweep).
// Lingering and cancelled: the live running rows of the handles compacted into one dense range, sorted by (task id,
// handle), then one stable compaction per list in that order.  Stragglers: the live records of the checked groups
// sorted by (group, runtime) and cut into segments, one limit per group; the running rows' group lists expanded into
// (group, task id, runtime) entries, sorted by (group, task id, handle), and compacted by their group's limit.
namespace {

// warp per finished row w: a successful row's group list becomes records (group, whole seconds since its start) at
// the record table's tail plus the exclusive scan of the successful rows' list lengths
struct FinishLen {
  const int32_t* slot; const uint8_t* ok; const int32_t* len;
  __device__ void operator()(int p, int (&x)[1]) const { x[0] = ok[p] ? len[slot[p]] : 0; }
};
__global__ void finish_records_kernel(OrderScan<int, 1> os, const int32_t* slot, const uint8_t* ok, const int64_t* end,
                                      int n, void* const* rc, const int32_t* arena, int32_t* r_grp, int32_t* r_rt,
                                      uint8_t* r_live, int32_t tail) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n || !ok[w]) return;
  const int s = slot[w];
  const int l = static_cast<const int32_t*>(rc[R_GLEN])[s], o = static_cast<const int32_t*>(rc[R_GOFF])[s];
  const int start = tail + os.at(0, w) - l;
  const int32_t rt = (int32_t)((end[w] - static_cast<const int64_t*>(rc[R_START])[s]) / 1000);
  for (int i = lane; i < l; i += 32) {
    r_grp[start + i] = arena[o + i];
    r_rt[start + i] = rt;
    r_live[start + i] = 1;
  }
}

// the history's append: finished row p whose running row starts at or after the horizon goes, in batch order, to the
// table's tail; user, start, cpus and mem from the running row, the reason from the batch or else the row's fact
struct HistAppend {
  const int32_t* slot; const int64_t* end; const uint8_t* ok; const int32_t* reason; void* const* rc; int64_t since;
  HistCols h; int64_t tail;
  __device__ bool keep(int p) const { return static_cast<const int64_t*>(rc[R_START])[slot[p]] >= since; }
  __device__ void emit(int p, int d) const {
    const int s = slot[p];
    const int64_t t = tail + d;
    h.tid[t] = static_cast<const int64_t*>(rc[R_TID])[s];
    h.user[t] = static_cast<const int32_t*>(rc[R_USER])[s];
    h.start[t] = static_cast<const int64_t*>(rc[R_START])[s];
    h.end[t] = end[p];
    h.cpus[t] = static_cast<const double*>(rc[R_CPUS])[s];
    h.mem[t] = static_cast<const double*>(rc[R_MEM])[s];
    h.reason[t] = reason ? reason[p] : static_cast<const int32_t*>(rc[R_REASON])[s];
    h.ok[t] = ok[p] ? 1 : 0;
  }
};

// thread per record: a live record of a group in forget[0, n) (ascending) leaves
__global__ void forget_records_kernel(const int32_t* grp, uint8_t* live, int n_rec, const int32_t* forget, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rec || !live[i]) return;
  const int32_t g = grp[i];
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (forget[m] < g) lo = m + 1;
    else hi = m;
  }
  if (lo < n && forget[lo] == g) live[i] = 0;
}

// A log's compaction into a target of its shape: every column copied by its width, in order, for the rows whose live
// byte is set (live non-null) or else whose int64 key is at or after the horizon
struct LogKeep {
  static constexpr int MAXC = 8;   // the widest log, the history
  const char* s[MAXC]; char* d[MAXC]; int w[MAXC]; int n;
  const uint8_t* live; const int64_t* key; int64_t since;
  LogKeep(const Columns& from, const Columns& to, const uint8_t* lv, const int64_t* k, int64_t t)
      : n(from.n), live(lv), key(k), since(t) {
    assert(n <= MAXC);
    for (int c = 0; c < n; c++) { s[c] = from.at<const char>(c); d[c] = to.at<char>(c); w[c] = from.w[c]; }
  }
  __device__ bool keep(int i) const { return live ? live[i] != 0 : key[i] >= since; }
  __device__ void emit(int i, int k) const {
#pragma unroll
    for (int c = 0; c < MAXC; c++) {
      if (c >= n) break;
      if (w[c] == 8) reinterpret_cast<int64_t*>(d[c])[k] = reinterpret_cast<const int64_t*>(s[c])[i];
      else if (w[c] == 4) reinterpret_cast<int32_t*>(d[c])[k] = reinterpret_cast<const int32_t*>(s[c])[i];
      else d[c][k] = s[c][i];   // width 1 (Columns allows 1, 4 and 8)
    }
  }
};

// the arena rule on the record table: compacted once its dead records outnumber the live ones
int32_t compact_records(cook_pool* pool, PoolState* S, cudaStream_t st, int* nl) {
  Records& R = S->rec;
  if (R.tail - R.n_live <= R.n_live) return COOK_OK;
  if (R.n_live > 0) {
    CK(pool, R.alt.grow(R.c.cap, 0, st));
    int32_t* blk = nullptr;
    CK(pool, carve(S->scratch, st, nullptr, nullptr, [&](Carve& c) { blk = c.take<int32_t>((size_t)R.tail / CP_BLOCK + 2); }));
    compact(LogKeep(R.c, R.alt, R.c.at<uint8_t>(RC_LIVE), nullptr, 0), (int)R.tail, nullptr, blk, S->counters + 6,
            (int)R.n_live, st, nl);
    CK(pool, cudaGetLastError());
    std::swap(R.c, R.alt);
  }
  R.tail = R.n_live;
  return COOK_OK;
}

int32_t task_facts(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* task_id,
                   const int64_t* max_runtime_ms, const uint8_t* cancelled, const uint8_t* unknown) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && !task_id) return set_err(pool, COOK_E_BADARG, "%s: null task_id", who);
  for (int i = 0; max_runtime_ms && i < n; i++)
    if (max_runtime_ms[i] < -1) return set_err(pool, COOK_E_BADARG, "%s: a max_runtime_ms below -1", who);
  std::vector<int32_t> slot;
  if (int32_t rc = live_slots(pool, who, S->run, "task", n, task_id, &slot)) return rc;
  // ---- host side: each row's bits, the given ones replaced
  const bool bits = cancelled || unknown;
  std::vector<uint8_t> facts(bits ? n : 0);
  for (int i = 0; bits && i < n; i++) {
    uint8_t& f = S->rfacts[slot[i]];
    if (cancelled) f = (uint8_t)((f & ~RF_CANCELLED) | (cancelled[i] ? RF_CANCELLED : 0));
    if (unknown) f = (uint8_t)((f & ~RF_UNKNOWN) | (unknown[i] ? RF_UNKNOWN : 0));
    facts[i] = f;
  }
  // ---- device: a patch scatter (live flag and generation kept)
  const bool cols = n && (max_runtime_ms || bits);
  ScatterArgs pa;
  memset(&pa, 0, sizeof(pa));
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (cols)
      patch_args(c, pa, S->run, slot.data(), n, {{R_MAXRT, max_runtime_ms, -1}, {R_FACTS, bits ? facts.data() : nullptr, 0}});
  }))
    return rc;
  scatter(pa, S->run, cols ? n : 0, 0, -1, nullptr, w.st, &w.nl);
  return w.end();
}

// the reason code of each listed live running row, in place (live flag and generation kept)
int32_t task_reason(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* task_id,
                    const int32_t* reason_code) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && (!task_id || !reason_code)) return set_err(pool, COOK_E_BADARG, "%s: null task_id or reason_code", who);
  if (!idx_in_range(reason_code, n, -1, INT32_MAX)) return set_err(pool, COOK_E_BADARG, "%s: a reason code below -1", who);
  std::vector<int32_t> slot;
  if (int32_t rc = live_slots(pool, who, S->run, "task", n, task_id, &slot)) return rc;
  for (int i = 0; i < n; i++) S->rreason[slot[i]] = reason_code[i];   // cook_state_status decides from it
  ScatterArgs pa;
  memset(&pa, 0, sizeof(pa));
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (n) patch_args(c, pa, S->run, slot.data(), n, {{R_REASON, reason_code, -1}});
  }))
    return rc;
  scatter(pa, S->run, n, 0, -1, nullptr, w.st, &w.nl);
  return w.end();
}

// What cook_state_finish_history adds to cook_state_finish: the rows' reason codes (NULL: each row's reason fact).
struct FinishHistory { const int32_t* reason_code; };
// What cook_state_status adds to cook_state_finish_history: the rows' preempted flags (NULL: none) and the outputs.
struct FinishStatus { const uint8_t* preempted; int32_t* outcome; int32_t* attempts; };

// running_rm_task_id = task_id, plus one record per group of each successful row; with `fh`, the rows that start at
// or after the horizon of an enabled history are also appended to it
int32_t finish(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* task_id, const int64_t* end_time_ms,
               const uint8_t* success, const FinishHistory* fh = nullptr, const FinishStatus* fs = nullptr) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (fs && n && (!fs->outcome || !fs->attempts)) return set_err(pool, COOK_E_BADARG, "%s: null out_outcome or out_attempts", who);
  if (n && !task_id) return set_err(pool, COOK_E_BADARG, "%s: null task_id", who);
  if (n && success && !end_time_ms) return set_err(pool, COOK_E_BADARG, "%s: success without end_time_ms", who);
  if (fh && n && (!end_time_ms || !success)) return set_err(pool, COOK_E_BADARG, "%s: null end_time_ms or success", who);
  if (fh && !idx_in_range(fh->reason_code, n, -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "%s: a reason code below -1", who);
  std::vector<int32_t> slot;
  if (int32_t rc = live_slots(pool, who, S->run, "task", n, task_id, &slot)) return rc;
  History& H = S->hist;
  int64_t nhist = 0;   // the rows the history appends
  for (int i = 0; fh && i < n; i++) {
    if (end_time_ms[i] < S->rstart[slot[i]]) return set_err(pool, COOK_E_BADARG, "%s: a row that ends before its start", who);
    if (H.on && S->rstart[slot[i]] >= H.since) nhist++;
  }
  if (H.tail + nhist > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 history rows", who);
  int64_t nrec = 0;   // the records the successful rows append
  for (int i = 0; success && i < n; i++) {
    if (!success[i]) continue;
    const int32_t s = slot[i];
    if (end_time_ms[i] < S->rstart[s]) return set_err(pool, COOK_E_BADARG, "%s: a success that ends before its start", who);
    if ((end_time_ms[i] - S->rstart[s]) / 1000 > INT32_MAX)
      return set_err(pool, COOK_E_BADARG, "%s: a runtime of 2^31 s or more", who);
    nrec += (int64_t)S->rgroups[s].size();
  }
  if (S->rec.tail + nrec > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 records", who);
  cudaStream_t st = pool->stream;
  // ---- host side: cook_state_apply's removals, then the records' counts.  With retry facts, in batch order: the
  // status's job decision (cook_state_status) or, for a job's last live instance, its parked copy freed.
  std::vector<int32_t> unparked, rq_slot, ap_slot, ap_code;
  for (int i = 0; i < n; i++) {
    const int32_t s = slot[i];
    S->run.slot_of.erase(task_id[i]);
    S->add_running(s, -1);
    S->run.free.push_back(s);
    if (success && success[i])
      for (int32_t g : S->rgroups[s]) count_add(S->rec_groups, g, +1);
    const int64_t j = S->rjid[s];
    auto f = S->retry.find(j);
    if (fs && f == S->retry.end()) {
      fs->outcome[i] = COOK_JOB_NO_FACTS;
      fs->attempts[i] = -1;
    }
    if (f == S->retry.end()) continue;
    const bool other = S->jobs_r.count(j) != 0;   // another live running or unknown instance
    if (!fs) {
      if (!other) {
        S->unpark(j, &unparked);
        if (!S->pend.slot_of.count(j)) S->retry.erase(f);
      }
      continue;
    }
    // :instance/update-state's job-state cond (schema.clj:1242-1300) for this one status
    RetryFacts& F = f->second;
    F.done[fh->reason_code ? fh->reason_code[i] : S->rreason[s]]++;
    const int32_t att = S->attempts(F);
    fs->attempts[i] = att;
    int32_t oc;
    if (F.flags & COOK_RF_COMPLETED) oc = COOK_JOB_COMPLETED;
    else if (success[i] || (!other && att >= F.max_retries)) oc = COOK_JOB_COMPLETED;
    else if (other) oc = COOK_JOB_RUNNING;
    else oc = S->parked.count(j) ? COOK_JOB_WAITING : COOK_JOB_WAITING_UNRETAINED;
    fs->outcome[i] = oc;
    if (oc == COOK_JOB_COMPLETED) {
      F.flags |= COOK_RF_COMPLETED;
      S->unpark(j, &unparked);
      if (!other && !S->pend.slot_of.count(j)) S->retry.erase(f);
    } else if (oc == COOK_JOB_WAITING) {   // the requeue: the parked copy becomes the live row an upsert would write
      auto it = S->parked.find(j);
      const int32_t p = it->second;
      S->parked.erase(it);
      PendingInfo& pi = S->pinfo[p];
      for (int l = 0; l < 3; l++) S->park_len[l] -= pi.len[l];
      const int32_t h = S->rhost[s];
      if (h != -1 && !(fs->preempted && fs->preempted[i]) && std::find(pi.novel.begin(), pi.novel.end(), h) == pi.novel.end()) {
        pi.novel.push_back(h);
        pi.len[L_NOVEL]++;
        ap_slot.push_back(p);
        ap_code.push_back(h);
      }
      if (rq_slot.empty()) S->pend_epoch++;
      if ((pi.flags >> F_RESERVED) & 1) pi.flags ^= (uint16_t)(1u << F_RESERVED);   // reserved_host -1
      pi.jf = 0;                                                                     // no job facts
      pi.touched = S->pend_epoch;
      S->pend.slot_of.emplace(j, p);
      S->add_pending(p, pi, +1);
      rq_slot.push_back(p);
    }
  }
  const int nrq = (int)rq_slot.size(), nap = (int)ap_slot.size(), nuk = (int)unparked.size();
  int64_t nadd = 0;   // the novel-host entries the requeue's moved lists take
  for (int32_t p : ap_slot) nadd += S->pinfo[p].len[L_NOVEL];
  // ---- device: the records (read before the removal empties the rows' lists), the removal, the arena rules
  Records& RC = S->rec;
  const int32_t rtail = (int32_t)RC.tail;
  CK(pool, RC.grow(RC.tail + nrec, st));
  RC.tail += nrec;
  RC.n_live += nrec;
  const int64_t htail = H.tail;
  if (nhist) CK(pool, H.grow(H.tail + nhist, st));
  H.tail += nhist;
  const int32_t rgtail = (int32_t)S->lists[L_RGROUP].tail;
  ListArena& NV = S->lists[L_NOVEL];
  const int32_t ntail = (int32_t)NV.tail;
  if (nadd) {
    CK(pool, NV.grow(NV.tail + nadd, st));
    NV.tail += nadd;
  }
  const int32_t* d_slot = nullptr;
  const uint8_t* d_ok = nullptr;
  const int64_t* d_end = nullptr;
  const int32_t* d_reason = nullptr;
  const int32_t *d_ap_slot = nullptr, *d_ap_code = nullptr;
  int32_t* hblk = nullptr;
  OrderScan<int, 1> os, aos;
  ScatterArgs rq, uk;
  memset(&rq, 0, sizeof(rq)); memset(&uk, 0, sizeof(uk));
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (!n) return;
    if (nrq) {   // live again with a new generation, reserved_host -1, no job facts, no longer parked
      rq.nc = 0;   // carve runs this body twice: once to size, once to upload
      rq.c[rq.nc++] = ScatterCol{static_cast<char*>(S->pend.col[P_RESERVED]), nullptr, -1, P_SZ[P_RESERVED]};
      rq.c[rq.nc++] = ScatterCol{static_cast<char*>(S->pend.col[P_JF]), nullptr, 0, P_SZ[P_JF]};
      rq.c[rq.nc++] = ScatterCol{S->park.at<char>(0), nullptr, 0, 1};
      rq.slot = c.up(rq_slot.data(), nrq);
    }
    if (nap) {
      d_ap_slot = c.up(ap_slot.data(), nap);
      d_ap_code = c.up(ap_code.data(), nap);
      aos.part[0] = c.take<int32_t>(nap);
      aos.tile[0] = c.take<int32_t>((nap + OS_TILE - 1) / OS_TILE + 1);
    }
    if (nuk) {
      uk.c[0] = ScatterCol{S->park.at<char>(0), nullptr, 0, 1};
      uk.nc = 1;
      uk.slot = c.up(unparked.data(), nuk);
    }
    d_slot = c.up(slot.data(), n);
    if (success) { d_ok = c.up(success, n); d_end = c.up(end_time_ms, n); }
    if (nrec) {   // device-only buffers: nothing uploaded
      os.part[0] = c.take<int32_t>(n);
      os.tile[0] = c.take<int32_t>((n + OS_TILE - 1) / OS_TILE + 1);
    }
    if (nhist) {
      d_reason = c.up(fh->reason_code, n);
      hblk = c.take<int32_t>((size_t)n / CP_BLOCK + 2);
    }
  }))
    return rc;
  int& nl = w.nl;
  if (nrec) {
    order_scan(os, FinishLen{d_slot, d_ok, S->run.at<int32_t>(R_GLEN)}, n, S->gf0, st, &nl);
    finish_records_kernel<<<(n + 7) / 8, 256, 0, st>>>(os, d_slot, d_ok, d_end, n, S->run.d_col,
                                                       S->lists[L_RGROUP].at(0), RC.c.at<int32_t>(RC_GRP),
                                                       RC.c.at<int32_t>(RC_RT), RC.c.at<uint8_t>(RC_LIVE), rtail);
    nl++;
  }
  if (nhist)   // read from the running rows before the removal
    compact(HistAppend{d_slot, d_end, d_ok, d_reason, S->run.d_col, H.since, H.cols(), htail}, n, nullptr, hblk,
            S->counters + 7, (int)nhist, st, &nl);
  if (n) {
    ScatterArgs rr;
    memset(&rr, 0, sizeof(rr));
    rr.slot = d_slot;
    scatter(rr, S->run, n, 0, R_LIVE, &rgtail, st, &nl);
  }
  if (nap) {   // the requeued rows' novel-host lists, each with its one new entry, to the arena's tail
    order_scan(aos, NovelLen{d_ap_slot, S->pend.at<int32_t>(P_NLEN)}, nap, S->gf0, st, &nl);
    requeue_novel_kernel<<<(nap + 7) / 8, 256, 0, st>>>(aos, d_ap_slot, d_ap_code, nap,
                                                        static_cast<int32_t*>(S->pend.col[P_NOFF]),
                                                        static_cast<int32_t*>(S->pend.col[P_NLEN]), NV.at(0), ntail);
    nl++;
  }
  scatter(rq, S->pend, nrq, 1, P_LIVE, nullptr, st, &nl);
  scatter(uk, S->pend, nuk, 0, -1, nullptr, st, &nl);
  int32_t rc = compact_lists(pool, S, st, &nl);
  if (rc == COOK_OK) rc = compact_records(pool, S, st, &nl);
  return rc != COOK_OK ? rc : w.end();
}

// the reason dictionary and the global mea-culpa limit; host only
int32_t retry_config(cook_pool* pool, PoolState* S, const char* who, int32_t mea_culpa_limit, int n,
                     const int32_t* reason_code, const uint8_t* mea_culpa, const int32_t* failure_limit) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n_reasons < 0", who);
  if (n && (!reason_code || !mea_culpa || !failure_limit)) return set_err(pool, COOK_E_BADARG, "%s: null array", who);
  if (mea_culpa_limit < -1) return set_err(pool, COOK_E_BADARG, "%s: a mea_culpa_limit below -1", who);
  std::unordered_map<int32_t, RetryReason> m;
  m.reserve((size_t)n);
  for (int i = 0; i < n; i++) {
    if (reason_code[i] < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative reason code", who);
    if (failure_limit[i] < -2) return set_err(pool, COOK_E_BADARG, "%s: a failure limit below -2", who);
    if (!m.emplace(reason_code[i], RetryReason{mea_culpa[i] != 0, failure_limit[i]}).second)
      return set_err(pool, COOK_E_BADARG, "%s: reason code twice", who);
  }
  S->mc_limit = mea_culpa_limit;
  S->reasons.swap(m);
  return COOK_OK;
}

// the retry facts of jobs the handle holds (a live pending row, a parked copy or a live running instance)
int32_t retry_facts(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* job_id,
                    const int32_t* max_retries, const uint8_t* flags, const int32_t* done_off, const int32_t* done_reason) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && (!job_id || !max_retries || !flags)) return set_err(pool, COOK_E_BADARG, "%s: null job_id, max_retries or flags", who);
  if (!csr_ok(done_off, n, done_reason, nullptr, false)) return set_err(pool, COOK_E_BADARG, "%s: malformed CSR offsets", who);
  if (done_off && !idx_in_range(done_reason, done_off[n], -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "%s: a reason code below -1", who);
  {
    std::unordered_set<int64_t> seen;
    seen.reserve((size_t)n);
    for (int i = 0; i < n; i++) {
      if (max_retries[i] < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative max_retries", who);
      if (flags[i] & ~(COOK_RF_DISABLE_MEA_CULPA | COOK_RF_COMPLETED)) return set_err(pool, COOK_E_BADARG, "%s: unknown flag bits", who);
      if (!seen.insert(job_id[i]).second) return set_err(pool, COOK_E_BADARG, "%s: job id twice", who);
      if (!S->pend.slot_of.count(job_id[i]) && !S->parked.count(job_id[i]) && !S->jobs_r.count(job_id[i]))
        return set_err(pool, COOK_E_BADARG, "%s: unknown job id", who);
    }
  }
  // ---- host side: the facts replaced; a completed job without a live instance loses its parked copy and its facts
  std::vector<int32_t> unparked;
  for (int i = 0; i < n; i++) {
    const int64_t j = job_id[i];
    if ((flags[i] & COOK_RF_COMPLETED) && !S->jobs_r.count(j) && S->parked.count(j)) {
      S->unpark(j, &unparked);
      S->retry.erase(j);
      continue;
    }
    RetryFacts& F = S->retry[j];
    F.max_retries = max_retries[i];
    F.flags = flags[i];
    F.done.clear();
    for (int k = done_off ? done_off[i] : 0; done_off && k < done_off[i + 1]; k++) F.done[done_reason[k]]++;
  }
  // ---- device: the freed copies' park flags
  const int nuk = (int)unparked.size();
  ScatterArgs uk;
  memset(&uk, 0, sizeof(uk));
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (!nuk) return;
    uk.c[0] = ScatterCol{S->park.at<char>(0), nullptr, 0, 1};
    uk.nc = 1;
    uk.slot = c.up(unparked.data(), nuk);
  }))
    return rc;
  scatter(uk, S->pend, nuk, 0, -1, nullptr, w.st, &w.nl);
  return w.end();
}

bool bad_amount(double x) { return !std::isfinite(x) || x < 0 || std::signbit(x); }

// the history replaced by n rows at horizon since_ms, and on; the rows are copied straight into the table's columns
int32_t history_seed(cook_pool* pool, PoolState* S, const char* who, int64_t since_ms, int n, const int64_t* task_id,
                     const int32_t* user, const int64_t* start_ms, const int64_t* end_ms, const double* cpus,
                     const double* mem, const uint8_t* success, const int32_t* reason_code) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && (!task_id || !user || !start_ms || !end_ms || !cpus || !mem || !success || !reason_code))
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (!idx_in_range(user, n, 0, INT32_MAX)) return set_err(pool, COOK_E_BADARG, "%s: a negative user code", who);
  if (!idx_in_range(reason_code, n, -1, INT32_MAX)) return set_err(pool, COOK_E_BADARG, "%s: a reason code below -1", who);
  std::unordered_set<int64_t> seen;
  seen.reserve((size_t)n);
  for (int i = 0; i < n; i++) {
    if (start_ms[i] < since_ms) return set_err(pool, COOK_E_BADARG, "%s: a row that starts before since_ms", who);
    if (end_ms[i] < start_ms[i]) return set_err(pool, COOK_E_BADARG, "%s: a row that ends before its start", who);
    if (bad_amount(cpus[i]) || bad_amount(mem[i]))
      return set_err(pool, COOK_E_BADARG, "%s: cpus or mem negative, -0.0 or not finite", who);
    if (!seen.insert(task_id[i]).second) return set_err(pool, COOK_E_BADARG, "%s: task id twice", who);
    if (S->run.slot_of.count(task_id[i])) return set_err(pool, COOK_E_BADARG, "%s: a live running task id", who);
  }
  History& H = S->hist;
  H.tail = 0;
  H.since = since_ms;
  H.on = true;
  CK(pool, H.grow(n, pool->stream));
  H.tail = n;
  StateWrite w(pool, S);
  if (int32_t rc = w.direct([&](Carve& c) {
    if (!n) return;
    H.c.copy(c, 0, n, {task_id, start_ms, end_ms, cpus, mem, user, reason_code, success});
  }))
    return rc;
  return w.end();
}

// A log's horizon raised to since_ms: its rows whose int64 column `key` is before it leave in one compaction into new
// columns of its capacity (blk: the compaction's block counts), and the log takes them and the kept count, or is left
// as it was.
int32_t log_advance(cook_pool* pool, PoolState* S, StateWrite& w, Log& L, int key, int64_t since_ms, int32_t* blk) {
  const int T = (int)L.tail;
  Columns nc = L.c.shape();
  CK(pool, nc.grow(L.c.cap, 0, w.st));
  compact(LogKeep(L.c, nc, nullptr, L.c.at<int64_t>(key), since_ms), T, nullptr, blk, S->counters + 7, T, w.st, &w.nl);
  int32_t kept = 0;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = download(&kept, S->counters + 7, 1, w.st, &w.d2h);
  if (e == cudaSuccess) e = cudaStreamSynchronize(w.st);
  if (e != cudaSuccess) { nc.release(); CK(pool, e); }
  L.c.release();
  L.c = nc;
  L.tail = kept;
  return COOK_OK;
}

// the horizon raised to since_ms: the rows that start before it leave in one compaction into new columns
int32_t history_advance(cook_pool* pool, PoolState* S, const char* who, int64_t since_ms) {
  History& H = S->hist;
  if (!H.on) return set_err(pool, COOK_E_BADARG, "%s: history is off", who);
  if (since_ms < H.since) return set_err(pool, COOK_E_BADARG, "%s: since_ms below the horizon", who);
  int32_t* blk = nullptr;
  const int T = (int)H.tail;
  StateWrite w(pool, S);
  if (int32_t rc = w.up(S->scratch, [&](Carve& c) {
    if (T && since_ms > H.since) blk = c.take<int32_t>((size_t)T / CP_BLOCK + 2);
  }))
    return rc;
  if (T && since_ms > H.since)
    if (int32_t rc = log_advance(pool, S, w, H, H_START, since_ms, blk)) return rc;
  H.since = since_ms;
  return w.end();
}

// the records of the forgotten groups leave, then the seeds are appended
int32_t group_runtimes(cook_pool* pool, PoolState* S, const char* who, int n_add, const int32_t* group,
                       const int32_t* runtime_s, int n_forget, const int32_t* forget_group) {
  if (n_add < 0 || n_forget < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative size", who);
  if ((n_add && (!group || !runtime_s)) || (n_forget && !forget_group))
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (!idx_in_range(group, n_add, 0, INT32_MAX) || !idx_in_range(forget_group, n_forget, 0, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "%s: a negative group code", who);
  if (!idx_in_range(runtime_s, n_add, 0, INT32_MAX)) return set_err(pool, COOK_E_BADARG, "%s: a negative runtime", who);
  Records& RC = S->rec;
  if (RC.tail + n_add > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 records", who);
  cudaStream_t st = pool->stream;
  // ---- host side
  std::vector<int32_t> forget(forget_group, forget_group + n_forget);
  std::sort(forget.begin(), forget.end());
  forget.erase(std::unique(forget.begin(), forget.end()), forget.end());
  for (int32_t g : forget) {
    auto it = S->rec_groups.find(g);
    if (it == S->rec_groups.end()) continue;
    RC.n_live -= it->second;
    S->rec_groups.erase(it);
  }
  for (int i = 0; i < n_add; i++) count_add(S->rec_groups, group[i], +1);
  // ---- device
  const int32_t tail0 = (int32_t)RC.tail;
  CK(pool, RC.grow(RC.tail + n_add, st));
  const int nf = (int)forget.size();
  const int32_t* d_forget = nullptr;
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (nf) d_forget = c.up(forget.data(), nf);
    if (c.base && n_add) RC.c.copy(c, tail0, n_add, {group, runtime_s});
  }))
    return rc;
  if (nf && tail0) {
    forget_records_kernel<<<(tail0 + 255) / 256, 256, 0, st>>>(RC.c.at<int32_t>(RC_GRP), RC.c.at<uint8_t>(RC_LIVE),
                                                               tail0, d_forget, nf);
    w.nl++;
  }
  if (n_add) CK(pool, cudaMemsetAsync(RC.c.at<uint8_t>(RC_LIVE) + tail0, 1, (size_t)n_add, st));
  RC.tail += n_add;
  RC.n_live += n_add;
  if (int32_t rc = compact_records(pool, S, st, &w.nl)) return rc;
  return w.end();
}

// ---- cook_state_sweep
// every live running row of one handle, dense after those of the handles before it (base)
struct SweepRows {
  void* const* col; int base; int32_t pool;
  int64_t* tid; int32_t* pidx; int64_t* start; int64_t* maxrt; uint8_t* facts;
  __device__ bool keep(int i) const { return static_cast<const uint8_t*>(col[R_LIVE])[i]; }
  __device__ void emit(int i, int d) const {
    d += base;
    tid[d] = static_cast<const int64_t*>(col[R_TID])[i];
    pidx[d] = pool;
    start[d] = static_cast<const int64_t*>(col[R_START])[i];
    maxrt[d] = static_cast<const int64_t*>(col[R_MAXRT])[i];
    facts[d] = static_cast<const uint8_t*>(col[R_FACTS])[i];
  }
};
// position p of the (task id, handle) order: lingering, now - start > min(max-runtime or the default, max timeout), or
// (cancelled) the cancelled bit
struct KillSel {
  const int32_t* ord; const int64_t* tid; const int32_t* pidx; const int64_t* start; const int64_t* maxrt;
  const uint8_t* facts; int64_t now, dflt, cap; bool cancelled;
  int64_t* o_tid; int32_t* o_pool;
  __device__ bool keep(int p) const {
    const int i = ord[p];
    if (cancelled) return facts[i] & RF_CANCELLED;
    const int64_t m = maxrt[i] < 0 ? dflt : maxrt[i];
    return now - start[i] > (m < cap ? m : cap);
  }
  __device__ void emit(int p, int d) const { const int i = ord[p]; o_tid[d] = tid[i]; o_pool[d] = pidx[i]; }
};
// the live records of one handle whose group is checked, dense after the handles before it
struct SweepRecords {
  const int32_t* grp; const int32_t* rt; const uint8_t* live; const int32_t* kind; int base;
  int32_t* d_grp; int64_t* d_rt;
  __device__ bool keep(int i) const { return live[i] && kind[grp[i]] == COOK_SWEEP_QUANTILE_DEVIATION; }
  __device__ void emit(int i, int d) const { d_grp[base + d] = grp[i]; d_rt[base + d] = rt[i]; }
};
// thread per group: idx = (int)((n_jobs - 1) * quantile); with more than idx successes the limit is the idx-th
// smallest runtime times the multiplier, else (or unchecked, or idx < 0) +inf
__global__ void straggler_limit_kernel(const int32_t* kind, const double* quantile, const double* multiplier,
                                       const int32_t* n_jobs, const int32_t* seg_start, const int32_t* seg_end,
                                       const int32_t* ord, const int64_t* rt, int G, double* limit) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  double lim = INFINITY;
  if (kind[g] == COOK_SWEEP_QUANTILE_DEVIATION) {
    const int idx = (int)((double)(n_jobs[g] - 1) * quantile[g]);
    if (idx >= 0 && seg_end[g] - seg_start[g] > idx) lim = (double)rt[ord[seg_start[g] + idx]] * multiplier[g];
  }
  limit[g] = lim;
}
struct GroupedRows {   // one handle's live running rows with a group list, by slot
  const uint8_t* live; const int32_t* len; int32_t* slot;
  __device__ bool keep(int i) const { return live[i] && len[i] > 0; }
  __device__ void emit(int i, int d) const { slot[d] = i; }
};
struct ExpandArgs {
  OrderScan<int, 1> os;   // inclusive scan of the rows' list lengths
  const int32_t* slot; int K, ebase; int32_t pool;
  void* const* col; const int32_t* arena; const int32_t* kind; int64_t now;
  int32_t* e_grp; int64_t* e_tid; int32_t* e_pool;
  int64_t* e_rt;          // whole seconds run; -1: not judged (status unknown, or the group is not checked)
  int32_t* bad;           // set by a judged entry that starts after now
};
// thread per row: one entry per group of its list, at ebase plus where the scan puts the row
__global__ void straggler_expand_kernel(ExpandArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.K) return;
  const int s = a.slot[k];
  const int l = static_cast<const int32_t*>(a.col[R_GLEN])[s], o = static_cast<const int32_t*>(a.col[R_GOFF])[s];
  const int base = a.ebase + a.os.at(0, k) - l;
  const bool running = !(static_cast<const uint8_t*>(a.col[R_FACTS])[s] & RF_UNKNOWN);
  const int64_t t = static_cast<const int64_t*>(a.col[R_TID])[s], st = static_cast<const int64_t*>(a.col[R_START])[s];
  for (int i = 0; i < l; i++) {
    const int32_t g = a.arena[o + i];
    const bool judged = running && a.kind[g] == COOK_SWEEP_QUANTILE_DEVIATION;
    if (judged && st > a.now) *a.bad = 1;
    a.e_grp[base + i] = g;
    a.e_tid[base + i] = t;
    a.e_pool[base + i] = a.pool;
    a.e_rt[base + i] = judged ? (a.now - st) / 1000 : -1;
  }
}
// position p of the (group, task id, handle) order: a judged entry past its group's limit
struct StragglerSel {
  const int32_t* ord; const int32_t* e_grp; const int64_t* e_tid; const int32_t* e_pool; const int64_t* e_rt;
  const double* limit; int32_t* o_grp; int64_t* o_tid; int32_t* o_pool;
  __device__ bool keep(int p) const { const int i = ord[p]; return e_rt[i] >= 0 && (double)e_rt[i] > limit[e_grp[i]]; }
  __device__ void emit(int p, int d) const {
    const int i = ord[p];
    o_grp[d] = e_grp[i]; o_tid[d] = e_tid[i]; o_pool[d] = e_pool[i];
  }
};

int32_t sweep(cook_pool* const* pools, int n, int64_t now, int64_t dflt, int64_t max_to, int G, const int32_t* kind,
              const double* quantile, const double* multiplier, const int32_t* n_jobs, int32_t row_cap, int64_t* l_tid,
              int32_t* l_pool, int32_t* l_n, int64_t* c_tid, int32_t* c_pool, int32_t* c_n, int32_t entry_cap,
              int32_t* s_grp, int64_t* s_tid, int32_t* s_pool, int32_t* s_n, cook_phase_stats* out_stats) {
  const char* who = "cook_state_sweep";
  // ---- every check before any device work or output
  if (int32_t rc = check_handle_set(pools, n, who)) return rc;
  cook_pool* pool = pools[0];
  const bool linger = l_tid != nullptr, cancel = c_tid != nullptr, strag = s_tid != nullptr;
  if ((linger && (!l_pool || !l_n)) || (cancel && (!c_pool || !c_n)) || (strag && (!s_grp || !s_pool || !s_n)))
    return set_err(pool, COOK_E_BADARG, "%s: a list without its pool column or count", who);
  if (G < 0) return set_err(pool, COOK_E_BADARG, "%s: n_groups < 0", who);
  if (strag && G > 0 && (!kind || !quantile || !multiplier || !n_jobs))
    return set_err(pool, COOK_E_BADARG, "%s: null group_kind, quantile, multiplier or n_jobs", who);
  for (int g = 0; strag && g < G; g++) {
    if (kind[g] != COOK_SWEEP_NONE && kind[g] != COOK_SWEEP_QUANTILE_DEVIATION)
      return set_err(pool, COOK_E_BADARG, "%s: an unknown group kind", who);
    if (kind[g] == COOK_SWEEP_QUANTILE_DEVIATION && !(quantile[g] >= 0.0 && quantile[g] <= 1.0))
      return set_err(pool, COOK_E_BADARG, "%s: a quantile outside [0, 1]", who);
    if (n_jobs[g] < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative n_jobs", who);
  }
  // the handles with rows, their pool index; sizes from the host-side counts
  std::vector<std::pair<const PoolState*, int32_t>> hs;
  int64_t R = 0, N = 0, M = 0, K = 0;
  int hw = 0, kmax = 0;
  for (int k = 0; k < n; k++) {
    const PoolState* s = static_cast<const PoolState*>(pools[k]->state);
    if (!s) continue;
    if (strag && (count_max(s->groups_r) >= G || count_max(s->rec_groups) >= G))
      return set_err(pool, COOK_E_BADARG, "%s: a live group code >= n_groups", who);
    hs.push_back({s, k});
    R += (int64_t)s->run.slot_of.size();
    N += s->lists[L_RGROUP].live;
    K += s->grp_rows;
    kmax = std::max<int>(kmax, (int)s->grp_rows);
    hw = std::max({hw, s->run.hw, (int)s->rec.tail});
    for (const auto& kv : s->rec_groups)
      if (strag && kind[kv.first] == COOK_SWEEP_QUANTILE_DEVIATION) M += kv.second;
  }
  if (R > INT32_MAX || N > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 rows", who);
  if ((linger || cancel) && row_cap < R) return set_err(pool, COOK_E_BADARG, "%s: row_cap < the live running rows", who);
  if (strag && entry_cap < N) return set_err(pool, COOK_E_BADARG, "%s: entry_cap < the live group entries", who);
  const bool rows = (linger || cancel) && R > 0, groups = strag && N > 0;
  if (!rows && !groups) {   // nothing to judge: empty lists, no device work
    if (linger) *l_n = 0;
    if (cancel) *c_n = 0;
    if (strag) *s_n = 0;
    return no_rows(out_stats);
  }
  ReadCall r(pool);
  if (int32_t rc = r.open(who)) return rc;
  cudaStream_t st = r.st;
  hw = std::max({hw, (int)R, (int)N});
  // ---- one carve
  int32_t *cnt = nullptr, *blk = nullptr, *ord = nullptr, *tmp = nullptr, *pidx = nullptr;
  int64_t *tid = nullptr, *start = nullptr, *maxrt = nullptr;
  uint8_t* facts = nullptr;
  int64_t *o_ltid = nullptr, *o_ctid = nullptr, *o_stid = nullptr;
  int32_t *o_lpool = nullptr, *o_cpool = nullptr, *o_sgrp = nullptr, *o_spool = nullptr;
  const int32_t *d_kind = nullptr, *d_nj = nullptr;
  const double *d_q = nullptr, *d_m = nullptr;
  int32_t *r_grp = nullptr, *r_ord = nullptr, *r_tmp = nullptr, *seg_s = nullptr, *seg_e = nullptr, *slot = nullptr;
  int64_t* r_rt = nullptr;
  double* limit = nullptr;
  OrderScan<int, 1> os;
  int32_t *e_grp = nullptr, *e_pool = nullptr, *e_ord = nullptr, *e_tmp = nullptr;
  int64_t *e_tid = nullptr, *e_rt = nullptr;
  if (int32_t rc = r.scratch([&](Carve& c) {
    cnt = c.take<int32_t>(5);   // lingering, cancelled, stragglers, start after now, the compactions' own
    blk = c.take<int32_t>((size_t)hw / CP_BLOCK + 2);
    if (rows) {
      tid = c.take<int64_t>(R); pidx = c.take<int32_t>(R); start = c.take<int64_t>(R); maxrt = c.take<int64_t>(R);
      facts = c.take<uint8_t>(R); ord = c.take<int32_t>(R); tmp = c.take<int32_t>(R);
      if (linger) { o_ltid = c.take<int64_t>(R); o_lpool = c.take<int32_t>(R); }
      if (cancel) { o_ctid = c.take<int64_t>(R); o_cpool = c.take<int32_t>(R); }
    }
    if (groups) {
      d_kind = c.up(kind, G); d_q = c.up(quantile, G); d_m = c.up(multiplier, G); d_nj = c.up(n_jobs, G);
      r_grp = c.take<int32_t>(M); r_rt = c.take<int64_t>(M); r_ord = c.take<int32_t>(M); r_tmp = c.take<int32_t>(M);
      seg_s = c.take<int32_t>(G); seg_e = c.take<int32_t>(G); limit = c.take<double>(G);
      slot = c.take<int32_t>(K);
      os.part[0] = c.take<int32_t>(kmax);
      os.tile[0] = c.take<int32_t>((kmax + OS_TILE - 1) / OS_TILE + 1);
      e_grp = c.take<int32_t>(N); e_tid = c.take<int64_t>(N); e_pool = c.take<int32_t>(N); e_rt = c.take<int64_t>(N);
      e_ord = c.take<int32_t>(N); e_tmp = c.take<int32_t>(N);
      o_sgrp = c.take<int32_t>(N); o_stid = c.take<int64_t>(N); o_spool = c.take<int32_t>(N);
    }
  }))
    return rc;
  CK(pool, cudaMemsetAsync(cnt, 0, sizeof(int32_t) * 5, st));
  int& nl = r.nl;
  int64_t& d2h = r.d2h;
  if (rows) {
    int base = 0;
    for (const auto& h : hs) {
      const Table& t = h.first->run;
      const int live = (int)t.slot_of.size();
      if (!live) continue;
      compact(SweepRows{t.d_col, base, h.second, tid, pidx, start, maxrt, facts}, t.hw, nullptr, blk, cnt + 4, live, st,
              &nl);
      base += live;
    }
    CK(pool, csort::sort_indices(ord, tmp, (int)R, LessKeyTid{nullptr, tid}, st, &nl));
    if (linger)
      compact(KillSel{ord, tid, pidx, start, maxrt, facts, now, dflt, max_to, false, o_ltid, o_lpool}, (int)R, nullptr,
              blk, cnt + 0, (int)R, st, &nl);
    if (cancel)
      compact(KillSel{ord, tid, pidx, start, maxrt, facts, now, dflt, max_to, true, o_ctid, o_cpool}, (int)R, nullptr,
              blk, cnt + 1, (int)R, st, &nl);
  }
  if (groups) {
    // the limits, from the checked groups' records
    CK(pool, cudaMemsetAsync(seg_s, 0, sizeof(int32_t) * (size_t)G, st));
    CK(pool, cudaMemsetAsync(seg_e, 0, sizeof(int32_t) * (size_t)G, st));
    if (M > 0) {
      int base = 0;
      for (const auto& h : hs) {
        const Records& rc = h.first->rec;
        int64_t mk = 0;
        for (const auto& kv : h.first->rec_groups)
          if (kind[kv.first] == COOK_SWEEP_QUANTILE_DEVIATION) mk += kv.second;
        if (!mk) continue;
        compact(SweepRecords{rc.c.at<int32_t>(RC_GRP), rc.c.at<int32_t>(RC_RT), rc.c.at<uint8_t>(RC_LIVE), d_kind, base,
                             r_grp, r_rt}, (int)rc.tail, nullptr, blk, cnt + 4,
                (int)mk, st, &nl);
        base += (int)mk;
      }
      CK(pool, csort::sort_indices(r_ord, r_tmp, (int)M, LessKeyTid{r_grp, r_rt}, st, &nl));
      seg_bounds_kernel<<<((int)M + 255) / 256, 256, 0, st>>>(SortedKey{r_ord, nullptr, r_grp}, (int)M, seg_s, seg_e,
                                                              nullptr);
      nl++;
    }
    straggler_limit_kernel<<<(G + 255) / 256, 256, 0, st>>>(d_kind, d_q, d_m, d_nj, seg_s, seg_e, r_ord, r_rt, G, limit);
    nl++;
    // the entries, handle by handle
    int kbase = 0, ebase = 0;
    for (const auto& h : hs) {
      const PoolState* s = h.first;
      const int Kk = (int)s->grp_rows;
      if (!Kk) continue;
      const int32_t* glen = s->run.at<int32_t>(R_GLEN);
      compact(GroupedRows{s->run.at<uint8_t>(R_LIVE), glen, slot + kbase}, s->run.hw, nullptr, blk, cnt + 4, Kk, st, &nl);
      order_scan(os, RowLen{slot + kbase, glen}, Kk, r.S->gf0, st, &nl);
      ExpandArgs a = {os, slot + kbase, Kk, ebase, h.second, s->run.d_col, s->lists[L_RGROUP].at(0), d_kind, now,
                      e_grp, e_tid, e_pool, e_rt, cnt + 3};
      straggler_expand_kernel<<<(Kk + 255) / 256, 256, 0, st>>>(a);
      nl++;
      kbase += Kk;
      ebase += (int)s->lists[L_RGROUP].live;
    }
    CK(pool, csort::sort_indices(e_ord, e_tmp, (int)N, LessKeyTid{e_grp, e_tid}, st, &nl));
    compact(StragglerSel{e_ord, e_grp, e_tid, e_pool, e_rt, limit, o_sgrp, o_stid, o_spool}, (int)N, nullptr, blk,
            cnt + 2, (int)N, st, &nl);
  }
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  int32_t got[4];
  CK(pool, download(got, cnt, 4, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  if (got[3]) return set_err(pool, COOK_E_BADARG, "%s: a running task of a checked group starts after now_ms", who);
  if (rows && linger && got[0]) {
    CK(pool, download(l_tid, o_ltid, got[0], st, &d2h));
    CK(pool, download(l_pool, o_lpool, got[0], st, &d2h));
  }
  if (rows && cancel && got[1]) {
    CK(pool, download(c_tid, o_ctid, got[1], st, &d2h));
    CK(pool, download(c_pool, o_cpool, got[1], st, &d2h));
  }
  if (groups && got[2]) {
    CK(pool, download(s_grp, o_sgrp, got[2], st, &d2h));
    CK(pool, download(s_tid, o_stid, got[2], st, &d2h));
    CK(pool, download(s_pool, o_spool, got[2], st, &d2h));
  }
  if (int32_t rc = r.close(out_stats)) return rc;
  if (linger) *l_n = got[0];
  if (cancel) *c_n = got[1];
  if (strag) *s_n = got[2];
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_task_facts(cook_pool* pool, int32_t n, const int64_t* task_id,
                                         const int64_t* max_runtime_ms, const uint8_t* cancelled,
                                         const uint8_t* unknown) {
  const char* who = "cook_state_task_facts";
  return on_state(pool, who, [&](PoolState* S) {
    return task_facts(pool, S, who, n, task_id, max_runtime_ms, cancelled, unknown);
  });
}

extern "C" int32_t cook_state_task_reason(cook_pool* pool, int32_t n, const int64_t* task_id,
                                          const int32_t* reason_code) {
  const char* who = "cook_state_task_reason";
  return on_state(pool, who, [&](PoolState* S) { return task_reason(pool, S, who, n, task_id, reason_code); });
}

extern "C" int32_t cook_state_finish(cook_pool* pool, int32_t n, const int64_t* task_id, const int64_t* end_time_ms,
                                     const uint8_t* success) {
  const char* who = "cook_state_finish";
  return on_state(pool, who, [&](PoolState* S) { return finish(pool, S, who, n, task_id, end_time_ms, success); });
}

extern "C" int32_t cook_state_finish_history(cook_pool* pool, int32_t n, const int64_t* task_id,
                                             const int64_t* end_time_ms, const uint8_t* success,
                                             const int32_t* reason_code) {
  const char* who = "cook_state_finish_history";
  const FinishHistory fh{reason_code};
  return on_state(pool, who, [&](PoolState* S) { return finish(pool, S, who, n, task_id, end_time_ms, success, &fh); });
}

extern "C" int32_t cook_state_retry_config(cook_pool* pool, int32_t mea_culpa_limit, int32_t n_reasons,
                                           const int32_t* reason_code, const uint8_t* mea_culpa,
                                           const int32_t* failure_limit) {
  const char* who = "cook_state_retry_config";
  return on_state(pool, who, [&](PoolState* S) {
    return retry_config(pool, S, who, mea_culpa_limit, n_reasons, reason_code, mea_culpa, failure_limit);
  });
}

extern "C" int32_t cook_state_retry_facts(cook_pool* pool, int32_t n, const int64_t* job_id, const int32_t* max_retries,
                                          const uint8_t* flags, const int32_t* done_off, const int32_t* done_reason) {
  const char* who = "cook_state_retry_facts";
  return on_state(pool, who, [&](PoolState* S) {
    return retry_facts(pool, S, who, n, job_id, max_retries, flags, done_off, done_reason);
  });
}

extern "C" int32_t cook_state_status(cook_pool* pool, int32_t n, const int64_t* task_id, const uint8_t* success,
                                     const int64_t* end_time_ms, const int32_t* reason_code, const uint8_t* preempted,
                                     int32_t* out_outcome, int32_t* out_attempts) {
  const char* who = "cook_state_status";
  const FinishHistory fh{reason_code};
  const FinishStatus fs{preempted, out_outcome, out_attempts};
  return on_state(pool, who, [&](PoolState* S) {
    return finish(pool, S, who, n, task_id, end_time_ms, success, &fh, &fs);
  });
}

extern "C" int32_t cook_state_history_seed(cook_pool* pool, int64_t since_ms, int32_t n, const int64_t* task_id,
                                           const int32_t* user, const int64_t* start_ms, const int64_t* end_ms,
                                           const double* cpus, const double* mem, const uint8_t* success,
                                           const int32_t* reason_code) {
  const char* who = "cook_state_history_seed";
  return on_state(pool, who, [&](PoolState* S) {
    return history_seed(pool, S, who, since_ms, n, task_id, user, start_ms, end_ms, cpus, mem, success, reason_code);
  });
}

extern "C" int32_t cook_state_history_advance(cook_pool* pool, int64_t since_ms) {
  const char* who = "cook_state_history_advance";
  return on_state(pool, who, [&](PoolState* S) { return history_advance(pool, S, who, since_ms); });
}

extern "C" int32_t cook_state_group_runtimes(cook_pool* pool, int32_t n_add, const int32_t* group,
                                             const int32_t* runtime_s, int32_t n_forget, const int32_t* forget_group) {
  const char* who = "cook_state_group_runtimes";
  return on_state(pool, who, [&](PoolState* S) {
    return group_runtimes(pool, S, who, n_add, group, runtime_s, n_forget, forget_group);
  });
}

extern "C" int32_t cook_state_sweep(cook_pool* const* pools, int32_t n_pools, int64_t now_ms,
                                    int64_t default_timeout_ms, int64_t max_timeout_ms, int32_t n_groups,
                                    const int32_t* group_kind, const double* quantile, const double* multiplier,
                                    const int32_t* n_jobs, int32_t row_cap, int64_t* out_linger_task_id,
                                    int32_t* out_linger_pool, int32_t* out_n_linger, int64_t* out_cancel_task_id,
                                    int32_t* out_cancel_pool, int32_t* out_n_cancel, int32_t entry_cap,
                                    int32_t* out_straggler_group, int64_t* out_straggler_task_id,
                                    int32_t* out_straggler_pool, int32_t* out_n_straggler,
                                    cook_phase_stats* out_stats) {
  return sweep(pools, n_pools, now_ms, default_timeout_ms, max_timeout_ms, n_groups, group_kind, quantile, multiplier,
               n_jobs, row_cap, out_linger_task_id, out_linger_pool, out_n_linger, out_cancel_task_id, out_cancel_pool,
               out_n_cancel, entry_cap, out_straggler_group, out_straggler_task_id, out_straggler_pool, out_n_straggler,
               out_stats);
}

// ---- why a job is not scheduled (/unscheduled_jobs, unscheduled.clj:172-200): each queried job's status, its user's
// running usage plus the job, its place among its user's entries and the jobs ahead, and its plugin flag.  The host
// resolves each queried id to its row (a pending slot, or the running row of the job with the greatest task id) and
// its user; the device takes the live rows of the queried users, keeps one running row per (user, job), folds the
// users' usage over those in ascending task id and orders the users' entries as rank does.
namespace {

// the queried users: umap[user code] = its index k in quser, -1 for any other code; rank[k] = k (LessUserTask's name
// ranks: users in index order, and index nU last)
__global__ void unsched_users_kernel(const int32_t* quser, int nU, int32_t* umap, int32_t* rank) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > nU) return;
  rank[k] = k;
  if (k < nU) umap[quser[k]] = k;
}

// The entries: the queried users' live running rows dense in [0, R), their live pending rows in [R, R + J), as rank's
// task columns plus each entry's slot.  key: a pending entry's user index; the running entries' is written by
// job_rep_kernel.  ru: a running entry's user index.
struct UnschedCols {
  int32_t* key; int32_t* ru; int32_t* prio; int64_t* start; int64_t* tid; int64_t* jid; int32_t* slot;
  double* amt[3];   // [R]: the running entries' cpus, mem, gpus
};
struct UnschedRunRows {
  void* const* col; const int32_t* umap; UnschedCols o;
  __device__ bool keep(int i) const {
    return static_cast<const uint8_t*>(col[R_LIVE])[i] && umap[static_cast<const int32_t*>(col[R_USER])[i]] >= 0;
  }
  __device__ void emit(int i, int d) const {
    o.ru[d] = umap[static_cast<const int32_t*>(col[R_USER])[i]];
    o.prio[d] = static_cast<const int32_t*>(col[R_PRIO])[i];
    o.start[d] = static_cast<const int64_t*>(col[R_START])[i];
    o.tid[d] = static_cast<const int64_t*>(col[R_TID])[i];
    o.jid[d] = static_cast<const int64_t*>(col[R_JID])[i];
    o.slot[d] = i;
    o.amt[0][d] = static_cast<const double*>(col[R_CPUS])[i];
    o.amt[1][d] = static_cast<const double*>(col[R_MEM])[i];
    o.amt[2][d] = static_cast<const double*>(col[R_GPUS])[i];
  }
};
struct UnschedPendRows {
  void* const* col; const int32_t* umap; UnschedCols o; int R;
  __device__ bool keep(int i) const {
    return static_cast<const uint8_t*>(col[P_LIVE])[i] && umap[static_cast<const int32_t*>(col[P_USER])[i]] >= 0;
  }
  __device__ void emit(int i, int d) const {
    d += R;
    o.key[d] = umap[static_cast<const int32_t*>(col[P_USER])[i]];
    o.prio[d] = static_cast<const int32_t*>(col[P_PRIO])[i];
    o.start[d] = INT64_MAX;   // a pending job's synthetic task (tools.clj:582-588)
    o.tid[d] = -1;
    o.jid[d] = static_cast<const int64_t*>(col[P_JID])[i];
    o.slot[d] = i;
  }
};
// (scope, job id, task id, dense index): a (scope, job)'s running rows together, its greatest task id last.  The scope
// is a user (cook_state_unscheduled) or a handle (cook_state_user_usage).
struct LessScopeJobTask {
  const int32_t* scope; const int64_t* jid; const int64_t* tid;
  __device__ bool operator()(int32_t a, int32_t b) const {
    if (scope[a] != scope[b]) return scope[a] < scope[b];
    if (jid[a] != jid[b]) return jid[a] < jid[b];
    if (tid[a] != tid[b]) return tid[a] < tid[b];
    return a < b;
  }
};
// The representative of each (scope, job) is its last running row in that order: out[i] = val[i] for it, dead for
// the other rows.  out may be val: thread p reads no other row's val.
__global__ void job_rep_kernel(const int32_t* ord, int R, const int32_t* scope, const int64_t* jid, const int32_t* val,
                               int32_t dead, int32_t* out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  const int i = ord[p];
  bool rep = p == R - 1;
  if (!rep) {
    const int n = ord[p + 1];
    rep = scope[n] != scope[i] || jid[n] != jid[i];
  }
  out[i] = rep ? val[i] : dead;
}
// slot -> position in the entries' order, for the running representatives (rpos) and the pending rows (ppos)
__global__ void unsched_pos_kernel(const int32_t* ord, int E, int R, const int32_t* key, const int32_t* slot, int nU,
                                   int32_t* rpos, int32_t* ppos) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= E) return;
  const int i = ord[p];
  if (key[i] == nU) return;
  (i < R ? rpos : ppos)[slot[i]] = p;
}

struct UnschedArgs {
  const int32_t* qkey; int Q;   // per query: its pending slot, -2 - its running slot, or -1 (absent)
  const int32_t *ord, *key, *ostart, *rpos, *ppos; const int64_t* jid;
  const double* user_out; int nU;   // [4][nU]: count, cpus, mem, gpus of each user's running jobs
  void* const* pcol;
  double* usage; int32_t* pos; int32_t* n_ahead; int64_t* ahead; uint8_t* plugin;
};
// Thread per query: the position of its entry in its user's segment, the first min(position, AHEAD) entries' job
// ids (0 past them), and for a waiting job the usage fold continued by the job and the plugin flag.
__global__ void unsched_query_kernel(UnschedArgs a) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= a.Q) return;
  const int k = a.qkey[q];
  double u4[4] = {0.0, 0.0, 0.0, 0.0};
  int pos = -1, na = 0;
  uint8_t pl = 0;
  int64_t* ahead = a.ahead + (size_t)q * COOK_UNSCHED_AHEAD;
  if (k != -1) {
    const bool wait = k >= 0;
    const int p = wait ? a.ppos[k] : a.rpos[-2 - k];
    const int u = a.key[a.ord[p]], s0 = a.ostart[u];
    pos = p - s0;
    na = min(pos, (int)COOK_UNSCHED_AHEAD);
    for (int j = 0; j < na; j++) ahead[j] = a.jid[a.ord[s0 + j]];
    if (wait) {
      const int nU = a.nU;
      u4[0] = a.user_out[u] + 1.0;
      u4[1] = a.user_out[nU + u] + static_cast<const double*>(a.pcol[P_CPUS])[k];
      u4[2] = a.user_out[2 * nU + u] + static_cast<const double*>(a.pcol[P_MEM])[k];
      u4[3] = a.user_out[3 * nU + u] + static_cast<const double*>(a.pcol[P_GPUS])[k];
      pl = static_cast<const uint8_t*>(a.pcol[P_PLUGIN])[k] == 0;
    }
  }
  for (int j = na; j < COOK_UNSCHED_AHEAD; j++) ahead[j] = 0;
#pragma unroll
  for (int c = 0; c < 4; c++) a.usage[4 * (size_t)q + c] = u4[c];
  a.pos[q] = pos; a.n_ahead[q] = na; a.plugin[q] = pl;
}

int32_t unscheduled(cook_pool* pool, int n, const int64_t* job_id, uint8_t* out_status, double* out_usage,
                    int32_t* out_position, int32_t* out_n_ahead, int64_t* out_ahead, uint8_t* out_plugin,
                    cook_phase_stats* out_stats) {
  const char* who = "cook_state_unscheduled";
  // ---- every check before any device work or output
  if (n < 0) return pool ? set_err(pool, COOK_E_BADARG, "%s: n < 0", who) : COOK_E_BADARG;
  if (n == 0) {
    if (out_stats) *out_stats = cook_phase_stats{};
    return COOK_OK;
  }
  if (!pool) return COOK_E_BADARG;
  if (!job_id || !out_status || !out_usage || !out_position || !out_n_ahead || !out_ahead || !out_plugin)
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  // ---- host: each query's row and user, the queried users and their rows' counts, O(n log n)
  PoolState* S = state_of(pool, false);
  std::vector<int32_t> qkey(n, -1), qu(n, -1), quser;
  for (int i = 0; S && i < n; i++) {
    auto p = S->pend.slot_of.find(job_id[i]);
    if (p != S->pend.slot_of.end()) {
      qkey[i] = p->second;
      qu[i] = S->pinfo[p->second].user;
      continue;
    }
    auto r = S->jobs_r.find(job_id[i]);
    if (r == S->jobs_r.end()) continue;
    int32_t best = r->second[0];
    for (int32_t s : r->second) if (S->rtid[s] > S->rtid[best]) best = s;
    qkey[i] = -2 - best;
    qu[i] = S->ruser[best];
  }
  for (int i = 0; i < n; i++) {
    out_status[i] = qkey[i] == -1 ? COOK_UNSCHED_ABSENT : qkey[i] >= 0 ? COOK_UNSCHED_WAITING : COOK_UNSCHED_RUNNING;
    if (qu[i] >= 0) quser.push_back(qu[i]);
  }
  std::sort(quser.begin(), quser.end());
  quser.erase(std::unique(quser.begin(), quser.end()), quser.end());
  const int nU = (int)quser.size();
  if (nU == 0) {   // no queried job in the handle: without device work
    memset(out_usage, 0, sizeof(double) * 4 * (size_t)n);
    for (int i = 0; i < n; i++) out_position[i] = -1;
    memset(out_n_ahead, 0, sizeof(int32_t) * (size_t)n);
    memset(out_ahead, 0, sizeof(int64_t) * COOK_UNSCHED_AHEAD * (size_t)n);
    memset(out_plugin, 0, (size_t)n);
    return no_rows(out_stats);
  }
  int R = 0, J = 0;
  for (int32_t u : quser) {
    auto r = S->users_r.find(u);
    if (r != S->users_r.end()) R += (int)r->second;
    auto p = S->users_p.find(u);
    if (p != S->users_p.end()) J += (int)p->second;
  }
  const int E = R + J;
  const int n_codes = std::max(count_max(S->users_p), count_max(S->users_r)) + 1;
  ReadCall rd(pool);
  if (int32_t rc = rd.open(who)) return rc;   // S: the handle holds the queried rows
  cudaStream_t st = rd.st;
  // ---- one carve: the maps, the entries, the three orders, the fold, the outputs; up the users and the query keys
  UnschedCols o = {};
  int32_t *umap = nullptr, *rank = nullptr, *blk = nullptr, *cnt = nullptr, *ord1 = nullptr, *ord3 = nullptr;
  int32_t *tmp = nullptr, *ostart = nullptr, *oend = nullptr, *rpos = nullptr, *ppos = nullptr;
  const int32_t *d_quser = nullptr, *d_qkey = nullptr;
  UsageFold f;   // the users' fold over the running representatives: keyed by o.key, in ascending task id
  f.R = R; f.U = nU;
  UnschedArgs a = {};
  const int hw = std::max(S->run.hw, S->pend.hw);
  if (int32_t rc = rd.scratch([&](Carve& c) {
    umap = c.take<int32_t>(n_codes); rank = c.take<int32_t>(nU + 1);
    blk = c.take<int32_t>((size_t)hw / CP_BLOCK + 2); cnt = c.take<int32_t>(2);
    o.key = c.take<int32_t>(E); o.prio = c.take<int32_t>(E); o.start = c.take<int64_t>(E);
    o.tid = c.take<int64_t>(E); o.jid = c.take<int64_t>(E); o.slot = c.take<int32_t>(E);
    ord3 = c.take<int32_t>(E); tmp = c.take<int32_t>(E);
    ostart = c.take<int32_t>(nU + 2); oend = c.take<int32_t>(nU + 2);
    rpos = c.take<int32_t>(std::max(S->run.hw, 1)); ppos = c.take<int32_t>(std::max(S->pend.hw, 1));
    f.a.user_out = c.take<double>(4 * (size_t)nU);
    if (R) {
      o.ru = c.take<int32_t>(R);
      for (int k = 0; k < 3; k++) o.amt[k] = c.take<double>(R);
      ord1 = c.take<int32_t>(R);
      f.gf = c.take<GridFlag>(1);
      f.take_segs(c, US_USER, nU, true);   // nU + 1 bounds: the non-representatives' segment nU
    }
    a.usage = c.take<double>(4 * (size_t)n); a.pos = c.take<int32_t>(n); a.n_ahead = c.take<int32_t>(n);
    a.ahead = c.take<int64_t>(COOK_UNSCHED_AHEAD * (size_t)n); a.plugin = c.take<uint8_t>(n);
    d_quser = c.up(quser.data(), nU);
    d_qkey = c.up(qkey.data(), n);
  }))
    return rc;
  int& nl = rd.nl;
  int64_t& d2h = rd.d2h;
  CK(pool, cudaMemsetAsync(umap, 0xff, sizeof(int32_t) * (size_t)n_codes, st));
  unsched_users_kernel<<<(nU + 256) / 256, 256, 0, st>>>(d_quser, nU, umap, rank);
  nl++;
  // the entries
  if (R) compact(UnschedRunRows{S->run.d_col, umap, o}, S->run.hw, nullptr, blk, cnt, R, st, &nl);
  if (J) compact(UnschedPendRows{S->pend.d_col, umap, o, R}, S->pend.hw, nullptr, blk, cnt + 1, J, st, &nl);
  // one running row per (user, job): it keeps its user index as key, the other rows get nU, a segment after every
  // user's that no output reads; then the users' folds over the representatives in ascending task id
  if (R) {
    CK(pool, csort::sort_indices(ord1, tmp, R, LessScopeJobTask{o.ru, o.jid, o.tid}, st, &nl));
    job_rep_kernel<<<(R + 255) / 256, 256, 0, st>>>(ord1, R, o.ru, o.jid, o.ru, nU, o.key);
    nl++;
    f.rows.user = o.key; f.rows.id = o.tid;
    for (int k = 0; k < 3; k++) f.rows.amt[k] = o.amt[k];
    f.tmp = tmp;
    CK(pool, f.fold(st, &nl));
  } else {
    CK(pool, cudaMemsetAsync(f.a.user_out, 0, sizeof(double) * 4 * (size_t)nU, st));
  }
  // the users' entries in rank's same-user order, each entry's position by slot, then the queries
  CK(pool, csort::sort_indices(ord3, tmp, E, LessUserTask{o.key, o.prio, o.start, o.tid, o.jid, rank}, st, &nl));
  CK(pool, cudaMemsetAsync(ostart, 0, sizeof(int32_t) * (nU + 1), st));
  seg_bounds_kernel<<<(E + 255) / 256, 256, 0, st>>>(SortedKey{ord3, nullptr, o.key}, E, ostart, oend, nullptr);
  unsched_pos_kernel<<<(E + 255) / 256, 256, 0, st>>>(ord3, E, R, o.key, o.slot, nU, rpos, ppos);
  a.qkey = d_qkey; a.Q = n;
  a.ord = ord3; a.key = o.key; a.ostart = ostart; a.rpos = rpos; a.ppos = ppos; a.jid = o.jid;
  a.user_out = f.a.user_out; a.nU = nU; a.pcol = S->pend.d_col;
  unsched_query_kernel<<<(n + 127) / 128, 128, 0, st>>>(a);
  nl += 3;
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  CK(pool, download(out_usage, a.usage, 4 * (size_t)n, st, &d2h));
  CK(pool, download(out_position, a.pos, n, st, &d2h));
  CK(pool, download(out_n_ahead, a.n_ahead, n, st, &d2h));
  CK(pool, download(out_ahead, a.ahead, COOK_UNSCHED_AHEAD * (size_t)n, st, &d2h));
  CK(pool, download(out_plugin, a.plugin, n, st, &d2h));
  return rd.close(out_stats);
}

}  // namespace

extern "C" int32_t cook_state_unscheduled(cook_pool* pool, int32_t n, const int64_t* job_id, uint8_t* out_status,
                                          double* out_usage, int32_t* out_position, int32_t* out_n_ahead,
                                          int64_t* out_ahead_job_id, uint8_t* out_plugin_deferred,
                                          cook_phase_stats* out_stats) {
  return unscheduled(pool, n, job_id, out_status, out_usage, out_position, out_n_ahead, out_ahead_job_id,
                     out_plugin_deferred, out_stats);
}

// ---- the running usage of users (/usage, get-user-usage api.clj:2946-2969): per (user, scope, group) segment the
// number of running jobs and the left folds of cpus, mem and gpus over one representative per running job, and each
// group segment's job ids.  The host sizes every buffer from its per-user counts; the device takes the queried users'
// live running rows of every handle, keeps each (handle, job)'s row with the greatest task id, expands each
// representative into one entry per level the call asks for, sorts the entries once by (segment, task id, dense
// index) and folds each segment with fold.cuh's segment fold.
namespace {

constexpr int32_t UU_DEAD = INT32_MAX;   // the user of an entry whose row is not its job's representative: sorts last

__global__ void uu_users_kernel(const int32_t* quser, int nU, int32_t n_codes, uint8_t* umap) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < nU && quser[k] < n_codes) umap[quser[k]] = 1;
}

// one handle's live running rows of the queried users (umap null: every user), dense after the handles before it
struct UURows {
  void* const* col; const uint8_t* umap; int base; int32_t pool; const int32_t* arena;
  int32_t* user; int64_t* jid; int64_t* tid; int32_t* pidx; int32_t* grp; double* amt[3];
  __device__ bool keep(int i) const {
    return static_cast<const uint8_t*>(col[R_LIVE])[i] && (!umap || umap[static_cast<const int32_t*>(col[R_USER])[i]]);
  }
  __device__ void emit(int i, int d) const {
    d += base;
    user[d] = static_cast<const int32_t*>(col[R_USER])[i];
    jid[d] = static_cast<const int64_t*>(col[R_JID])[i];
    tid[d] = static_cast<const int64_t*>(col[R_TID])[i];
    pidx[d] = pool;
    const int32_t len = static_cast<const int32_t*>(col[R_GLEN])[i];
    grp[d] = len > 0 ? arena[static_cast<const int32_t*>(col[R_GOFF])[i]] : COOK_UU_UNGROUPED;
    amt[0][d] = static_cast<const double*>(col[R_CPUS])[i];
    amt[1][d] = static_cast<const double*>(col[R_MEM])[i];
    amt[2][d] = static_cast<const double*>(col[R_GPUS])[i];
  }
};
// The entries: entry l * R + i is row i at level l.  Bit 0 of the level's code scopes the entry to its handle, bit 1
// keys it by its group (per_pool: codes 0 .. L - 1; else 0 and, by_group, 2).  user: UU_DEAD for a row that is not
// a representative.
struct UUKey {
  int32_t* user; int32_t* scope; int32_t* grp;
  __device__ bool same(int a, int b) const { return user[a] == user[b] && scope[a] == scope[b] && grp[a] == grp[b]; }
};
__global__ void uu_expand_kernel(int R, int E, int per_pool, const int32_t* user, const int32_t* pidx,
                                 const int32_t* grp, UUKey k, int32_t* row) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= E) return;
  const int l = x / R, i = x - l * R, code = per_pool ? l : l << 1;
  k.user[x] = user[i];
  k.scope[x] = code & 1 ? pidx[i] : -1;
  k.grp[x] = code & 2 ? grp[i] : COOK_UU_TOTAL;
  row[x] = i;
}
// (user, scope, group, task id, dense index): the segments in the output order, each in its fold order
struct LessSegTid {
  UUKey k; const int32_t* row; const int64_t* tid;
  __device__ bool operator()(int32_t a, int32_t b) const {
    if (k.user[a] != k.user[b]) return k.user[a] < k.user[b];
    if (k.scope[a] != k.scope[b]) return k.scope[a] < k.scope[b];
    if (k.grp[a] != k.grp[b]) return k.grp[a] < k.grp[b];
    const int ra = row[a], rb = row[b];
    if (tid[ra] != tid[rb]) return tid[ra] < tid[rb];
    if (ra != rb) return ra < rb;
    return a < b;
  }
};
// the last position of each segment of the sorted entries: end[d] = one past segment d's last, segment d starting
// where segment d - 1 ends
struct UUSegEnds {
  const int32_t* ord; UUKey k; int E; int32_t* end;
  __device__ bool keep(int p) const {
    const int i = ord[p];
    return k.user[i] != UU_DEAD && (p == E - 1 || !k.same(i, ord[p + 1]));
  }
  __device__ void emit(int p, int d) const { end[d] = p + 1; }
};
// the group segments' job ids in segment order; head_off[p] of a segment's first position p: its first list index
struct UUListed {
  const int32_t* ord; UUKey k; const int32_t* row; const int64_t* jid; int64_t* o_jid; int32_t* head_off;
  __device__ bool keep(int p) const {
    const int i = ord[p];
    return k.user[i] != UU_DEAD && k.grp[i] != COOK_UU_TOTAL;
  }
  __device__ void emit(int p, int d) const {
    const int i = ord[p];
    o_jid[d] = jid[row[i]];
    if (p == 0 || !k.same(i, ord[p - 1])) head_off[p] = d;
  }
};
// the addends of the entry at position p of a sorted order: three columns of its row (the order-wide scan's and
// segment_fold's load, for /usage and the instance stats)
struct LoadEntry {
  const int32_t* ord; const int32_t* row; const double* col[3];
  __device__ void operator()(int p, double (&x)[3]) const {
    const int r = row[ord[p]];
    x[0] = col[0][r]; x[1] = col[1][r]; x[2] = col[2][r];
  }
};
// fold_segments' output: segment g's key, job count and cpus, mem and gpus folds in ascending (task id, dense index)
struct UUFoldOut {
  const int32_t* ord; UUKey k; const int32_t* head_off;   // head_off null: no lists
  int32_t *o_user, *o_scope, *o_grp, *o_off; int64_t* o_jobs; double* o_amt[3];
  __device__ void operator()(int g, int s, int e, const double (&acc)[3]) const {
    const int i = ord[s];
    o_user[g] = k.user[i]; o_scope[g] = k.scope[i]; o_grp[g] = k.grp[i];
    o_jobs[g] = e - s;
#pragma unroll
    for (int j = 0; j < 3; j++) o_amt[j][g] = acc[j];
    if (head_off) o_off[g] = k.grp[i] == COOK_UU_TOTAL ? -1 : head_off[s];
  }
};

int32_t user_usage(cook_pool* const* pools, int n, const int32_t* user, int nU, int per_pool, int by_group,
                   int seg_cap, int32_t* o_user, int32_t* o_scope, int32_t* o_group, int64_t* o_jobs, double* o_cpus,
                   double* o_mem, double* o_gpus, int32_t* o_off, int job_cap, int64_t* o_jid, int32_t* o_nseg,
                   int32_t* o_njob, cook_phase_stats* out_stats) {
  const char* who = "cook_state_user_usage";
  // ---- every check before any device work or output
  if (int32_t rc = check_handle_set(pools, n, who)) return rc;
  cook_pool* pool = pools[0];
  const bool pp = per_pool != 0, bg = by_group != 0;
  if (!o_user || !o_scope || !o_group || !o_jobs || !o_cpus || !o_mem || !o_gpus || !o_nseg || !o_njob ||
      (bg && (!o_off || !o_jid)))
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (user ? nU < 0 : nU != 0) return set_err(pool, COOK_E_BADARG, "%s: n_users < 0, or n_users without user", who);
  std::vector<int32_t> q(user, user + (user ? nU : 0));
  std::sort(q.begin(), q.end());
  if (!q.empty() && q[0] < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative user code", who);
  if (std::adjacent_find(q.begin(), q.end()) != q.end()) return set_err(pool, COOK_E_BADARG, "%s: a user code twice", who);
  // the handles with rows of the queried users, their pool index and row count; sizes from the host-side counts
  struct Src { const PoolState* s; int32_t k; int live; };
  std::vector<Src> hs;
  int64_t R = 0;
  int hw = 0;
  int32_t n_codes = 0;
  for (int k = 0; k < n; k++) {
    const PoolState* s = static_cast<const PoolState*>(pools[k]->state);
    if (!s) continue;
    int64_t r = 0;
    if (!user) {
      r = (int64_t)s->run.slot_of.size();
    } else {
      for (int32_t u : q) {
        auto it = s->users_r.find(u);
        if (it != s->users_r.end()) r += it->second;
      }
    }
    if (!r) continue;
    hs.push_back({s, k, (int)r});
    R += r;
    hw = std::max(hw, s->run.hw);
    n_codes = std::max(n_codes, count_max(s->users_r) + 1);
  }
  const int L = (1 + pp) * (1 + bg);
  if (R * L > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 entries", who);
  if (seg_cap < R * L) return set_err(pool, COOK_E_BADARG, "%s: seg_cap below the queried users' rows' bound", who);
  if (bg && job_cap < R * (1 + pp))
    return set_err(pool, COOK_E_BADARG, "%s: job_cap below the queried users' rows' bound", who);
  if (R == 0) {   // no row to read: empty results without device work
    *o_nseg = 0;
    *o_njob = 0;
    return no_rows(out_stats);
  }
  ReadCall r(pool);
  if (int32_t rc = r.open(who)) return rc;
  cudaStream_t st = r.st;
  const int Rn = (int)R, E = Rn * L, J = bg ? Rn * (1 + pp) : 0;
  hw = std::max(hw, E);
  // ---- one carve: the rows, the representatives, the entries and their order, the folds, the outputs
  int32_t *cnt = nullptr, *blk = nullptr, *ord1 = nullptr, *tmp = nullptr, *ord = nullptr, *end = nullptr;
  int32_t *r_user = nullptr, *r_pidx = nullptr, *r_grp = nullptr, *row = nullptr, *head_off = nullptr;
  int64_t *r_jid = nullptr, *r_tid = nullptr, *d_jid = nullptr;
  double* amt[3] = {};
  uint8_t* umap = nullptr;
  const int32_t* d_q = nullptr;
  GridFlag* gf = nullptr;
  UUKey key = {};
  OrderScan<double, 3> os = {};
  UUFoldOut a = {};
  if (int32_t rc = r.scratch([&](Carve& c) {
    cnt = c.take<int32_t>(3);   // segments, listed jobs, the row compactions' own
    blk = c.take<int32_t>((size_t)hw / CP_BLOCK + 2);
    if (user) umap = c.take<uint8_t>(n_codes);
    r_user = c.take<int32_t>(Rn); r_pidx = c.take<int32_t>(Rn); r_grp = c.take<int32_t>(Rn);
    r_jid = c.take<int64_t>(Rn); r_tid = c.take<int64_t>(Rn);
    for (int k = 0; k < 3; k++) amt[k] = c.take<double>(Rn);
    ord1 = c.take<int32_t>(Rn);
    gf = c.take<GridFlag>(1);
    key.user = c.take<int32_t>(E); key.scope = c.take<int32_t>(E); key.grp = c.take<int32_t>(E);
    row = c.take<int32_t>(E); ord = c.take<int32_t>(E); tmp = c.take<int32_t>(E); end = c.take<int32_t>(E);
    for (int k = 0; k < 3; k++) {
      os.part[k] = c.take<double>(E);
      os.tile[k] = c.take<double>(E / OS_TILE + 2);
    }
    a.o_user = c.take<int32_t>(E); a.o_scope = c.take<int32_t>(E); a.o_grp = c.take<int32_t>(E);
    a.o_jobs = c.take<int64_t>(E);
    for (int k = 0; k < 3; k++) a.o_amt[k] = c.take<double>(E);
    if (bg) {
      a.o_off = c.take<int32_t>(E); head_off = c.take<int32_t>(E);
      d_jid = c.take<int64_t>(J);
    }
    if (user) d_q = c.up(q.data(), nU);
  }))
    return rc;
  CK(pool, cudaMemsetAsync(cnt, 0, sizeof(int32_t) * 3, st));
  CK(pool, cudaMemsetAsync(gf, 0, sizeof(GridFlag), st));
  int& nl = r.nl;
  int64_t& d2h = r.d2h;
  if (user) {
    CK(pool, cudaMemsetAsync(umap, 0, (size_t)n_codes, st));
    uu_users_kernel<<<(nU + 255) / 256, 256, 0, st>>>(d_q, nU, n_codes, umap);
    nl++;
  }
  int base = 0;
  for (const Src& h : hs) {
    compact(UURows{h.s->run.d_col, umap, base, h.k, h.s->lists[L_RGROUP].at(0), r_user, r_jid, r_tid, r_pidx, r_grp,
                   {amt[0], amt[1], amt[2]}},
            h.s->run.hw, nullptr, blk, cnt + 2, h.live, st, &nl);
    base += h.live;
  }
  grid_check_kernel<<<(Rn + 255) / 256, 256, 0, st>>>(amt[0], amt[1], amt[2], Rn, gf);
  nl++;
  // one representative per (handle, job): the other rows' user becomes UU_DEAD in place; then every level's entries
  // in one (segment, task id) order, and each segment's left folds
  CK(pool, csort::sort_indices(ord1, tmp, Rn, LessScopeJobTask{r_pidx, r_jid, r_tid}, st, &nl));
  job_rep_kernel<<<(Rn + 255) / 256, 256, 0, st>>>(ord1, Rn, r_pidx, r_jid, r_user, UU_DEAD, r_user);
  uu_expand_kernel<<<(E + 255) / 256, 256, 0, st>>>(Rn, E, pp, r_user, r_pidx, r_grp, key, row);
  nl += 2;
  CK(pool, csort::sort_indices(ord, tmp, E, LessSegTid{key, row, r_tid}, st, &nl));
  compact(UUSegEnds{ord, key, E, end}, E, nullptr, blk, cnt + 0, E, st, &nl);
  if (bg) compact(UUListed{ord, key, row, r_jid, d_jid, head_off}, E, nullptr, blk, cnt + 1, J, st, &nl);
  const LoadEntry load{ord, row, {amt[0], amt[1], amt[2]}};
  order_scan(os, load, E, gf, st, &nl);
  a.ord = ord; a.k = key; a.head_off = head_off;
  fold_segments(end, cnt, E, true, os, gf, load, a, st, &nl);
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  int32_t got[2];
  CK(pool, download(got, cnt, 2, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  const int ns = got[0], nj = bg ? got[1] : 0;
  CK(pool, download(o_user, a.o_user, ns, st, &d2h));
  CK(pool, download(o_scope, a.o_scope, ns, st, &d2h));
  CK(pool, download(o_group, a.o_grp, ns, st, &d2h));
  CK(pool, download(o_jobs, a.o_jobs, ns, st, &d2h));
  CK(pool, download(o_cpus, a.o_amt[0], ns, st, &d2h));
  CK(pool, download(o_mem, a.o_amt[1], ns, st, &d2h));
  CK(pool, download(o_gpus, a.o_amt[2], ns, st, &d2h));
  if (bg) {
    CK(pool, download(o_off, a.o_off, ns, st, &d2h));
    CK(pool, download(o_jid, d_jid, nj, st, &d2h));
  }
  if (int32_t rc = r.close(out_stats)) return rc;
  *o_nseg = ns;
  *o_njob = nj;
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_user_usage(cook_pool* const* pools, int32_t n_pools, const int32_t* user,
                                         int32_t n_users, int32_t per_pool, int32_t by_group, int32_t seg_cap,
                                         int32_t* out_user, int32_t* out_scope, int32_t* out_group, int64_t* out_jobs,
                                         double* out_cpus, double* out_mem, double* out_gpus, int32_t* out_list_off,
                                         int32_t job_cap, int64_t* out_job_id, int32_t* out_n_seg,
                                         int32_t* out_n_job, cook_phase_stats* out_stats) {
  return user_usage(pools, n_pools, user, n_users, per_pool, by_group, seg_cap, out_user, out_scope, out_group,
                    out_jobs, out_cpus, out_mem, out_gpus, out_list_off, job_cap, out_job_id, out_n_seg, out_n_job,
                    out_stats);
}

// ---- instance stats (/stats/instances, task-stats/get-stats task_stats.clj): over the selected live running rows,
// per segment (overall, per reason, per (user, reason)) the count, and per metric (run-time, cpu and mem seconds)
// the left fold and the nearest-rank percentiles 50 75 95 99 100; and the ten users with the largest cpu and mem
// totals.  Two sources: the live running rows (cook_state_instance_stats: the live rows of every handle compacted
// into one range, the selection compacted from it with the metrics at one now) and the finished rows
// (cook_state_history_stats: the selection compacted straight from each handle's history table with end - start).
// From the selected rows on, one pipeline (is_answer): each selected row becomes one entry per level (overall, reason,
// (user, reason), user).  One sort by (segment, task id, pool index, table position) gives every segment's fold
// order; per metric, one sort of the first three levels by (segment, value) gives the ranks.  The user level's folds
// feed the leaders and are not returned.
namespace {

constexpr int IS_LEVELS = 4, IS_USER = 3;   // the levels' kinds: COOK_IS_OVERALL, _REASON, _USER_REASON, then users
__device__ __forceinline__ int is_pct(int j) { return j == 0 ? 50 : j == 1 ? 75 : j == 2 ? 95 : j == 3 ? 99 : 100; }

// one handle's live running rows, dense after the handles before it
struct ISRows {
  void* const* col; int base; int32_t pool;
  int32_t* user; int32_t* reason; int64_t* tid; int32_t* pidx; int64_t* start; double* cpus; double* mem;
  uint8_t* facts;
  __device__ bool keep(int i) const { return static_cast<const uint8_t*>(col[R_LIVE])[i]; }
  template <class V> void outs(V&& v) { v(user); v(reason); v(tid); v(pidx); v(start); v(cpus); v(mem); v(facts); }
  __device__ void emit(int i, int d) const {
    d += base;
    user[d] = static_cast<const int32_t*>(col[R_USER])[i];
    reason[d] = static_cast<const int32_t*>(col[R_REASON])[i];
    tid[d] = static_cast<const int64_t*>(col[R_TID])[i];
    pidx[d] = pool;
    start[d] = static_cast<const int64_t*>(col[R_START])[i];
    cpus[d] = static_cast<const double*>(col[R_CPUS])[i];
    mem[d] = static_cast<const double*>(col[R_MEM])[i];
    facts[d] = static_cast<const uint8_t*>(col[R_FACTS])[i];
  }
};
// the selected rows: status, task id in [tid_lo, tid_hi), start in [start_ms, end_ms); their metrics with one now
// (task->task-entry: run-time-seconds = (double) ms / 1000.0, times cpus and mem).  A selected row that starts after
// now sets *bad.
struct ISSel {
  const int32_t* user; const int32_t* reason; const int64_t* tid; const int32_t* pidx; const int64_t* start;
  const double* cpus; const double* mem; const uint8_t* facts;
  int64_t now, start_ms, end_ms, tid_lo, tid_hi; int unknown;
  int32_t* s_user; int32_t* s_reason; int64_t* s_tid; int32_t* s_pidx; double* met[3]; int32_t* bad;
  __device__ bool keep(int i) const {
    return ((facts[i] & RF_UNKNOWN) != 0) == (unknown != 0) && tid[i] >= tid_lo && tid[i] < tid_hi &&
           start[i] >= start_ms && start[i] < end_ms;
  }
  __device__ void emit(int i, int d) const {
    s_user[d] = user[i]; s_reason[d] = reason[i]; s_tid[d] = tid[i]; s_pidx[d] = pidx[i];
    if (start[i] > now) *bad = 1;
    const double rt = (double)(now - start[i]) / 1000.0;
    met[0][d] = rt;
    met[1][d] = rt * cpus[i];
    met[2][d] = rt * mem[i];
  }
};

// The entries: entry l * S + i is selected row i at level l, keyed (kind, user, reason); the segment of an entry is
// its key.
struct ISKey {
  int32_t* kind; int32_t* user; int32_t* reason;
  __device__ bool same(int a, int b) const { return kind[a] == kind[b] && user[a] == user[b] && reason[a] == reason[b]; }
  __device__ int cmp(int a, int b) const {
    if (kind[a] != kind[b]) return kind[a] < kind[b] ? -1 : 1;
    if (user[a] != user[b]) return user[a] < user[b] ? -1 : 1;
    if (reason[a] != reason[b]) return reason[a] < reason[b] ? -1 : 1;
    return 0;
  }
};
__global__ void is_expand_kernel(int S, const int32_t* user, const int32_t* reason, ISKey k, int32_t* row) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= IS_LEVELS * S) return;
  const int l = x / S, i = x - l * S;
  k.kind[x] = l;
  k.user[x] = l >= COOK_IS_USER_REASON ? user[i] : -1;
  k.reason[x] = l == COOK_IS_REASON || l == COOK_IS_USER_REASON ? reason[i] : -1;
  row[x] = i;
}
// (segment, task id, pool index, table position when given, entry): the segments in the output order, each in its
// fold order
struct LessSegTidPool {
  ISKey k; const int32_t* row; const int64_t* tid; const int32_t* pidx; const int32_t* pos;
  __device__ bool operator()(int32_t a, int32_t b) const {
    const int c = k.cmp(a, b);
    if (c) return c < 0;
    const int ra = row[a], rb = row[b];
    if (tid[ra] != tid[rb]) return tid[ra] < tid[rb];
    if (pidx[ra] != pidx[rb]) return pidx[ra] < pidx[rb];
    if (pos && pos[ra] != pos[rb]) return pos[ra] < pos[rb];
    return a < b;
  }
};
// (segment, value, entry): the ranks of one metric; no value is NaN or -0.0, so equal values are equal bits
struct LessSegValue {
  ISKey k; const int32_t* row; const double* v;
  __device__ bool operator()(int32_t a, int32_t b) const {
    const int c = k.cmp(a, b);
    if (c) return c < 0;
    const double va = v[row[a]], vb = v[row[b]];
    if (va != vb) return va < vb;
    return a < b;
  }
};
struct ISSegEnds {   // end[d] = one past segment d's last position, segment d starting where segment d - 1 ends
  const int32_t* ord; ISKey k; int E; int32_t* end;
  __device__ bool keep(int p) const { return p == E - 1 || !k.same(ord[p], ord[p + 1]); }
  __device__ void emit(int p, int d) const { end[d] = p + 1; }
};
// fold_segments' output: segment g's key, count and the left folds of the three metrics in ascending (task id, pool
// index)
struct ISFoldOut {
  const int32_t* ord; ISKey k;
  int32_t *o_kind, *o_user, *o_reason; int64_t* o_count; double* o_total;   // o_total [3 * segment + metric]
  __device__ void operator()(int g, int s, int e, const double (&acc)[3]) const {
    const int i = ord[s];
    o_kind[g] = k.kind[i]; o_user[g] = k.user[i]; o_reason[g] = k.reason[i];
    o_count[g] = e - s;
#pragma unroll
    for (int j = 0; j < 3; j++) o_total[3 * g + j] = acc[j];
  }
};
// thread per (returned segment, metric): element ceil(p * n / 100) - 1 of the segment's ascending values
// (percentile, task_stats.clj: p/100 is a ratio, so exact integer arithmetic).  The user segments come last and are
// skipped.
__global__ void is_pct_kernel(const int32_t* n_seg, const int32_t* end, const int32_t* o_kind, const int32_t* ord0,
                              const int32_t* ord1, const int32_t* ord2, const int32_t* row, const double* m0,
                              const double* m1, const double* m2, double* o_pct) {
  const int n = *n_seg;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < 3 * n; t += gridDim.x * blockDim.x) {
    const int g = t / 3, m = t - 3 * g;
    if (o_kind[g] == IS_USER) continue;
    const int s = g ? end[g - 1] : 0;
    const int64_t c = end[g] - s;
    const int32_t* ord = m == 0 ? ord0 : m == 1 ? ord1 : ord2;
    const double* v = m == 0 ? m0 : m == 1 ? m1 : m2;
#pragma unroll
    for (int j = 0; j < 5; j++) o_pct[15 * g + 5 * m + j] = v[row[ord[s + (int)((is_pct(j) * c + 99) / 100) - 1]]];
  }
}
// block k (0: cpu seconds, 1: mem seconds): the first COOK_IS_LEADERS users in (total descending, user ascending)
// order, one block-wide selection per place, each of the users after the previous pick.  The user segments are the
// last ones, [n_ret, n_seg), in ascending user; block 0 writes n_ret and the leaders' number to counts[0, 2).
__global__ void __launch_bounds__(256) is_leaders_kernel(const int32_t* n_seg, const int32_t* o_kind,
                                                         const int32_t* o_user, const double* o_total,
                                                         int32_t* l_user, double* l_total, int32_t* counts) {
  __shared__ int s_ret;
  __shared__ double s_v[8];
  __shared__ int32_t s_u[8];
  const int n = *n_seg, k = blockIdx.x + 1, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n;   // the first user segment: kinds ascend
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (o_kind[mid] < IS_USER) lo = mid + 1;
      else hi = mid;
    }
    s_ret = lo;
  }
  __syncthreads();
  const int first = s_ret, U = n - first, L = min(U, COOK_IS_LEADERS);
  double pv = 0.0;
  int32_t pu = -1;
  for (int r = 0; r < L; r++) {
    double bv = -1.0;
    int32_t bu = INT32_MAX;
    for (int g = first + threadIdx.x; g < n; g += blockDim.x) {
      const double v = o_total[3 * g + k];
      const int32_t u = o_user[g];
      const bool after = r == 0 || v < pv || (v == pv && u > pu);
      if (after && (v > bv || (v == bv && u < bu))) { bv = v; bu = u; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double v = __shfl_xor_sync(FULL_MASK, bv, o);
      const int32_t u = __shfl_xor_sync(FULL_MASK, bu, o);
      if (v > bv || (v == bv && u < bu)) { bv = v; bu = u; }
    }
    if (lane == 0) { s_v[w] = bv; s_u[w] = bu; }
    __syncthreads();
    bv = s_v[0]; bu = s_u[0];
    for (int q = 1; q < 8; q++)
      if (s_v[q] > bv || (s_v[q] == bv && s_u[q] < bu)) { bv = s_v[q]; bu = s_u[q]; }
    __syncthreads();
    if (threadIdx.x == 0) {
      l_user[blockIdx.x * COOK_IS_LEADERS + r] = bu;
      l_total[blockIdx.x * COOK_IS_LEADERS + r] = bv;
    }
    pv = bv; pu = bu;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    counts[0] = first;
    counts[1] = L;
  }
}

// The answer's outputs (cook_state_instance_stats' and cook_state_history_stats' out_* arguments).
struct ISOut {
  int32_t *kind, *user, *reason; int64_t* count; double *total, *pct; int32_t* lead_user; double* lead_total;
  int32_t *n_seg, *n_lead;
};
bool is_out_null(const ISOut& o) {
  return !o.kind || !o.user || !o.reason || !o.count || !o.total || !o.pct || !o.lead_user || !o.lead_total ||
         !o.n_seg || !o.n_lead;
}

// The selected rows with their metrics, and the pipeline's device buffers, carved by take() for at most Smax rows.
// cnt: [0] selected, [1] the source's flag, [2] segments, [3] returned segments, [4] leaders, [5] the compactions' own.
struct ISPipe {
  int32_t *cnt = nullptr, *blk = nullptr;
  int32_t *s_user = nullptr, *s_reason = nullptr, *s_pidx = nullptr, *s_pos = nullptr;
  int64_t* s_tid = nullptr;
  double* met[3] = {};
  GridFlag* gf = nullptr;
  ISKey key = {};
  int32_t *row = nullptr, *ord = nullptr, *tmp = nullptr, *end = nullptr, *vord[3] = {}, *l_user = nullptr;
  double *pct = nullptr, *l_total = nullptr;
  OrderScan<double, 3> os = {};
  ISFoldOut a = {};
  // blk_n: the most items any compaction of the call runs over; pos: the selection carries table positions
  void take(Carve& c, int Smax, int blk_n, bool pos) {
    const int Emax = IS_LEVELS * Smax;
    blk_n = std::max(blk_n, Emax);
    cnt = c.take<int32_t>(6);
    blk = c.take<int32_t>((size_t)blk_n / CP_BLOCK + 2);
    s_user = c.take<int32_t>(Smax); s_reason = c.take<int32_t>(Smax); s_pidx = c.take<int32_t>(Smax);
    if (pos) s_pos = c.take<int32_t>(Smax);
    s_tid = c.take<int64_t>(Smax);
    for (int k = 0; k < 3; k++) met[k] = c.take<double>(Smax);
    gf = c.take<GridFlag>(1);
    key.kind = c.take<int32_t>(Emax); key.user = c.take<int32_t>(Emax); key.reason = c.take<int32_t>(Emax);
    row = c.take<int32_t>(Emax); ord = c.take<int32_t>(Emax); tmp = c.take<int32_t>(Emax); end = c.take<int32_t>(Emax);
    for (int k = 0; k < 3; k++) vord[k] = c.take<int32_t>(Emax);
    for (int k = 0; k < 3; k++) {
      os.part[k] = c.take<double>(Emax);
      os.tile[k] = c.take<double>(Emax / OS_TILE + 2);
    }
    a.o_kind = c.take<int32_t>(Emax); a.o_user = c.take<int32_t>(Emax); a.o_reason = c.take<int32_t>(Emax);
    a.o_count = c.take<int64_t>(Emax); a.o_total = c.take<double>(3 * (size_t)Emax);
    pct = c.take<double>(15 * (size_t)Emax);
    l_user = c.take<int32_t>(2 * COOK_IS_LEADERS); l_total = c.take<double>(2 * COOK_IS_LEADERS);
  }
  cudaError_t clear(cudaStream_t st) const {
    cudaError_t e = cudaMemsetAsync(cnt, 0, sizeof(int32_t) * 6, st);
    return e == cudaSuccess ? cudaMemsetAsync(gf, 0, sizeof(GridFlag), st) : e;
  }
};

// From S selected rows on: the entries, the fold order and its segments, the folds, the ranks and the leaders; then
// ev[22], the downloads and the close.  More segments than seg_cap: only *o.n_seg is written, COOK_E_TOO_LARGE.
int32_t is_answer(ReadCall& r, ISPipe& p, int S, int32_t seg_cap, const ISOut& o, cook_phase_stats* out_stats) {
  cook_pool* pool = r.pool;
  cudaStream_t st = r.st;
  int* nl = &r.nl;
  int64_t* d2h = &r.d2h;
  const int E = IS_LEVELS * S, E3 = 3 * S;
  int32_t got[2] = {0, 0};
  ISFoldOut& a = p.a;
  if (S > 0) {
    // ---- the entries, the fold order and its segments, the folds
    grid_check_kernel<<<(S + 255) / 256, 256, 0, st>>>(p.met[0], p.met[1], p.met[2], S, p.gf);
    is_expand_kernel<<<(E + 255) / 256, 256, 0, st>>>(S, p.s_user, p.s_reason, p.key, p.row);
    *nl += 2;
    CK(pool, csort::sort_indices(p.ord, p.tmp, E, LessSegTidPool{p.key, p.row, p.s_tid, p.s_pidx, p.s_pos}, st, nl));
    compact(ISSegEnds{p.ord, p.key, E, p.end}, E, nullptr, p.blk, p.cnt + 2, E, st, nl);
    const LoadEntry load{p.ord, p.row, {p.met[0], p.met[1], p.met[2]}};
    order_scan(p.os, load, E, p.gf, st, nl);
    a.ord = p.ord; a.k = p.key;
    fold_segments(p.end, p.cnt + 2, E, true, p.os, p.gf, load, a, st, nl);
    // ---- the ranks: the three levels returned are entries [0, 3 S), whose segments lead the fold order's
    for (int k = 0; k < 3; k++)
      CK(pool, csort::sort_indices(p.vord[k], p.tmp, E3, LessSegValue{p.key, p.row, p.met[k]}, st, nl));
    is_pct_kernel<<<std::min((3 * E + 255) / 256, 4096), 256, 0, st>>>(p.cnt + 2, p.end, a.o_kind, p.vord[0], p.vord[1],
                                                                      p.vord[2], p.row, p.met[0], p.met[1], p.met[2],
                                                                      p.pct);
    is_leaders_kernel<<<2, 256, 0, st>>>(p.cnt + 2, a.o_kind, a.o_user, a.o_total, p.l_user, p.l_total, p.cnt + 3);
    *nl += 2;
    CK(pool, cudaGetLastError());
    CK(pool, download(got, p.cnt + 3, 2, st, d2h));
    CK(pool, cudaStreamSynchronize(st));
  }
  CK(pool, cudaEventRecord(pool->ev[22], st));
  const int ns = got[0], nlead = got[1];
  if (ns > seg_cap) {
    *o.n_seg = ns;
    return set_err(pool, COOK_E_TOO_LARGE, "more segments than seg_cap: %d", ns);
  }
  if (ns) {
    CK(pool, download(o.kind, a.o_kind, ns, st, d2h));
    CK(pool, download(o.user, a.o_user, ns, st, d2h));
    CK(pool, download(o.reason, a.o_reason, ns, st, d2h));
    CK(pool, download(o.count, a.o_count, ns, st, d2h));
    CK(pool, download(o.total, a.o_total, 3 * (size_t)ns, st, d2h));
    CK(pool, download(o.pct, p.pct, 15 * (size_t)ns, st, d2h));
  }
  for (int k = 0; k < 2 && nlead; k++) {
    CK(pool, download(o.lead_user + k * COOK_IS_LEADERS, p.l_user + k * COOK_IS_LEADERS, nlead, st, d2h));
    CK(pool, download(o.lead_total + k * COOK_IS_LEADERS, p.l_total + k * COOK_IS_LEADERS, nlead, st, d2h));
  }
  if (int32_t rc = r.close(out_stats)) return rc;
  *o.n_seg = ns;
  *o.n_lead = nlead;
  return COOK_OK;
}

int32_t is_empty(const ISOut& o, cook_phase_stats* out_stats) {
  *o.n_seg = 0;
  *o.n_lead = 0;
  return no_rows(out_stats);
}

int32_t instance_stats(cook_pool* const* pools, int n, int64_t now, int32_t status, int64_t start_ms, int64_t end_ms,
                       int64_t tid_lo, int64_t tid_hi, int32_t seg_cap, const ISOut& o, cook_phase_stats* out_stats) {
  const char* who = "cook_state_instance_stats";
  // ---- every check before any device work or output
  if (int32_t rc = check_handle_set(pools, n, who, true)) return rc;
  cook_pool* pool = pools[0];
  if (status != COOK_IS_RUNNING && status != COOK_IS_UNKNOWN) return set_err(pool, COOK_E_BADARG, "%s: an unknown status", who);
  if (end_ms <= start_ms) return set_err(pool, COOK_E_BADARG, "%s: end_ms <= start_ms", who);
  if (is_out_null(o)) return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  // the handles with rows and their pool index; sizes from the host-side counts
  std::vector<std::pair<const PoolState*, int32_t>> hs;
  int64_t R = 0;
  int hw = 0;
  for (int k = 0; k < n; k++) {
    const PoolState* s = static_cast<const PoolState*>(pools[k]->state);
    if (!s || s->run.slot_of.empty()) continue;
    hs.push_back({s, k});
    R += (int64_t)s->run.slot_of.size();
    hw = std::max(hw, s->run.hw);
  }
  if (R * IS_LEVELS > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 entries", who);
  if (seg_cap < 1 + 2 * R) return set_err(pool, COOK_E_BADARG, "%s: seg_cap below 1 + 2 * the live running rows", who);
  if (R == 0) return is_empty(o, out_stats);   // no row to read
  ReadCall r(pool);
  if (int32_t rc = r.open(who)) return rc;
  cudaStream_t st = r.st;
  const int Rn = (int)R;
  // ---- one carve, sized by the live rows: the rows, then the selection and the pipeline's buffers
  int32_t *a_user = nullptr, *a_reason = nullptr, *a_pidx = nullptr;
  int64_t *a_tid = nullptr, *a_start = nullptr;
  double *a_cpus = nullptr, *a_mem = nullptr;
  uint8_t* a_facts = nullptr;
  ISPipe p;
  if (int32_t rc = r.scratch([&](Carve& c) {
    a_user = c.take<int32_t>(Rn); a_reason = c.take<int32_t>(Rn); a_pidx = c.take<int32_t>(Rn);
    a_tid = c.take<int64_t>(Rn); a_start = c.take<int64_t>(Rn);
    a_cpus = c.take<double>(Rn); a_mem = c.take<double>(Rn); a_facts = c.take<uint8_t>(Rn);
    p.take(c, Rn, hw, false);
  }))
    return rc;
  CK(pool, p.clear(st));
  // ---- the selection and its metrics
  Gather g(pool);
  int base = 0;
  for (const auto& h : hs) {
    const int live = (int)h.first->run.slot_of.size();
    CK(pool, g.rows(pools[h.second],
                    ISRows{h.first->run.d_col, base, h.second, a_user, a_reason, a_tid, a_pidx, a_start, a_cpus, a_mem,
                           a_facts},
                    h.first->run.hw, live, p.blk, p.cnt + 5, &r.nl));
    base += live;
  }
  compact(ISSel{a_user, a_reason, a_tid, a_pidx, a_start, a_cpus, a_mem, a_facts, now, start_ms, end_ms, tid_lo, tid_hi,
                status == COOK_IS_UNKNOWN, p.s_user, p.s_reason, p.s_tid, p.s_pidx, {p.met[0], p.met[1], p.met[2]},
                p.cnt + 1},
          Rn, nullptr, p.blk, p.cnt + 0, Rn, st, &r.nl);
  CK(pool, cudaGetLastError());
  int32_t sel[2];
  CK(pool, download(sel, p.cnt, 2, st, &r.d2h));
  CK(pool, cudaStreamSynchronize(st));
  if (sel[1]) return set_err(pool, COOK_E_BADARG, "%s: a selected task starts after now_ms", who);
  return is_answer(r, p, sel[0], seg_cap, o, out_stats);
}

// one handle's finished rows of the status with task id in [tid_lo, tid_hi) and start in [start_ms, end_ms), dense
// after the handles before it, with their metrics (task-run-time with the instance's end: (double)(end - start) /
// 1000.0, times cpus and mem) and table position
struct HSSel {
  HistCols h; int base; int32_t pool; int success;
  int64_t start_ms, end_ms, tid_lo, tid_hi;
  int32_t* s_user; int32_t* s_reason; int64_t* s_tid; int32_t* s_pidx; int32_t* s_pos; double* met[3];
  __device__ bool keep(int i) const {
    return (h.ok[i] != 0) == (success != 0) && h.tid[i] >= tid_lo && h.tid[i] < tid_hi && h.start[i] >= start_ms &&
           h.start[i] < end_ms;
  }
  template <class V> void outs(V&& v) {
    v(s_user); v(s_reason); v(s_tid); v(s_pidx); v(s_pos); v(met[0]); v(met[1]); v(met[2]);
  }
  __device__ void emit(int i, int d) const {
    d += base;
    s_user[d] = h.user[i]; s_reason[d] = h.reason[i]; s_tid[d] = h.tid[i]; s_pidx[d] = pool; s_pos[d] = i;
    const double rt = (double)(h.end[i] - h.start[i]) / 1000.0;
    met[0][d] = rt;
    met[1][d] = rt * h.cpus[i];
    met[2][d] = rt * h.mem[i];
  }
};
// the selected rows' count, *out += (integer adds: any order is exact)
__global__ void hs_count_kernel(HSSel f, int n, int32_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = __reduce_add_sync(FULL_MASK, (i < n && f.keep(i)) ? 1 : 0);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

int32_t history_stats(cook_pool* const* pools, int n, int32_t status, int64_t start_ms, int64_t end_ms, int64_t tid_lo,
                      int64_t tid_hi, int32_t seg_cap, const ISOut& o, cook_phase_stats* out_stats) {
  const char* who = "cook_state_history_stats";
  // ---- every check before any device work or output
  if (int32_t rc = check_handle_set(pools, n, who, true)) return rc;
  cook_pool* pool = pools[0];
  if (status != COOK_IS_SUCCESS && status != COOK_IS_FAILED) return set_err(pool, COOK_E_BADARG, "%s: an unknown status", who);
  if (end_ms <= start_ms) return set_err(pool, COOK_E_BADARG, "%s: end_ms <= start_ms", who);
  if (is_out_null(o)) return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (seg_cap < 0) return set_err(pool, COOK_E_BADARG, "%s: seg_cap < 0", who);
  // the handles with rows and their pool index
  std::vector<std::pair<const History*, int32_t>> hs;
  int Tmax = 0;
  for (int k = 0; k < n; k++) {
    const PoolState* s = static_cast<const PoolState*>(pools[k]->state);
    if (!s || !s->hist.on) return set_err(pool, COOK_E_BADARG, "%s: a handle whose history is off", who);
    if (s->hist.since > start_ms) return set_err(pool, COOK_E_BADARG, "%s: start_ms before a handle's horizon", who);
    if (!s->hist.tail) continue;
    hs.push_back({&s->hist, k});
    Tmax = std::max(Tmax, (int)s->hist.tail);
  }
  if (hs.empty()) return is_empty(o, out_stats);   // no row to read
  ReadCall r(pool);
  if (int32_t rc = r.open(who)) return rc;
  cudaStream_t st = r.st;
  const int H = (int)hs.size();
  const bool ok = status == COOK_IS_SUCCESS;
  auto sel = [&](int j, int base, const ISPipe& p) {
    return HSSel{hs[j].first->cols(), base, hs[j].second, ok, start_ms, end_ms, tid_lo, tid_hi,
                 p.s_user, p.s_reason, p.s_tid, p.s_pidx, p.s_pos, {p.met[0], p.met[1], p.met[2]}};
  };
  // ---- the selection's size per handle, so that every buffer after it is sized by the selection.  A staged handle
  // (Gather) counts on its own device, into its own scratch.
  Gather g(pool);
  int32_t* hcnt = nullptr;
  if (int32_t rc = r.scratch([&](Carve& c) { hcnt = c.take<int32_t>(H); })) return rc;
  CK(pool, cudaMemsetAsync(hcnt, 0, sizeof(int32_t) * H, st));
  int& nl = r.nl;
  int64_t& d2h = r.d2h;
  std::vector<int32_t> cnt(H);
  for (int j = 0; j < H; j++) {
    const int T = (int)hs[j].first->tail;
    cook_pool* h = pools[hs[j].second];
    if (!g.staged(h)) {
      hs_count_kernel<<<(T + 255) / 256, 256, 0, st>>>(sel(j, 0, ISPipe{}), T, hcnt + j);
      nl++;
      continue;
    }
    CK(pool, g.on(h, [&]() -> cudaError_t {
      int32_t* rc = nullptr;
      cudaError_t e = carve(state_of(h, false)->scratch, h->stream, nullptr, nullptr,
                            [&](Carve& c) { rc = c.take<int32_t>(1); });
      if (e == cudaSuccess) e = cudaMemsetAsync(rc, 0, sizeof(int32_t), h->stream);
      if (e != cudaSuccess) return e;
      hs_count_kernel<<<(T + 255) / 256, 256, 0, h->stream>>>(sel(j, 0, ISPipe{}), T, rc);
      nl++;
      return (e = cudaGetLastError()) == cudaSuccess ? download(&cnt[j], rc, 1, h->stream, &d2h) : e;
    }));
  }
  CK(pool, cudaGetLastError());
  int n_staged = 0;
  for (int j = 0; j < H; j++) n_staged += g.staged(pools[hs[j].second]) ? 1 : 0;
  if (!n_staged) {
    CK(pool, download(cnt.data(), hcnt, H, st, &d2h));
  } else {   // 4 bytes per handle either way
    for (int j = 0; j < H; j++) {
      cook_pool* h = pools[hs[j].second];
      if (g.staged(h)) CK(pool, cudaStreamSynchronize(h->stream));
      else CK(pool, download(&cnt[j], hcnt + j, 1, st, &d2h));
    }
  }
  CK(pool, cudaStreamSynchronize(st));
  int64_t S = 0;
  for (int32_t c : cnt) S += c;
  if (S * IS_LEVELS > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 entries", who);
  // ---- the selection and its metrics, then the pipeline
  ISPipe p;
  CK(pool, carve(r.S->scratch, st, nullptr, &r.h2d, [&](Carve& c) { p.take(c, (int)S, Tmax, true); }));
  CK(pool, p.clear(st));
  int base = 0;
  for (int j = 0; j < H && S; j++) {
    if (cnt[j])
      CK(pool, g.rows(pools[hs[j].second], sel(j, base, p), (int)hs[j].first->tail, cnt[j], p.blk, p.cnt + 5, &nl));
    base += cnt[j];
  }
  CK(pool, cudaGetLastError());
  return is_answer(r, p, (int)S, seg_cap, o, out_stats);
}

}  // namespace

extern "C" int32_t cook_state_instance_stats(cook_pool* const* pools, int32_t n_pools, int64_t now_ms, int32_t status,
                                             int64_t start_ms, int64_t end_ms, int64_t task_id_lo, int64_t task_id_hi,
                                             int32_t seg_cap, int32_t* out_kind, int32_t* out_user,
                                             int32_t* out_reason, int64_t* out_count, double* out_total,
                                             double* out_pct, int32_t* out_leader_user, double* out_leader_total,
                                             int32_t* out_n_seg, int32_t* out_n_leader, cook_phase_stats* out_stats) {
  return instance_stats(pools, n_pools, now_ms, status, start_ms, end_ms, task_id_lo, task_id_hi, seg_cap,
                        ISOut{out_kind, out_user, out_reason, out_count, out_total, out_pct, out_leader_user,
                              out_leader_total, out_n_seg, out_n_leader},
                        out_stats);
}

extern "C" int32_t cook_state_history_stats(cook_pool* const* pools, int32_t n_pools, int32_t status, int64_t start_ms,
                                            int64_t end_ms, int64_t task_id_lo, int64_t task_id_hi, int32_t seg_cap,
                                            int32_t* out_kind, int32_t* out_user, int32_t* out_reason,
                                            int64_t* out_count, double* out_total, double* out_pct,
                                            int32_t* out_leader_user, double* out_leader_total, int32_t* out_n_seg,
                                            int32_t* out_n_leader, cook_phase_stats* out_stats) {
  return history_stats(pools, n_pools, status, start_ms, end_ms, task_id_lo, task_id_hi, seg_cap,
                       ISOut{out_kind, out_user, out_reason, out_count, out_total, out_pct, out_leader_user,
                             out_leader_total, out_n_seg, out_n_leader},
                       out_stats);
}

// ---- audit: the read side (cook_state_digest, cook_state_export, cook_state_queue).  The digest is one pass per
// table: a thread hashes its slot's columns and short lists, a long list is read by the warp and absorbed by the
// owning lane; fingerprints and counts are reduced per warp with shuffles, per block in shared memory, then one
// atomic per block and word.  The export compacts the live (and selected) slots, sorts them by id, gathers the
// requested columns and rebuilds each list as CSR with the match's own csr_gather_kernel.  All of it lives in
// `scratch`: the queue arena and the match plan are only read.
namespace {

__device__ __forceinline__ uint64_t fp_mix(uint64_t z) {
  z ^= z >> 30; z *= 0xbf58476d1ce4e5b9ULL;
  z ^= z >> 27; z *= 0x94d049bb133111ebULL;
  return z ^ (z >> 31);
}
__device__ __forceinline__ uint64_t fp_absorb(uint64_t h, uint64_t w) { return fp_mix((h ^ w) + 0x9e3779b97f4a7c15ULL); }
__device__ __forceinline__ uint64_t fp_i32(int32_t x) { return (uint64_t)(int64_t)x; }

// what a digest downloads: the fingerprints of the pending rows, the running rows and the queue, then the recount
// (a maximum is kept as code + 1, so that zero is "none")
struct AuditDev {
  cook_fp fp[3];
  long long c[COOK_AUDIT_N];
};
constexpr int AUDIT_SUMS_P = 4 + F_N, AUDIT_SUMS_R = 4, AUDIT_MAXS = 3;
constexpr int AUDIT_SHORT = 8;        // a list up to this long is absorbed by its own thread
constexpr int AUDIT_SHARED_BUCKETS = 1024;   // up to this many buckets are reduced per block in shared memory

// the COOK_AUDIT_* index of a table pass's k-th sum and k-th maximum
__device__ __forceinline__ int audit_sum_index(bool pend, int k) {
  if (pend) return k == 0 ? (int)COOK_AUDIT_PENDING_ROWS : k < 4 ? COOK_AUDIT_ENTRIES + k - 1 : COOK_AUDIT_FLAGS + k - 4;
  return k == 0 ? (int)COOK_AUDIT_RUNNING_ROWS : k == 1 ? COOK_AUDIT_ENTRIES + L_RGROUP
         : k == 2 ? (int)COOK_AUDIT_COT_ROWS : (int)COOK_AUDIT_COT_ENTRIES;
}
__device__ __forceinline__ int audit_max_index(bool pend, int k) {   // user, group, then attribute column / hostname
  if (pend) return k == 0 ? COOK_AUDIT_MAX_USER_PENDING : k == 1 ? COOK_AUDIT_MAX_GROUP_PENDING : COOK_AUDIT_MAX_ATTR_COL;
  return k == 0 ? COOK_AUDIT_MAX_USER_RUNNING : k == 1 ? COOK_AUDIT_MAX_GROUP_RUNNING : COOK_AUDIT_MAX_HOSTNAME_RUNNING;
}

struct AuditArgs {
  void* const* col;            // the table's columns
  int n;                       // slots ever used
  const int32_t* v0[3];        // the arenas of the table's lists
  const int32_t* v1[3];        // non-null: (v0, v1) pairs
  AuditDev* out;
  cook_fp* bucket;             // [nb], null: no buckets
  unsigned nb;
  int sb;                      // nb when the block reduces the buckets in shared memory, else 0
};

__device__ __forceinline__ void fp_add(cook_fp* f, uint64_t sum, uint64_t xr, long long n) {
  atomicAdd(reinterpret_cast<unsigned long long*>(&f->sum), (unsigned long long)sum);
  atomicXor(reinterpret_cast<unsigned long long*>(&f->xr), (unsigned long long)xr);
  atomicAdd(reinterpret_cast<unsigned long long*>(&f->n), (unsigned long long)n);
}

// thread per slot of the pending (PEND) or running table
template <bool PEND>
__global__ void __launch_bounds__(256) audit_table_kernel(AuditArgs a) {
  extern __shared__ unsigned long long s_bkt[];   // [3 * a.sb]: sum, xor, n per bucket
  __shared__ unsigned long long s_fp[3];
  __shared__ int s_sum[AUDIT_SUMS_P], s_max[AUDIT_MAXS];
  constexpr int NS = PEND ? AUDIT_SUMS_P : AUDIT_SUMS_R, NL = PEND ? 3 : 1;
  if (threadIdx.x < 3) s_fp[threadIdx.x] = 0;
  if (threadIdx.x < AUDIT_SUMS_P) s_sum[threadIdx.x] = 0;
  if (threadIdx.x < AUDIT_MAXS) s_max[threadIdx.x] = 0;
  for (int b = threadIdx.x; b < 3 * a.sb; b += blockDim.x) s_bkt[b] = 0;
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  void* const* c = a.col;
  const bool live = i < a.n && static_cast<const uint8_t*>(c[PEND ? (int)P_LIVE : (int)R_LIVE])[i];
  uint64_t h = 0, id = 0;
  int sum[NS], mx[AUDIT_MAXS] = {0, 0, 0};
#pragma unroll
  for (int k = 0; k < NS; k++) sum[k] = 0;
  bool cot = false;
  if (live) {
    sum[0] = 1;
    const auto i32 = [&](int k) { return static_cast<const int32_t*>(c[k])[i]; };
    const auto i64 = [&](int k) { return static_cast<const long long*>(c[k])[i]; };   // doubles: the bits as stored
    const auto u8 = [&](int k) { return static_cast<const uint8_t*>(c[k])[i]; };
    if (PEND) {
      id = (uint64_t)i64(P_JID);
      h = fp_absorb(1, id);
      const int32_t user = i32(P_USER), ports = i32(P_PORTS), model = i32(P_GPU_MODEL), ckpt = i32(P_CKPT),
                    reserved = i32(P_RESERVED);
      const long long gpus = i64(P_GPUS), disk = i64(P_DISK_REQ), est = i64(P_EST);
      const uint8_t allowed = u8(P_ALLOWED), plugin = u8(P_PLUGIN);
      h = fp_absorb(h, fp_i32(user)); h = fp_absorb(h, fp_i32(i32(P_PRIO)));
      h = fp_absorb(h, (uint64_t)i64(P_CPUS)); h = fp_absorb(h, (uint64_t)i64(P_MEM)); h = fp_absorb(h, (uint64_t)gpus);
      h = fp_absorb(h, fp_i32(ports)); h = fp_absorb(h, allowed); h = fp_absorb(h, plugin);
      h = fp_absorb(h, fp_i32(model)); h = fp_absorb(h, (uint64_t)disk); h = fp_absorb(h, fp_i32(i32(P_DISK_TYPE)));
      h = fp_absorb(h, (uint64_t)est); h = fp_absorb(h, fp_i32(ckpt)); h = fp_absorb(h, fp_i32(reserved));
      mx[0] = user + 1;
      const bool f[F_N] = {__longlong_as_double(gpus) != 0.0, ports != 0, !allowed, !plugin, model != -1,
                           __longlong_as_double(disk) >= 0.0, est != -1, ckpt != -1, reserved != -1};
#pragma unroll
      for (int k = 0; k < F_N; k++) sum[4 + k] = f[k] ? 1 : 0;
    } else {
      id = (uint64_t)i64(R_TID);
      h = fp_absorb(2, id);
      const int32_t user = i32(R_USER), host = i32(R_HOST);
      h = fp_absorb(h, fp_i32(user)); h = fp_absorb(h, fp_i32(i32(R_PRIO))); h = fp_absorb(h, (uint64_t)i64(R_START));
      h = fp_absorb(h, (uint64_t)i64(R_JID)); h = fp_absorb(h, (uint64_t)i64(R_CPUS)); h = fp_absorb(h, (uint64_t)i64(R_MEM));
      h = fp_absorb(h, (uint64_t)i64(R_GPUS)); h = fp_absorb(h, fp_i32(host));
      mx[0] = user + 1; mx[2] = host + 1;
      cot = host != -1;
    }
  }
  // the lists: length, then the entries in order
#pragma unroll
  for (int l = 0; l < NL; l++) {
    const int oc = PEND ? (l == 0 ? (int)P_NOFF : l == 1 ? (int)P_AOFF : (int)P_GOFF) : (int)R_GOFF;
    const int len = live ? static_cast<const int32_t*>(c[oc + 1])[i] : 0;
    const int off = live ? static_cast<const int32_t*>(c[oc])[i] : 0;
    const int32_t* v0 = a.v0[l];
    const int32_t* v1 = a.v1[l];
    int m = 0;   // the largest first word + 1
    if (live) h = fp_absorb(h, fp_i32(len));
    if (len <= AUDIT_SHORT)
      for (int e = 0; e < len; e++) {
        const int32_t w = v0[off + e];
        h = fp_absorb(h, fp_i32(w));
        m = max(m, w + 1);
        if (v1) h = fp_absorb(h, fp_i32(v1[off + e]));
      }
    unsigned longer = __ballot_sync(FULL_MASK, len > AUDIT_SHORT);
    while (longer) {   // the warp reads the list, its owner absorbs it
      const int src = __ffs(longer) - 1;
      longer &= longer - 1;
      const int o = __shfl_sync(FULL_MASK, off, src), n = __shfl_sync(FULL_MASK, len, src);
      for (int base = 0; base < n; base += 32) {
        const int e = base + lane, cnt = min(32, n - base);
        const int32_t x0 = e < n ? v0[o + e] : 0, x1 = v1 && e < n ? v1[o + e] : 0;
        for (int k = 0; k < cnt; k++) {
          const int32_t w0 = __shfl_sync(FULL_MASK, x0, k), w1 = __shfl_sync(FULL_MASK, x1, k);
          if (lane == src) {
            h = fp_absorb(h, fp_i32(w0));
            m = max(m, w0 + 1);
            if (v1) h = fp_absorb(h, fp_i32(w1));
          }
        }
      }
    }
    sum[1 + l] = len;
    if (PEND && l == 1) mx[2] = m;
    if (PEND ? l == 2 : l == 0) mx[1] = m;
    if (!PEND && cot && len > 0) { sum[2] = 1; sum[3] = len; }
  }
  // ---- the warp's fingerprint and counts, then the block's, then one atomic per word
  uint64_t hs = live ? h : 0, hx = hs;
  for (int o = 16; o > 0; o >>= 1) {
    hs += __shfl_xor_sync(FULL_MASK, hs, o);
    hx ^= __shfl_xor_sync(FULL_MASK, hx, o);
  }
  const int nlive = __reduce_add_sync(FULL_MASK, sum[0]);
  if (lane == 0 && nlive) {
    atomicAdd(&s_fp[0], (unsigned long long)hs);
    atomicXor(&s_fp[1], (unsigned long long)hx);
    atomicAdd(&s_fp[2], (unsigned long long)nlive);
  }
#pragma unroll
  for (int k = 0; k < NS; k++) {
    const int v = __reduce_add_sync(FULL_MASK, sum[k]);
    if (lane == 0 && v) atomicAdd(&s_sum[k], v);
  }
#pragma unroll
  for (int k = 0; k < AUDIT_MAXS; k++) {
    const int v = __reduce_max_sync(FULL_MASK, mx[k]);
    if (lane == 0 && v) atomicMax(&s_max[k], v);
  }
  if (live && a.nb) {
    const unsigned b = (unsigned)fp_mix(id) & (a.nb - 1u);
    if (a.sb) {
      atomicAdd(&s_bkt[3 * b], (unsigned long long)h);
      atomicXor(&s_bkt[3 * b + 1], (unsigned long long)h);
      atomicAdd(&s_bkt[3 * b + 2], 1ULL);
    } else {
      fp_add(a.bucket + b, h, h, 1);
    }
  }
  __syncthreads();
  const int t = threadIdx.x;
  if (t == 0 && s_fp[2]) fp_add(&a.out->fp[PEND ? 0 : 1], s_fp[0], s_fp[1], (long long)s_fp[2]);
  if (t >= 32 && t < 32 + NS && s_sum[t - 32])
    atomicAdd(reinterpret_cast<unsigned long long*>(&a.out->c[audit_sum_index(PEND, t - 32)]), (unsigned long long)s_sum[t - 32]);
  if (t >= 64 && t < 64 + AUDIT_MAXS && s_max[t - 64])
    atomicMax(&a.out->c[audit_max_index(PEND, t - 64)], (long long)s_max[t - 64]);
  for (int b = t; b < a.sb; b += blockDim.x)
    if (s_bkt[3 * b + 2]) fp_add(a.bucket + b, s_bkt[3 * b], s_bkt[3 * b + 1], (long long)s_bkt[3 * b + 2]);
}

// the live queue's job ids, in queue order
struct QueueIds {
  QueueLive q; const int64_t* q_jid; int64_t* out;
  __device__ bool keep(int k) const { return q.keep(k); }
  __device__ void emit(int k, int d) const { out[d] = q_jid[k]; }
};
// position d < *n of the live queue: absorb(absorb(3, d), job id)
__global__ void audit_queue_kernel(const int64_t* ids, const int32_t* n, cook_fp* out) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  const bool on = d < *n;
  uint64_t hs = on ? fp_absorb(fp_absorb(3, (uint64_t)d), (uint64_t)ids[d]) : 0, hx = hs;
  for (int o = 16; o > 0; o >>= 1) {
    hs += __shfl_xor_sync(FULL_MASK, hs, o);
    hx ^= __shfl_xor_sync(FULL_MASK, hx, o);
  }
  const int c = __reduce_add_sync(FULL_MASK, on ? 1 : 0);
  if ((threadIdx.x & 31) == 0 && c) fp_add(out, hs, hx, c);
}

// the counts the host side keeps, in COOK_AUDIT_* order
void host_counts(const PoolState* S, int64_t* c) {
  c[COOK_AUDIT_PENDING_ROWS] = (int64_t)S->pend.slot_of.size();
  c[COOK_AUDIT_RUNNING_ROWS] = (int64_t)S->run.slot_of.size();
  for (int l = 0; l < L_N; l++) c[COOK_AUDIT_ENTRIES + l] = S->lists[l].live;
  for (int f = 0; f < F_N; f++) c[COOK_AUDIT_FLAGS + f] = S->nflag[f];
  c[COOK_AUDIT_RESERVED_ROWS] = (int64_t)S->reserved.size();
  c[COOK_AUDIT_COT_ROWS] = S->cot_rows;
  c[COOK_AUDIT_COT_ENTRIES] = S->cot_n;
  c[COOK_AUDIT_MAX_USER_PENDING] = count_max(S->users_p);
  c[COOK_AUDIT_MAX_USER_RUNNING] = count_max(S->users_r);
  c[COOK_AUDIT_MAX_GROUP_PENDING] = count_max(S->groups);
  c[COOK_AUDIT_MAX_GROUP_RUNNING] = count_max(S->groups_r);
  c[COOK_AUDIT_MAX_ATTR_COL] = count_max(S->attr_cols);
  c[COOK_AUDIT_MAX_HOSTNAME_RUNNING] = count_max(S->hosts_r);
}

bool buckets_ok(int32_t nb) { return nb >= 0 && nb <= 65536 && (nb & (nb - 1)) == 0; }

int32_t digest(cook_pool* pool, PoolState* S, int nb, cook_state_digest_out* out, cook_fp* out_pb, cook_fp* out_rb) {
  const char* who = "cook_state_digest";
  if (!out) return set_err(pool, COOK_E_BADARG, "%s: null out", who);
  if (!buckets_ok(nb)) return set_err(pool, COOK_E_BADARG, "%s: n_buckets is not 0 or a power of two up to 65536", who);
  if (nb ? (!out_pb || !out_rb) : (out_pb || out_rb))
    return set_err(pool, COOK_E_BADARG, "%s: the bucket outputs go with n_buckets > 0", who);
  if (!S || S->pend.slot_of.size() + S->run.slot_of.size() == 0) {   // nothing live
    memset(out, 0, sizeof(*out));
    out->consistent = 1;
    out->first_mismatch = -1;
    if (nb) { memset(out_pb, 0, sizeof(cook_fp) * (size_t)nb); memset(out_rb, 0, sizeof(cook_fp) * (size_t)nb); }
    pool->phase[COOK_PHASE_AUDIT] = cook_phase_stats{};
    return COOK_OK;
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  const int nq = S->ranked ? S->n_q : 0;
  AuditDev* dev = nullptr;
  cook_fp* bkt = nullptr;
  int64_t* ids = nullptr;
  int32_t* blk = nullptr;
  int64_t h2d = 0, d2h = 0;
  CK(pool, carve(S->scratch, st, pool->ev[20], &h2d, [&](Carve& c) {
    dev = c.take<AuditDev>(1);
    if (nb) bkt = c.take<cook_fp>(2 * (size_t)nb);
    if (nq) { ids = c.take<int64_t>(nq); blk = c.take<int32_t>((size_t)nq / CP_BLOCK + 2); }
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  CK(pool, cudaMemsetAsync(dev, 0, sizeof(AuditDev), st));
  if (nb) CK(pool, cudaMemsetAsync(bkt, 0, sizeof(cook_fp) * 2 * (size_t)nb, st));
  int nl = 0;
  AuditArgs a = {};
  a.out = dev; a.nb = (unsigned)nb; a.sb = nb <= AUDIT_SHARED_BUCKETS ? nb : 0;
  const size_t shm = sizeof(unsigned long long) * 3 * (size_t)a.sb;
  if (S->pend.hw) {
    a.col = S->pend.d_col; a.n = S->pend.hw; a.bucket = bkt;
    for (int l = 0; l < 3; l++) { a.v0[l] = S->lists[l].at(0); a.v1[l] = S->lists[l].at(1); }
    audit_table_kernel<true><<<(a.n + 255) / 256, 256, shm, st>>>(a);
    nl++;
  }
  if (S->run.hw) {
    a.col = S->run.d_col; a.n = S->run.hw; a.bucket = bkt ? bkt + nb : nullptr;
    a.v0[0] = S->lists[L_RGROUP].at(0); a.v1[0] = nullptr;
    audit_table_kernel<false><<<(a.n + 255) / 256, 256, shm, st>>>(a);
    nl++;
  }
  if (nq) {
    const QueueLive ql{S->q_slot, S->q_gen, S->pend.at<uint8_t>(P_LIVE), S->pend.at<uint32_t>(P_GEN), nullptr};
    compact(QueueIds{ql, S->q_jid, ids}, nq, nullptr, blk, S->counters + 5, nq, st, &nl);
    audit_queue_kernel<<<(nq + 255) / 256, 256, 0, st>>>(ids, S->counters + 5, &dev->fp[2]);
    nl++;
  }
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  AuditDev got;
  CK(pool, download(&got, dev, 1, st, &d2h));
  if (nb) {
    CK(pool, download(out_pb, bkt, (size_t)nb, st, &d2h));
    CK(pool, download(out_rb, bkt + nb, (size_t)nb, st, &d2h));
  }
  CK(pool, cudaEventRecord(pool->ev[23], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_AUDIT, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[23], h2d, d2h, nl);
  // ---- the recount against the host side
  int64_t hostc[COOK_AUDIT_N], devc[COOK_AUDIT_N];
  host_counts(S, hostc);
  for (int k = 0; k < COOK_AUDIT_N; k++) devc[k] = got.c[k] - (k >= COOK_AUDIT_MAX_USER_PENDING ? 1 : 0);
  devc[COOK_AUDIT_RESERVED_ROWS] = devc[COOK_AUDIT_FLAGS + F_RESERVED];
  out->pending = got.fp[0]; out->running = got.fp[1]; out->queue = got.fp[2];
  for (int l = 0; l < L_N; l++) out->entries[l] = devc[COOK_AUDIT_ENTRIES + l];
  cook_state_counts_compare(hostc, devc, &out->first_mismatch);
  out->consistent = out->first_mismatch < 0 ? 1 : 0;
  return COOK_OK;
}

// ---- export
// the live slots of a table whose id's bucket is selected (mask null: all), with their ids
struct SelectedRows {
  const uint8_t* live; const int64_t* id; const uint8_t* mask; unsigned nb; int32_t* sel; int64_t* key;
  __device__ bool keep(int i) const { return live[i] && (!mask || mask[(unsigned)fp_mix((uint64_t)id[i]) & (nb - 1u)]); }
  __device__ void emit(int i, int d) const { sel[d] = i; key[d] = id[i]; }
};
struct ExportCols { char* dst[MAXC]; int sz[MAXC]; int nc; };
// row p of the export is slot sel[ord[p]]: the requested data columns (a null dst is skipped)
__global__ void export_rows_kernel(void* const* col, const int32_t* sel, const int32_t* ord, int n, int32_t* rowslot,
                                   ExportCols c) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int s = sel[ord[p]];
  rowslot[p] = s;
#pragma unroll
  for (int k = 0; k < MAXC; k++) {
    if (k >= c.nc) break;
    if (!c.dst[k]) continue;
    if (c.sz[k] == 1) reinterpret_cast<uint8_t*>(c.dst[k])[p] = static_cast<const uint8_t*>(col[k])[s];
    else if (c.sz[k] == 4) reinterpret_cast<int32_t*>(c.dst[k])[p] = static_cast<const int32_t*>(col[k])[s];
    else reinterpret_cast<long long*>(c.dst[k])[p] = static_cast<const long long*>(col[k])[s];
  }
}
__global__ void list_total_kernel(OrderScan<int, 1> os, int n, int32_t* out) { *out = os.at(0, n - 1); }

int32_t export_rows(cook_pool* pool, PoolState* S, int nb, const uint8_t* mask, const cook_state_sizes* cap,
                    const cook_state_rows* out, cook_state_sizes* out_n) {
  const char* who = "cook_state_export";
  const bool query = !out;
  if (!out_n || (!query && !cap)) return set_err(pool, COOK_E_BADARG, "%s: null out_n or cap", who);
  if (!buckets_ok(nb)) return set_err(pool, COOK_E_BADARG, "%s: n_buckets is not 0 or a power of two up to 65536", who);
  if (mask && !nb) return set_err(pool, COOK_E_BADARG, "%s: a mask without buckets", who);
  // ---- what goes where: table t's data column k to dst[t][k], list l (of table l == L_RGROUP) to loff / lv
  void* dst[2][MAXC] = {};
  int32_t* loff[L_N] = {};
  int32_t* lv[L_N][2] = {};
  if (!query) {
    const cook_jobs_rows& p = out->pending;
    const cook_tasks_rows& r = out->running;
    void* pd[P_NDATA] = {p.user, out->pending_priority, out->pending_job_id, p.cpus, p.mem, p.gpus, p.ports, p.allowed,
                         p.plugin_accept, p.gpu_model, p.disk_request, p.disk_type, p.est_end_ms, p.ckpt_location,
                         p.reserved_host};
    void* rd[R_NDATA] = {r.user, r.priority, r.start_time, r.task_id, r.job_id, r.cpus, r.mem, r.gpus,
                         out->running_hostname_id};
    std::copy(pd, pd + P_NDATA, dst[0]);
    std::copy(rd, rd + R_NDATA, dst[1]);
    loff[L_NOVEL] = p.novel_off; lv[L_NOVEL][0] = p.novel_host;
    loff[L_ATTR] = p.attr_off; lv[L_ATTR][0] = p.attr_col; lv[L_ATTR][1] = p.attr_val;
    loff[L_GROUP] = p.group_off; lv[L_GROUP][0] = p.group_idx;
    loff[L_RGROUP] = out->running_group_off; lv[L_RGROUP][0] = out->running_group_idx;
    for (int l = 0; l < L_N; l++)
      if (loff[l] && (!lv[l][0] || (l == L_ATTR && !lv[l][1])))
        return set_err(pool, COOK_E_BADARG, "%s: a list's offsets without its values", who);
  }
  // ---- the sizes the host side knows: exact without a mask, an upper bound with one
  int64_t N[2] = {0, 0}, E[L_N] = {};
  if (S) {
    N[0] = (int64_t)S->pend.slot_of.size(); N[1] = (int64_t)S->run.slot_of.size();
    for (int l = 0; l < L_N; l++) E[l] = S->lists[l].live;
  }
  const auto fits = [&](const int64_t* rows, const int64_t* entries) {
    if (rows[0] > cap->pending || rows[1] > cap->running) return false;
    for (int l = 0; l < L_N; l++) if (loff[l] && entries[l] > cap->entries[l]) return false;
    return true;
  };
  if (!query && !mask && !fits(N, E)) return set_err(pool, COOK_E_BADARG, "%s: a capacity below the required size", who);
  if (N[0] + N[1] == 0 || (query && !mask)) {   // no device work
    if (N[0] + N[1] == 0) {
      for (int l = 0; l < L_N; l++) if (loff[l]) loff[l][0] = 0;
      memset(out_n, 0, sizeof(*out_n));
    } else {
      out_n->pending = (int32_t)N[0]; out_n->running = (int32_t)N[1];
      for (int l = 0; l < L_N; l++) out_n->entries[l] = (int32_t)E[l];
    }
    pool->phase[COOK_PHASE_AUDIT] = cook_phase_stats{};
    return COOK_OK;
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  Table* tbl[2] = {&S->pend, &S->run};
  const int live_col[2] = {P_LIVE, R_LIVE}, id_col[2] = {P_JID, R_TID}, ndata[2] = {P_NDATA, R_NDATA};
  const int* sz[2] = {P_SZ, R_SZ};
  const int table_of[L_N] = {0, 0, 0, 1}, off_col[L_N] = {P_NOFF, P_AOFF, P_GOFF, R_GOFF};
  int32_t *sel[2] = {}, *ord[2] = {}, *tmp[2] = {}, *rowslot[2] = {}, *blk = nullptr, *d_cnt = nullptr;
  int64_t* key[2] = {};
  ExportCols cols[2] = {};
  int32_t* d_off[L_N] = {};
  int32_t* d_v[L_N][2] = {};
  const uint8_t* d_mask = nullptr;
  OrderScan<int, 1> os;
  int64_t h2d = 0, d2h = 0;
  CK(pool, carve(S->scratch, st, pool->ev[20], &h2d, [&](Carve& c) {
    for (int t = 0; t < 2; t++) {
      sel[t] = c.take<int32_t>(N[t]); key[t] = c.take<int64_t>(N[t]);
      if (query) continue;
      ord[t] = c.take<int32_t>(N[t]); tmp[t] = c.take<int32_t>(N[t]); rowslot[t] = c.take<int32_t>(N[t]);
      cols[t].nc = ndata[t];
      for (int k = 0; k < ndata[t]; k++) {
        cols[t].sz[k] = sz[t][k];
        cols[t].dst[k] = dst[t][k] ? c.take<char>((size_t)N[t] * sz[t][k]) : nullptr;
      }
    }
    const int64_t nmax = std::max(N[0], N[1]);
    blk = c.take<int32_t>((size_t)std::max(S->pend.hw, S->run.hw) / CP_BLOCK + 2);
    os.part[0] = c.take<int32_t>(nmax);
    os.tile[0] = c.take<int32_t>((nmax + OS_TILE - 1) / OS_TILE + 1);
    d_cnt = c.take<int32_t>(2 + L_N);
    for (int l = 0; l < L_N; l++) {
      if (!loff[l]) continue;
      d_off[l] = c.take<int32_t>(N[table_of[l]] + 1);
      for (int i = 0; i < S->lists[l].v.n; i++) d_v[l][i] = c.take<int32_t>(std::max<int64_t>(E[l], 1));
    }
    if (mask) d_mask = c.up(mask, nb);
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int nl = 0;
  CK(pool, cudaMemsetAsync(d_cnt, 0, sizeof(int32_t) * (2 + L_N), st));
  for (int t = 0; t < 2; t++)
    if (N[t])
      compact(SelectedRows{tbl[t]->at<uint8_t>(live_col[t]), tbl[t]->at<int64_t>(id_col[t]), d_mask, (unsigned)nb, sel[t],
                           key[t]}, tbl[t]->hw, nullptr, blk, d_cnt + t, (int)N[t], st, &nl);
  CK(pool, cudaGetLastError());
  int32_t n[2] = {(int32_t)N[0], (int32_t)N[1]};
  if (mask) {   // how many rows the mask selects: the sort and the scans are sized by it
    CK(pool, download(n, d_cnt, 2, st, &d2h));
    CK(pool, cudaStreamSynchronize(st));
  }
  for (int t = 0; t < 2; t++) {
    if (query || !n[t]) continue;
    CK(pool, csort::sort_indices(ord[t], tmp[t], n[t], LessKeyTid{nullptr, key[t]}, st, &nl));
    export_rows_kernel<<<(n[t] + 255) / 256, 256, 0, st>>>(tbl[t]->d_col, sel[t], ord[t], n[t], rowslot[t], cols[t]);
    nl++;
  }
  for (int l = 0; l < L_N; l++) {
    const int t = table_of[l];
    if (!n[t]) {
      if (d_off[l]) CK(pool, cudaMemsetAsync(d_off[l], 0, sizeof(int32_t), st));
      continue;
    }
    const int32_t* rs = query ? sel[t] : rowslot[t];
    const int32_t* len = tbl[t]->at<int32_t>(off_col[l] + 1);
    order_scan(os, RowLen{rs, len}, n[t], S->gf0, st, &nl);
    list_total_kernel<<<1, 1, 0, st>>>(os, n[t], d_cnt + 2 + l);
    nl++;
    if (!d_off[l]) continue;
    csr_gather_kernel<<<(n[t] + 7) / 8, 256, 0, st>>>(os, rs, n[t], tbl[t]->at<int32_t>(off_col[l]), len, S->lists[l].at(0),
                                                       S->lists[l].at(1), d_off[l], d_v[l][0], d_v[l][1]);
    nl++;
  }
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  int32_t cnt[2 + L_N];
  CK(pool, download(cnt, d_cnt, 2 + L_N, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  const int64_t rows[2] = {cnt[0], cnt[1]};
  int64_t entries[L_N];
  for (int l = 0; l < L_N; l++) entries[l] = cnt[2 + l];
  if (!query) {
    if (!fits(rows, entries)) return set_err(pool, COOK_E_BADARG, "%s: a capacity below the required size", who);
    for (int t = 0; t < 2; t++)
      for (int k = 0; k < ndata[t]; k++)
        if (dst[t][k] && rows[t])
          CK(pool, download(static_cast<char*>(dst[t][k]), cols[t].dst[k], (size_t)rows[t] * sz[t][k], st, &d2h));
    for (int l = 0; l < L_N; l++) {
      if (!loff[l]) continue;
      CK(pool, download(loff[l], d_off[l], (size_t)rows[table_of[l]] + 1, st, &d2h));
      for (int i = 0; i < S->lists[l].v.n; i++)
        if (entries[l]) CK(pool, download(lv[l][i], d_v[l][i], (size_t)entries[l], st, &d2h));
    }
  }
  CK(pool, cudaEventRecord(pool->ev[23], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_AUDIT, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[23], h2d, d2h, nl);
  out_n->pending = cnt[0]; out_n->running = cnt[1];
  for (int l = 0; l < L_N; l++) out_n->entries[l] = cnt[2 + l];
  return COOK_OK;
}

int32_t live_queue(cook_pool* pool, PoolState* S, int cap, int64_t* out_job_id, int32_t* out_n) {
  const char* who = "cook_state_queue";
  if (!out_n) return set_err(pool, COOK_E_BADARG, "%s: null out_n", who);
  if (!S || !S->ranked) return set_err(pool, COOK_E_BADARG, "%s: no cook_state_rank on this handle yet", who);
  const int nq = S->n_q;
  if (nq == 0) {
    *out_n = 0;
    pool->phase[COOK_PHASE_AUDIT] = cook_phase_stats{};
    return COOK_OK;
  }
  CK(pool, cudaSetDevice(pool->device));
  cudaStream_t st = pool->stream;
  int64_t* ids = nullptr;
  int32_t* blk = nullptr;
  int64_t h2d = 0, d2h = 0;
  CK(pool, carve(S->scratch, st, pool->ev[20], &h2d, [&](Carve& c) {
    ids = c.take<int64_t>(nq);
    blk = c.take<int32_t>((size_t)nq / CP_BLOCK + 2);
  }));
  CK(pool, cudaEventRecord(pool->ev[21], st));
  int nl = 0;
  const QueueLive ql{S->q_slot, S->q_gen, S->pend.at<uint8_t>(P_LIVE), S->pend.at<uint32_t>(P_GEN), nullptr};
  compact(QueueIds{ql, S->q_jid, ids}, nq, nullptr, blk, S->counters + 5, nq, st, &nl);
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  int32_t n = 0;
  CK(pool, download(&n, S->counters + 5, 1, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  if (out_job_id) {
    if (cap < n) return set_err(pool, COOK_E_BADARG, "%s: cap < the live queue entries", who);
    if (n > 0) CK(pool, download(out_job_id, ids, (size_t)n, st, &d2h));
  }
  CK(pool, cudaEventRecord(pool->ev[23], st));
  CK(pool, cudaStreamSynchronize(st));
  record_phase(pool, COOK_PHASE_AUDIT, pool->ev[20], pool->ev[21], pool->ev[22], pool->ev[23], h2d, d2h, nl);
  *out_n = n;
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_counts_compare(const int64_t* host, const int64_t* device, int32_t* out_first) {
  if (!host || !device || !out_first) return COOK_E_BADARG;
  *out_first = -1;
  for (int k = 0; k < COOK_AUDIT_N; k++)
    if (host[k] != device[k]) { *out_first = k; break; }
  return COOK_OK;
}

extern "C" int32_t cook_state_digest(cook_pool* pool, int32_t n_buckets, cook_state_digest_out* out,
                                     cook_fp* out_pending_bucket, cook_fp* out_running_bucket) {
  if (!pool) return COOK_E_BADARG;
  return digest(pool, static_cast<PoolState*>(pool->state), n_buckets, out, out_pending_bucket, out_running_bucket);
}

extern "C" int32_t cook_state_export(cook_pool* pool, int32_t n_buckets, const uint8_t* bucket_mask,
                                     const cook_state_sizes* cap, const cook_state_rows* out, cook_state_sizes* out_n) {
  if (!pool) return COOK_E_BADARG;
  return export_rows(pool, static_cast<PoolState*>(pool->state), n_buckets, bucket_mask, cap, out, out_n);
}

extern "C" int32_t cook_state_queue(cook_pool* pool, int32_t cap, int64_t* out_job_id, int32_t* out_n) {
  if (!pool) return COOK_E_BADARG;
  return live_queue(pool, static_cast<PoolState*>(pool->state), cap, out_job_id, out_n);
}

// ---- match-cycle metrics (handle-match-cycle-metrics scheduler.clj:1210-1280 and the unmatched tracking :1399-1486)
// over the last resident match round: the considerable rows gathered in take order with their job facts; per user
// integer counts; cpus and mem folded in take order and sorted by (value, position) for the nearest-rank percentiles,
// the last position of each order being the last maximal row; the keyed totals' entries sorted by (kind, code,
// position) and folded per key; the unmatched cycles looked up by job id in the last counted round's sorted pairs.
namespace {

enum { MM_GPUS = 0, MM_DISK_REQ = 1, MM_DISK_LIM = 2, MM_KINDS = 3 };
constexpr int MM_FIRST = COOK_MM_FIRST_N;
// the result block the device writes and the call downloads in one copy, then spreads over the caller's arrays
struct MMRow {
  int64_t job_id; int32_t position, user; double cpus, mem, gpus; int32_t ports, facts, gpu_model, disk_type;
  double disk_request, disk_limit;
};
struct MMOut {
  int32_t n_considerable, n_matched; int64_t head_job_id; int32_t head_matched, n_uris, uris_position, n_keys;
  double total_cpus, total_mem, pct_cpus[3], pct_mem[3];
  MMRow row[COOK_MM_ROWS];
  int32_t n_too_long, n_first; int64_t first_job_id[MM_FIRST]; int32_t first_cycles[MM_FIRST];
};
static_assert(sizeof(MMOut) == 440, "the result block's size is part of the transfer formula");
// cnt: [0] matched after the drops, [1] rows with uris, [2] 1 + the position of one of them, [3] keys, [4] rows unmatched
// too long, [5] key entries, [6] unmatched rows, [7] a dropped position that holds no assignment
enum { MMC_MATCHED, MMC_URIS, MMC_URI_POS, MMC_KEYS, MMC_TOO_LONG, MMC_ENTRIES, MMC_UNMATCHED, MMC_BAD, MMC_N };

struct MMCols {   // row k: the k-th considerable job
  int32_t* slot; int32_t* user; int64_t* jid; double* cpus; double* mem; double* gpus; int32_t* ports; uint8_t* jf;
  int32_t* gmodel; int32_t* dtype; double* dreq; double* dlim; uint8_t* matched; int32_t* cyc;
};

__global__ void mm_gather_kernel(void* const* col, const int32_t* rslot, const int32_t* cons, const int32_t* assign,
                                 int N, MMCols r) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= N) return;
  const int s = rslot[cons[k]];
  const uint8_t jf = static_cast<const uint8_t*>(col[P_JF])[s];
  r.slot[k] = s;
  r.user[k] = static_cast<const int32_t*>(col[P_USER])[s];
  r.jid[k] = static_cast<const int64_t*>(col[P_JID])[s];
  r.cpus[k] = static_cast<const double*>(col[P_CPUS])[s];
  r.mem[k] = static_cast<const double*>(col[P_MEM])[s];
  r.gpus[k] = static_cast<const double*>(col[P_GPUS])[s];
  r.ports[k] = static_cast<const int32_t*>(col[P_PORTS])[s];
  r.jf[k] = jf;
  r.gmodel[k] = jf & COOK_JF_GPUS ? static_cast<const int32_t*>(col[P_JF_GPU])[s] : -1;
  r.dtype[k] = jf & COOK_JF_DISK ? static_cast<const int32_t*>(col[P_JF_DTYPE])[s] : -1;
  r.dreq[k] = jf & COOK_JF_DISK_REQUEST ? static_cast<const double*>(col[P_JF_DREQ])[s] : 0.0;
  r.dlim[k] = jf & COOK_JF_DISK_LIMIT ? static_cast<const double*>(col[P_JF_DLIM])[s] : 0.0;
  r.matched[k] = assign[k] >= 0;
}

// the launch-rate filter's drops: their jobs count as unmatched; one that holds no assignment sets the flag
__global__ void mm_drop_kernel(const int32_t* dropped, int D, const int32_t* assign, uint8_t* matched, int32_t* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  const int k = dropped[i];
  if (assign[k] < 0) atomicOr(bad, 1);
  matched[k] = 0;
}

// per row: its user's counts (a code >= U is skipped: the round is then refused), the matched and uris counts, and its
// unmatched cycles: 0 when matched, else 1 + its cycles in the last counted round (u_jid ascending, u_n pairs)
__global__ void mm_count_kernel(MMCols r, int N, int U, const int64_t* u_jid, const int32_t* u_cyc, int u_n,
                                int32_t* ucons, int32_t* umat, int32_t* cnt) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned act = __ballot_sync(FULL_MASK, k < N);
  if (k >= N) return;
  const int lane = threadIdx.x & 31;
  const int u = r.user[k];
  const bool m = r.matched[k];
  const unsigned same = __match_any_sync(act, u);
  const unsigned same_m = same & __ballot_sync(act, m);
  if (u < U) {
    if (lane == __ffs(same) - 1) atomicAdd(&ucons[u], __popc(same));
    if (m && lane == __ffs(same_m) - 1) atomicAdd(&umat[u], __popc(same_m));
  }
  const unsigned mm = __ballot_sync(act, m);
  if (lane == __ffs(act) - 1 && mm) atomicAdd(&cnt[MMC_MATCHED], __popc(mm));
  if (r.jf[k] & COOK_JF_URIS) {
    atomicAdd(&cnt[MMC_URIS], 1);
    atomicMax(&cnt[MMC_URI_POS], k + 1);
  }
  int c = 0;
  if (!m) {
    const int64_t j = r.jid[k];
    int lo = 0, hi = u_n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (u_jid[mid] < j) lo = mid + 1;
      else hi = mid;
    }
    c = 1 + (lo < u_n && u_jid[lo] == j ? u_cyc[lo] : 0);
  }
  r.cyc[k] = c;
}

// entry e = kind * N + k: row k's key of that kind, when the row carries it
struct MMKey {
  const uint8_t* jf; const int32_t* gmodel; const int32_t* dtype; const double* dreq; const double* dlim; int N;
  __device__ int kind(int e) const { return e / N; }
  __device__ int row(int e) const { return e - (e / N) * N; }
  __device__ int code(int e) const { return kind(e) == MM_GPUS ? gmodel[row(e)] : dtype[row(e)]; }
  __device__ double value(int e, const double* gpus) const {
    const int t = kind(e), k = row(e);
    return t == MM_GPUS ? gpus[k] : t == MM_DISK_REQ ? dreq[k] : dlim[k];
  }
  __device__ bool present(int e) const {
    const int t = kind(e);
    return jf[row(e)] & (t == MM_GPUS ? COOK_JF_GPUS : t == MM_DISK_REQ ? COOK_JF_DISK_REQUEST : COOK_JF_DISK_LIMIT);
  }
  __device__ bool same(int a, int b) const { return kind(a) == kind(b) && code(a) == code(b); }
};
struct MMEntries {
  MMKey key; int32_t* ent;
  __device__ bool keep(int e) const { return key.present(e); }
  __device__ void emit(int e, int d) const { ent[d] = e; }
};
struct LessKindCodePos {   // (kind, code, position): each key's entries in take order
  MMKey key; const int32_t* ent;
  __device__ bool operator()(int32_t a, int32_t b) const {
    const int ea = ent[a], eb = ent[b];
    const int ka = key.kind(ea), kb = key.kind(eb);
    if (ka != kb) return ka < kb;
    const int ca = key.code(ea), cb = key.code(eb);
    if (ca != cb) return ca < cb;
    return key.row(ea) < key.row(eb);
  }
};
struct MMSegEnds {   // end[d] = one past key d's last position in the sorted entries
  MMKey key; const int32_t* ent; const int32_t* ord; const int32_t* n; int32_t* end;
  __device__ bool keep(int p) const { return p == *n - 1 || !key.same(ent[ord[p]], ent[ord[p + 1]]); }
  __device__ void emit(int p, int d) const { end[d] = p + 1; }
};
// a key's left fold in take order (fold_segments without the order-wide scan: on the grid or by the serial chain)
struct MMKeyLoad {
  MMKey key; const double* gpus; const int32_t* ent; const int32_t* ord;
  __device__ void operator()(int p, double (&x)[1]) const { x[0] = key.value(ent[ord[p]], gpus); }
};
struct MMKeyOut {
  MMKey key; const int32_t* ent; const int32_t* ord; int32_t* o_kind; int32_t* o_code; double* o_total;
  __device__ void operator()(int g, int s, int, const double (&acc)[1]) const {
    const int e0 = ent[ord[s]];
    o_kind[g] = key.kind(e0);
    o_code[g] = key.code(e0);
    o_total[g] = acc[0];
  }
};

struct LessValuePos {   // (value, position): no amount is NaN, and -0.0 and 0.0 compare equal as in Clojure's compare
  const double* v;
  __device__ bool operator()(int32_t a, int32_t b) const { return v[a] != v[b] ? v[a] < v[b] : a < b; }
};
struct MMTooLong {   // rows unmatched for more than thr cycles, in take order: the first MM_FIRST recorded
  const int32_t* cyc; const int64_t* jid; int thr; int64_t* f_jid; int32_t* f_cyc;
  __device__ bool keep(int k) const { return cyc[k] > thr; }
  __device__ void emit(int k, int d) const {
    if (d < MM_FIRST) { f_jid[d] = jid[k]; f_cyc[d] = cyc[k]; }
  }
};
struct MMUnmatched {   // the unmatched rows' (job id, cycles), in take order
  const int32_t* cyc; const int64_t* jid; int64_t* o_jid; int32_t* o_cyc;
  __device__ bool keep(int k) const { return cyc[k] > 0; }
  __device__ void emit(int k, int d) const { o_jid[d] = jid[k]; o_cyc[d] = cyc[k]; }
};
struct LessJid {
  const int64_t* jid;
  __device__ bool operator()(int32_t a, int32_t b) const { return jid[a] < jid[b]; }
};
__global__ void mm_map_kernel(const int32_t* ord, int n, const int64_t* jid, const int32_t* cyc, int64_t* o_jid,
                              int32_t* o_cyc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  o_jid[i] = jid[ord[i]];
  o_cyc[i] = cyc[ord[i]];
}

__device__ void mm_row(const MMCols& r, int k, MMRow* o) {
  o->job_id = r.jid[k]; o->position = k; o->user = r.user[k];
  o->cpus = r.cpus[k]; o->mem = r.mem[k]; o->gpus = r.gpus[k]; o->ports = r.ports[k]; o->facts = r.jf[k];
  o->gpu_model = r.gmodel[k]; o->disk_type = r.dtype[k]; o->disk_request = r.dreq[k]; o->disk_limit = r.dlim[k];
}
// one warp: the cpus and mem totals (left folds in take order), then lane 0 writes the result block
__global__ void __launch_bounds__(32) mm_finish_kernel(MMCols r, int N, const GridFlag* gf, const int32_t* ord_c,
                                                       const int32_t* ord_m, const int32_t* cnt, const int64_t* f_jid,
                                                       const int32_t* f_cyc, MMOut* o) {
  __shared__ double stage[1][2][32];
  double acc[2] = {0.0, 0.0};
  warp_fold_sum<2, 4>(acc, N, grid_exact(gf, N), [&](int k, double (&x)[2]) {
    x[0] = r.cpus[k]; x[1] = r.mem[k];
    return true;
  }, stage[0]);
  if (threadIdx.x) return;
  o->n_considerable = N;
  o->n_matched = cnt[MMC_MATCHED];
  o->head_job_id = r.jid[0];
  o->head_matched = r.matched[0];
  o->n_uris = cnt[MMC_URIS];
  o->uris_position = cnt[MMC_URIS] == 1 ? cnt[MMC_URI_POS] - 1 : -1;
  o->n_keys = cnt[MMC_KEYS];
  o->total_cpus = acc[0];
  o->total_mem = acc[1];
  const int pcts[3] = {50, 95, 100};
  for (int j = 0; j < 3; j++) {
    const int p = (int)(((int64_t)pcts[j] * N + 99) / 100) - 1;
    o->pct_cpus[j] = r.cpus[ord_c[p]];
    o->pct_mem[j] = r.mem[ord_m[p]];
  }
  mm_row(r, 0, &o->row[COOK_MM_HEAD]);
  mm_row(r, ord_c[N - 1], &o->row[COOK_MM_LARGEST_CPUS]);
  mm_row(r, ord_m[N - 1], &o->row[COOK_MM_LARGEST_MEM]);
  o->n_too_long = cnt[MMC_TOO_LONG];
  o->n_first = min(cnt[MMC_TOO_LONG], MM_FIRST);
  for (int i = 0; i < MM_FIRST; i++) {
    o->first_job_id[i] = i < o->n_first ? f_jid[i] : -1;
    o->first_cycles[i] = i < o->n_first ? f_cyc[i] : 0;
  }
}

// capacity for n pairs in both halves of the counters, the current half's u_n pairs kept
int32_t mm_counters_room(cook_pool* pool, MetricsRound& R, int64_t n, cudaStream_t st) {
  cudaError_t e = R.u[1 - R.cur].grow(n, 0, st);
  if (e == cudaSuccess) e = R.u[R.cur].grow(n, R.u_n, st);
  if (e != cudaSuccess) return set_err(pool, COOK_E_OOM, "cook_state_match_metrics: out of device memory");
  return COOK_OK;
}

int32_t job_facts(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* job_id, const uint8_t* flags,
                  const int32_t* gpu_model, const double* disk_request, const double* disk_limit,
                  const int32_t* disk_type) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && !job_id) return set_err(pool, COOK_E_BADARG, "%s: null job_id", who);
  const int all = COOK_JF_GPUS | COOK_JF_DISK | COOK_JF_DISK_REQUEST | COOK_JF_DISK_LIMIT | COOK_JF_URIS;
  for (int i = 0; flags && i < n; i++) {
    if (flags[i] & ~all) return set_err(pool, COOK_E_BADARG, "%s: an unknown flag bit", who);
    if ((flags[i] & (COOK_JF_DISK_REQUEST | COOK_JF_DISK_LIMIT)) && !(flags[i] & COOK_JF_DISK))
      return set_err(pool, COOK_E_BADARG, "%s: a disk request or limit without the disk flag", who);
  }
  if (!idx_in_range(gpu_model, n, -1, INT32_MAX) || !idx_in_range(disk_type, n, -1, INT32_MAX))
    return set_err(pool, COOK_E_BADARG, "%s: a gpu model or disk type code below -1", who);
  for (const double* v : {disk_request, disk_limit})
    for (int i = 0; v && i < n; i++)
      if (std::isnan(v[i])) return set_err(pool, COOK_E_BADARG, "%s: a NaN disk amount", who);
  std::vector<int32_t> slot;
  if (int32_t rc = live_slots(pool, who, S->pend, "job", n, job_id, &slot)) return rc;
  // ---- host side: the rows' bits, for the count of rows with a keyed resource
  for (int i = 0; flags && i < n; i++) {
    PendingInfo& pi = S->pinfo[slot[i]];
    S->jf_keyed -= (pi.jf & (COOK_JF_GPUS | COOK_JF_DISK)) ? 1 : 0;
    pi.jf = flags[i];
    S->jf_keyed += (pi.jf & (COOK_JF_GPUS | COOK_JF_DISK)) ? 1 : 0;
  }
  // ---- device: a patch scatter (live flag and generation kept)
  const bool cols = n && (flags || gpu_model || disk_request || disk_limit || disk_type);
  ScatterArgs pa;
  memset(&pa, 0, sizeof(pa));
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (cols)
      patch_args(c, pa, S->pend, slot.data(), n,
                 {{P_JF, flags, 0}, {P_JF_GPU, gpu_model, 0}, {P_JF_DREQ, disk_request, 0}, {P_JF_DLIM, disk_limit, 0},
                  {P_JF_DTYPE, disk_type, 0}});
  }))
    return rc;
  scatter(pa, S->pend, cols ? n : 0, 0, -1, nullptr, w.st, &w.nl);
  return w.end();
}

// The caller's arrays of cook_state_match_metrics
struct MMArrays {
  int64_t* counts; double* amounts; int64_t* row_int; double* row_amount; int64_t* first_jid; int32_t* first_cyc;
  int32_t* ucons; int32_t* umat; int32_t* kind; int32_t* code; double* total;
  void put(const MMOut& o) const {
    const int64_t c[COOK_MMC_N] = {o.n_considerable, o.n_matched, o.head_job_id, o.head_matched, o.n_uris,
                                   o.uris_position, o.n_keys, o.n_too_long, o.n_first};
    std::copy(c, c + COOK_MMC_N, counts);
    const double a[COOK_MMA_N] = {o.total_cpus, o.total_mem, o.pct_cpus[0], o.pct_cpus[1], o.pct_cpus[2],
                                  o.pct_mem[0], o.pct_mem[1], o.pct_mem[2]};
    std::copy(a, a + COOK_MMA_N, amounts);
    for (int r = 0; r < COOK_MM_ROWS; r++) {
      const MMRow& w = o.row[r];
      const int64_t ri[COOK_MMR_NI] = {w.job_id, w.position, w.user, w.ports, w.facts, w.gpu_model, w.disk_type};
      const double ra[COOK_MMR_NF] = {w.cpus, w.mem, w.gpus, w.disk_request, w.disk_limit};
      std::copy(ri, ri + COOK_MMR_NI, row_int + COOK_MMR_NI * r);
      std::copy(ra, ra + COOK_MMR_NF, row_amount + COOK_MMR_NF * r);
    }
    std::copy(o.first_job_id, o.first_job_id + MM_FIRST, first_jid);
    std::copy(o.first_cycles, o.first_cycles + MM_FIRST, first_cyc);
  }
};

int32_t match_metrics(cook_pool* pool, PoolState* S, int32_t U, int32_t D, const int32_t* dropped, int32_t thr,
                      int32_t key_cap, const MMArrays& out, cook_phase_stats* out_stats) {
  const char* who = "cook_state_match_metrics";
  int32_t *out_ucons = out.ucons, *out_umat = out.umat, *out_kind = out.kind, *out_code = out.code;
  double* out_total = out.total;
  // ---- every check the host can make, before any device work
  if (!out.counts || !out.amounts || !out.row_int || !out.row_amount || !out.first_jid || !out.first_cyc || !out_ucons || !out_umat || !out_kind || !out_code || !out_total)
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  if (U <= 0 || D < 0 || thr < 0 || key_cap < 0 || (D && !dropped))
    return set_err(pool, COOK_E_BADARG, "%s: bad sizes or threshold", who);
  if (!S || !S->mm.on) return set_err(pool, COOK_E_BADARG, "%s: no resident match round on this handle", who);
  MetricsRound& R = S->mm;
  if (R.counted) return set_err(pool, COOK_E_BADARG, "%s: the round has already been counted", who);
  int32_t N = 0;
  const int32_t *cons = nullptr, *assign = nullptr;
  if (R.n_rows > 0 && !match_round(pool, R.run, &N, &cons, &assign))
    return set_err(pool, COOK_E_BADARG, "%s: no resident match round on this handle (a later match ran)", who);
  if (count_max(S->users_p) >= U) return set_err(pool, COOK_E_BADARG, "%s: a pending row's user code is >= n_users", who);
  {
    std::vector<uint8_t> seen(N, 0);
    for (int i = 0; i < D; i++) {
      if (dropped[i] < 0 || dropped[i] >= N) return set_err(pool, COOK_E_BADARG, "%s: a dropped position out of range", who);
      if (seen[dropped[i]]++) return set_err(pool, COOK_E_BADARG, "%s: a dropped position twice", who);
    }
  }
  if (out_stats) *out_stats = cook_phase_stats{};
  if (N == 0) {   // an empty round: the counts, the counters zeroed, no device work
    std::fill(out.counts, out.counts + COOK_MMC_N, 0);
    out.counts[COOK_MMC_HEAD_JOB_ID] = out.counts[COOK_MMC_URIS_POSITION] = -1;
    R.u_n = 0;
    R.counted = true;
    return COOK_OK;
  }
  ReadCall rd(pool);
  if (int32_t rc = rd.open(who)) return rc;   // S: the handle holds the round
  cudaStream_t st = rd.st;
  if (int32_t rc = mm_counters_room(pool, R, N, st)) return rc;
  const bool changed = S->pend_epoch != R.epoch;
  const bool keyed = S->jf_keyed > 0;
  const int E = keyed ? 3 * N : 0;
  // ---- one carve: the rows, the orders, the entries, the counters' new pairs, the result block; up the drops
  MMCols r = {};
  int32_t *cnt = nullptr, *blk = nullptr, *ucons = nullptr, *umat = nullptr, *ord_c = nullptr, *ord_m = nullptr,
          *tmp = nullptr, *ent = nullptr, *ord_e = nullptr, *end = nullptr, *o_kind = nullptr, *o_code = nullptr,
          *f_cyc = nullptr, *n_cyc = nullptr, *ord_u = nullptr;
  const int32_t* d_drop = nullptr;
  int64_t *f_jid = nullptr, *n_jid = nullptr;
  double* o_total = nullptr;
  GridFlag* gf = nullptr;
  MMOut* d_out = nullptr;
  if (int32_t rc = rd.scratch([&](Carve& c) {
    r.slot = c.take<int32_t>(N); r.user = c.take<int32_t>(N); r.jid = c.take<int64_t>(N);
    r.cpus = c.take<double>(N); r.mem = c.take<double>(N); r.gpus = c.take<double>(N); r.ports = c.take<int32_t>(N);
    r.jf = c.take<uint8_t>(N); r.gmodel = c.take<int32_t>(N); r.dtype = c.take<int32_t>(N);
    r.dreq = c.take<double>(N); r.dlim = c.take<double>(N); r.matched = c.take<uint8_t>(N); r.cyc = c.take<int32_t>(N);
    cnt = c.take<int32_t>(MMC_N);
    blk = c.take<int32_t>((size_t)std::max(N, E) / CP_BLOCK + 2);
    ucons = c.take<int32_t>(U); umat = c.take<int32_t>(U);
    ord_c = c.take<int32_t>(N); ord_m = c.take<int32_t>(N); tmp = c.take<int32_t>(std::max(N, E));
    if (keyed) {
      ent = c.take<int32_t>(E); ord_e = c.take<int32_t>(E); end = c.take<int32_t>(E);
      o_kind = c.take<int32_t>(E); o_code = c.take<int32_t>(E); o_total = c.take<double>(E);
    }
    f_jid = c.take<int64_t>(MM_FIRST); f_cyc = c.take<int32_t>(MM_FIRST);
    n_jid = c.take<int64_t>(N); n_cyc = c.take<int32_t>(N); ord_u = c.take<int32_t>(N);
    gf = c.take<GridFlag>(2);
    d_out = c.take<MMOut>(1);
    d_drop = c.up(D ? dropped : nullptr, D);
  }))
    return rc;
  CK(pool, cudaMemsetAsync(cnt, 0, sizeof(int32_t) * MMC_N, st));
  CK(pool, cudaMemsetAsync(ucons, 0, sizeof(int32_t) * U, st));
  CK(pool, cudaMemsetAsync(umat, 0, sizeof(int32_t) * U, st));
  CK(pool, cudaMemsetAsync(gf, 0, sizeof(GridFlag) * 2, st));
  int& nl = rd.nl;
  int64_t& d2h = rd.d2h;
  // ---- the rows, the drops, the counts and cycles, the entries; the first-ten and the new pairs in take order
  mm_gather_kernel<<<(N + 255) / 256, 256, 0, st>>>(S->pend.d_col, R.slot.at<int32_t>(0), cons, assign, N, r);
  nl++;
  if (D) {
    mm_drop_kernel<<<(D + 255) / 256, 256, 0, st>>>(d_drop, D, assign, r.matched, cnt + MMC_BAD);
    nl++;
  }
  mm_count_kernel<<<(N + 255) / 256, 256, 0, st>>>(r, N, U, R.u[R.cur].at<int64_t>(0), R.u[R.cur].at<int32_t>(1), R.u_n,
                                                    ucons, umat, cnt);
  grid_check_kernel<<<(N + 255) / 256, 256, 0, st>>>(r.cpus, r.mem, nullptr, N, gf);
  nl += 2;
  const MMKey key{r.jf, r.gmodel, r.dtype, r.dreq, r.dlim, N};
  if (keyed) {
    grid_check_kernel<<<(N + 255) / 256, 256, 0, st>>>(r.gpus, r.dreq, r.dlim, N, gf + 1);
    nl++;
    compact(MMEntries{key, ent}, E, nullptr, blk, cnt + MMC_ENTRIES, E, st, &nl);
  }
  compact(MMTooLong{r.cyc, r.jid, thr, f_jid, f_cyc}, N, nullptr, blk, cnt + MMC_TOO_LONG, N, st, &nl);
  compact(MMUnmatched{r.cyc, r.jid, n_jid, n_cyc}, N, nullptr, blk, cnt + MMC_UNMATCHED, N, st, &nl);
  CK(pool, cudaGetLastError());
  int32_t c0[MMC_N];
  std::vector<int32_t> slots(changed ? N : 0);
  CK(pool, download(c0, cnt, MMC_N, st, &d2h));
  if (changed) CK(pool, download(slots.data(), r.slot, N, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  // ---- the checks only the device could make, before anything is written
  if (c0[MMC_BAD]) return set_err(pool, COOK_E_BADARG, "%s: a dropped position holds no assignment", who);
  for (int k = 0; k < (int)slots.size(); k++)
    if (S->pinfo[slots[k]].touched > R.epoch)
      return set_err(pool, COOK_E_BADARG, "%s: a considerable row changed since the match", who);
  // ---- the orders, the keyed totals, the counters' new pairs by job id, the result block
  CK(pool, csort::sort_indices(ord_c, tmp, N, LessValuePos{r.cpus}, st, &nl));
  CK(pool, csort::sort_indices(ord_m, tmp, N, LessValuePos{r.mem}, st, &nl));
  const int ne = c0[MMC_ENTRIES], nu = c0[MMC_UNMATCHED];
  if (ne) {
    CK(pool, csort::sort_indices(ord_e, tmp, ne, LessKindCodePos{key, ent}, st, &nl));
    compact(MMSegEnds{key, ent, ord_e, cnt + MMC_ENTRIES, end}, ne, nullptr, blk, cnt + MMC_KEYS, ne, st, &nl);
    fold_segments(end, cnt + MMC_KEYS, ne, false, OrderScan<double, 1>{}, gf + 1, MMKeyLoad{key, r.gpus, ent, ord_e},
                  MMKeyOut{key, ent, ord_e, o_kind, o_code, o_total}, st, &nl);
  }
  const int nxt = 1 - R.cur;
  if (nu) {
    CK(pool, csort::sort_indices(ord_u, tmp, nu, LessJid{n_jid}, st, &nl));
    mm_map_kernel<<<(nu + 255) / 256, 256, 0, st>>>(ord_u, nu, n_jid, n_cyc, R.u[nxt].at<int64_t>(0),
                                                    R.u[nxt].at<int32_t>(1));
    nl++;
  }
  mm_finish_kernel<<<1, 32, 0, st>>>(r, N, gf, ord_c, ord_m, cnt, f_jid, f_cyc, d_out);
  nl++;
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  MMOut res;
  CK(pool, download(&res, d_out, 1, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  if (res.n_keys > key_cap) {
    out.counts[COOK_MMC_KEYS] = res.n_keys;
    return set_err(pool, COOK_E_TOO_LARGE, "%s: more keys than key_cap: %d", who, res.n_keys);
  }
  CK(pool, download(out_ucons, ucons, U, st, &d2h));
  CK(pool, download(out_umat, umat, U, st, &d2h));
  if (res.n_keys) {
    CK(pool, download(out_kind, o_kind, res.n_keys, st, &d2h));
    CK(pool, download(out_code, o_code, res.n_keys, st, &d2h));
    CK(pool, download(out_total, o_total, res.n_keys, st, &d2h));
  }
  if (int32_t rc = rd.close(out_stats)) return rc;
  out.put(res);
  R.cur = nxt;
  R.u_n = nu;
  R.counted = true;
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_job_facts(cook_pool* pool, int32_t n, const int64_t* job_id, const uint8_t* flags,
                                        const int32_t* gpu_model, const double* disk_request, const double* disk_limit,
                                        const int32_t* disk_type) {
  const char* who = "cook_state_job_facts";
  return on_state(pool, who, [&](PoolState* S) {
    return job_facts(pool, S, who, n, job_id, flags, gpu_model, disk_request, disk_limit, disk_type);
  });
}

extern "C" int32_t cook_state_match_metrics(cook_pool* pool, int32_t n_users, int32_t n_dropped, const int32_t* dropped,
                                            int32_t unmatched_warn_cycles, int32_t key_cap, int64_t* out_counts,
                                            double* out_amounts, int64_t* out_row_int, double* out_row_amount,
                                            int64_t* out_first_job_id, int32_t* out_first_cycles,
                                            int32_t* out_user_considerable, int32_t* out_user_matched,
                                            int32_t* out_key_kind, int32_t* out_key_code, double* out_key_total,
                                            cook_phase_stats* out_stats) {
  if (!pool) return COOK_E_BADARG;
  const MMArrays out{out_counts, out_amounts, out_row_int, out_row_amount, out_first_job_id, out_first_cycles,
                     out_user_considerable, out_user_matched, out_key_kind, out_key_code, out_key_total};
  return match_metrics(pool, static_cast<PoolState*>(pool->state), n_users, n_dropped, dropped, unmatched_warn_cycles,
                       key_cap, out, out_stats);
}

// ---- job listing (/list, /jobs for the waiting and running states; get-active-jobs-by-user-and-state,
// tools.clj:445-466).  Per state: one flag pass per handle marks the user's live rows and counts those in the id window
// without list facts; a compaction gathers them (job id, task id, pool index, submit time and whether the entry passes
// the filters) after the handles before; one sort by (job id, pool index, task id descending) orders them across the
// handles and puts each running job's representative first; a second compaction keeps the first row of each
// (job id, pool index) that passes, up to `limit`, straight into the download buffers.
namespace {

struct LJCols {   // one table's columns the listing reads; tid null for the pending table
  const uint8_t* live; const int32_t* user; const int64_t* jid; const int64_t* tid; const int64_t* submit;
  const int32_t* spool; const uint8_t* exec;
};
struct LJSel { int64_t start, end, lo, hi; int32_t pool; int32_t all_exec; };

__global__ void lj_flag_kernel(LJCols c, int n, int32_t user, int64_t lo, int64_t hi, uint8_t* flag, int32_t* missing) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool miss = false;
  if (i < n) {
    const bool mine = c.live[i] && c.user[i] == user;
    flag[i] = mine;
    miss = mine && c.exec[i] == 0 && c.jid[i] >= lo && c.jid[i] < hi;
  }
  const int m = __reduce_add_sync(FULL_MASK, miss ? 1 : 0);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(missing, m);
}

// the flagged rows of one handle, dense after the handles before it (base); pool_ok: the handle is the requested pool
struct LJRows {
  LJCols c; const uint8_t* flag; int base; int32_t pidx; bool pool_ok; LJSel q;
  int64_t* jid; int64_t* tid; int32_t* pi; int64_t* submit; uint8_t* ok;
  __device__ bool keep(int i) const { return flag[i]; }
  __device__ void emit(int i, int d) const {
    d += base;
    const int64_t j = c.jid[i], s = c.submit[i];
    const uint8_t e = c.exec[i];
    jid[d] = j;
    if (tid) tid[d] = c.tid[i];
    pi[d] = pidx;
    submit[d] = s;
    ok[d] = e != 0 && s >= q.start && s < q.end && j >= q.lo && j < q.hi && (pool_ok || c.spool[i] == q.pool) &&
            (q.all_exec || e == 2);
  }
};

// (job id, pool index, task id descending, dense index): a job's rows in one handle together, the representative first
struct LessJobPoolTask {
  const int64_t* jid; const int32_t* pi; const int64_t* tid;
  __device__ bool operator()(int32_t a, int32_t b) const {
    if (jid[a] != jid[b]) return jid[a] < jid[b];
    if (pi[a] != pi[b]) return pi[a] < pi[b];
    if (tid && tid[a] != tid[b]) return tid[a] > tid[b];
    return a < b;
  }
};

// the first row of each job (BY_POOL: of each (job id, pool index)) in a sorted order, when it passes the filters
template <bool BY_POOL>
struct JobPick {
  const int32_t* ord; const int64_t* jid; const int32_t* pi; const int64_t* submit; const uint8_t* ok;
  int64_t* o_jid; int64_t* o_submit; int32_t* o_pi;
  __device__ bool keep(int p) const {
    const int i = ord[p];
    if (p > 0) {
      const int k = ord[p - 1];
      if (jid[k] == jid[i] && (!BY_POOL || pi[k] == pi[i])) return false;
    }
    return ok[i];
  }
  __device__ void emit(int p, int d) const {
    const int i = ord[p];
    o_jid[d] = jid[i]; o_submit[d] = submit[i]; o_pi[d] = pi[i];
  }
};
using LJPick = JobPick<true>;

LJCols lj_cols(const PoolState* s, bool running) {
  if (running) {
    const Table& t = s->run;
    return {t.at<uint8_t>(R_LIVE), t.at<int32_t>(R_USER), t.at<int64_t>(R_JID), t.at<int64_t>(R_TID),
            t.at<int64_t>(R_LF_SUBMIT), t.at<int32_t>(R_LF_POOL), t.at<uint8_t>(R_LF_EXEC)};
  }
  const Table& t = s->pend;
  return {t.at<uint8_t>(P_LIVE), t.at<int32_t>(P_USER), t.at<int64_t>(P_JID), nullptr, t.at<int64_t>(P_LF_SUBMIT),
          t.at<int32_t>(P_LF_POOL), t.at<uint8_t>(P_LF_EXEC)};
}

int32_t list_facts(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* job_id, const int64_t* submit_ms,
                   const int32_t* submit_pool, const int32_t* custom_executor) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && !job_id) return set_err(pool, COOK_E_BADARG, "%s: null job_id", who);
  for (int i = 0; custom_executor && i < n; i++)
    if (custom_executor[i] < -1 || custom_executor[i] > 1)
      return set_err(pool, COOK_E_BADARG, "%s: a custom_executor outside {-1, 0, 1}", who);
  if (!idx_in_range(submit_pool, n, -1, INT32_MAX)) return set_err(pool, COOK_E_BADARG, "%s: a submit pool code below -1", who);
  // the rows written: the job's live pending row, then each of its live running rows; k: the batch row it takes from
  std::vector<int32_t> pslot, pk, rslot, rk;
  {
    std::unordered_set<int64_t> seen;
    seen.reserve((size_t)n);
    for (int i = 0; i < n; i++) {
      if (!seen.insert(job_id[i]).second) return set_err(pool, COOK_E_BADARG, "%s: job id twice", who);
      auto p = S->pend.slot_of.find(job_id[i]);
      auto r = S->jobs_r.find(job_id[i]);
      if (p == S->pend.slot_of.end() && r == S->jobs_r.end())
        return set_err(pool, COOK_E_BADARG, "%s: a job id neither live-pending nor live-running", who);
      if (p != S->pend.slot_of.end()) { pslot.push_back(p->second); pk.push_back(i); }
      if (r != S->jobs_r.end())
        for (int32_t s : r->second) { rslot.push_back(s); rk.push_back(i); }
    }
  }
  // ---- the values per row written (LF_EXEC stores 2 + custom_executor), then one patch scatter per table
  const int np = (int)pslot.size(), nr = (int)rslot.size(), m = np + nr;
  std::vector<int64_t> sub(submit_ms ? m : 0);
  std::vector<int32_t> sp(submit_pool ? m : 0);
  std::vector<uint8_t> ex(custom_executor ? m : 0);
  for (int w = 0; w < m; w++) {
    const int i = w < np ? pk[w] : rk[w - np];
    if (submit_ms) sub[w] = submit_ms[i];
    if (submit_pool) sp[w] = submit_pool[i];
    if (custom_executor) ex[w] = (uint8_t)(custom_executor[i] + 2);
  }
  const bool cols = submit_ms || submit_pool || custom_executor;
  ScatterArgs pa, ra;
  memset(&pa, 0, sizeof(pa)); memset(&ra, 0, sizeof(ra));
  StateWrite w(pool, S);
  if (int32_t rc = w.up([&](Carve& c) {
    if (!cols) return;
    // the batch's values from row `off` on (null: the column is not written)
    const auto at = [](const auto& v, bool given, int off) { return given ? v.data() + off : nullptr; };
    if (np)
      patch_args(c, pa, S->pend, pslot.data(), np,
                 {{P_LF_SUBMIT, at(sub, submit_ms, 0), 0}, {P_LF_POOL, at(sp, submit_pool, 0), 0},
                  {P_LF_EXEC, at(ex, custom_executor, 0), 0}});
    if (nr)
      patch_args(c, ra, S->run, rslot.data(), nr,
                 {{R_LF_SUBMIT, at(sub, submit_ms, np), 0}, {R_LF_POOL, at(sp, submit_pool, np), 0},
                  {R_LF_EXEC, at(ex, custom_executor, np), 0}});
  }))
    return rc;
  scatter(pa, S->pend, cols ? np : 0, 0, -1, nullptr, w.st, &w.nl);
  scatter(ra, S->run, cols ? nr : 0, 0, -1, nullptr, w.st, &w.nl);
  return w.end();
}

// the listing arguments cook_state_list_jobs and cook_state_list_completed share
int32_t check_list_args(cook_pool* pool, const char* who, int32_t user, const LJSel& q, const int32_t* handle_pool,
                        int32_t limit, int32_t cap) {
  if (user < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative user", who);
  if (q.pool < -1 || (q.pool != -1 && !handle_pool))
    return set_err(pool, COOK_E_BADARG, "%s: pool_code below -1, or no handle_pool", who);
  if (q.all_exec != 0 && q.all_exec != 1) return set_err(pool, COOK_E_BADARG, "%s: include_custom_executor outside {0, 1}", who);
  if (limit < 0 || cap < 0) return set_err(pool, COOK_E_BADARG, "%s: limit < 0 or cap < 0", who);
  return COOK_OK;
}

// n listed entries down: job id, submit time, pool index (20 B each)
cudaError_t download_entries(int64_t* o_jid, int64_t* o_submit, int32_t* o_pool, const int64_t* jid, const int64_t* submit,
                             const int32_t* pi, int n, cudaStream_t st, int64_t* d2h) {
  cudaError_t e = download(o_jid, jid, n, st, d2h);
  if (e == cudaSuccess) e = download(o_submit, submit, n, st, d2h);
  if (e == cudaSuccess) e = download(o_pool, pi, n, st, d2h);
  return e;
}

int32_t list_jobs(cook_pool* const* pools, int n, int32_t user, int32_t states, const LJSel& q, const int32_t* handle_pool,
                  int32_t limit, int32_t cap, int32_t* o_state, int64_t* o_jid, int64_t* o_submit, int32_t* o_pool,
                  int32_t* o_n, int32_t* o_missing, cook_phase_stats* out_stats) {
  const char* who = "cook_state_list_jobs";
  // ---- every check before any device work or output
  if (int32_t rc = check_handle_set(pools, n, who)) return rc;
  cook_pool* pool = pools[0];
  if (states <= 0 || (states & ~(COOK_LJ_WAITING | COOK_LJ_RUNNING)))
    return set_err(pool, COOK_E_BADARG, "%s: states 0 or with unknown bits", who);
  if (int32_t rc = check_list_args(pool, who, user, q, handle_pool, limit, cap)) return rc;
  if (!o_state || !o_jid || !o_submit || !o_pool || !o_n || !o_missing) return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  // per state (0 waiting, 1 running): the handles holding a row of the user, and the rows (the host-side counts)
  struct Src { const PoolState* s; int32_t k; int rows; };
  std::vector<Src> hs[2];
  int64_t C[2] = {0, 0};
  int hw = 0;
  for (int t = 0; t < 2; t++) {
    if (!(states & (t ? COOK_LJ_RUNNING : COOK_LJ_WAITING))) continue;
    for (int k = 0; k < n; k++) {
      const PoolState* s = static_cast<const PoolState*>(pools[k]->state);
      if (!s) continue;
      const auto& users = t ? s->users_r : s->users_p;
      auto it = users.find(user);
      if (it == users.end()) continue;
      hs[t].push_back({s, k, (int)it->second});
      C[t] += it->second;
      hw = std::max(hw, t ? s->run.hw : s->pend.hw);
    }
  }
  if (C[0] > INT32_MAX || C[1] > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 rows in a state", who);
  if (C[0] + C[1] == 0) {   // no row to read: empty results without device work
    *o_n = 0;
    *o_missing = 0;
    return no_rows(out_stats);
  }
  ReadCall r(pool);
  if (int32_t rc = r.open(who)) return rc;
  cudaStream_t st = r.st;
  // ---- one carve: the flags, each state's rows, order and entries, the counts
  struct Dense { int64_t *jid, *tid, *submit, *o_jid, *o_submit; int32_t *pi, *ord, *o_pi; uint8_t* ok; };
  Dense D[2] = {};
  int32_t *cnt = nullptr, *blk = nullptr, *tmp = nullptr;
  uint8_t* flag = nullptr;
  const int Cmax = (int)std::max(C[0], C[1]);
  if (int32_t rc = r.scratch([&](Carve& c) {
    cnt = c.take<int32_t>(4);   // [0] [1] the states' entries, [2] rows without facts, [3] the row compactions' own
    blk = c.take<int32_t>((size_t)std::max(hw, Cmax) / CP_BLOCK + 2);
    flag = c.take<uint8_t>(hw);
    tmp = c.take<int32_t>(Cmax);
    for (int t = 0; t < 2; t++) {
      if (!C[t]) continue;
      const int Ct = (int)C[t], Ot = std::min(Ct, limit);
      Dense& d = D[t];
      d.jid = c.take<int64_t>(Ct); d.submit = c.take<int64_t>(Ct); d.pi = c.take<int32_t>(Ct);
      d.ok = c.take<uint8_t>(Ct); d.ord = c.take<int32_t>(Ct);
      if (t) d.tid = c.take<int64_t>(Ct);
      d.o_jid = c.take<int64_t>(Ot); d.o_submit = c.take<int64_t>(Ot); d.o_pi = c.take<int32_t>(Ot);
    }
  }))
    return rc;
  CK(pool, cudaMemsetAsync(cnt, 0, sizeof(int32_t) * 4, st));
  int& nl = r.nl;
  int64_t& d2h = r.d2h;
  for (int t = 0; t < 2; t++) {
    if (!C[t]) continue;
    Dense& d = D[t];
    int base = 0;
    for (const Src& h : hs[t]) {
      const LJCols cols = lj_cols(h.s, t == 1);
      const int T = t ? h.s->run.hw : h.s->pend.hw;
      lj_flag_kernel<<<(T + 255) / 256, 256, 0, st>>>(cols, T, user, q.lo, q.hi, flag, cnt + 2);
      nl++;
      const bool pool_ok = q.pool == -1 || handle_pool[h.k] == q.pool;
      compact(LJRows{cols, flag, base, h.k, pool_ok, q, d.jid, d.tid, d.pi, d.submit, d.ok}, T, nullptr, blk, cnt + 3,
              h.rows, st, &nl);
      base += h.rows;
    }
    const int Ct = (int)C[t];
    CK(pool, csort::sort_indices(d.ord, tmp, Ct, LessJobPoolTask{d.jid, d.pi, d.tid}, st, &nl));
    compact(LJPick{d.ord, d.jid, d.pi, d.submit, d.ok, d.o_jid, d.o_submit, d.o_pi}, Ct, nullptr, blk, cnt + t, limit, st,
            &nl);
  }
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  int32_t got[3];
  CK(pool, download(got, cnt, 3, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  const int64_t need = (int64_t)got[0] + got[1];
  if (need > cap) {
    *o_n = (int32_t)need;
    return set_err(pool, COOK_E_TOO_LARGE, "%s: more entries than cap: %lld", who, (long long)need);
  }
  int at = 0;
  for (int t = 0; t < 2; t++) {
    if (!got[t]) continue;
    CK(pool, download_entries(o_jid + at, o_submit + at, o_pool + at, D[t].o_jid, D[t].o_submit, D[t].o_pi, got[t], st,
                              &d2h));
    std::fill(o_state + at, o_state + at + got[t], t ? COOK_LJ_RUNNING : COOK_LJ_WAITING);
    at += got[t];
  }
  if (int32_t rc = r.close(out_stats)) return rc;
  *o_n = at;
  *o_missing = got[2];
  return COOK_OK;
}

// ---- the completed-job log (cook_state_completed_*) and its listing (cook_state_list_completed, the completed, success
// and failed states; get-completed-jobs-by-user, tools.clj:393-434).  The listing: a compaction per handle gathers the
// user's records (job id, stamp, submit time, pool index, and whether the record passes the filters) after the handles
// before; one sort by (job id, stamp descending, dense index descending) puts each job's latest record first (the dense
// index grows with (handle, row)); a second compaction keeps each job's first record when it passes, up to `limit`.
static_assert((int)COOK_CJ_SUCCESS == (int)COOK_LC_SUCCESS && (int)COOK_CJ_FAILED == (int)COOK_LC_FAILED,
              "a listed state names the record kind it keeps");
struct CJRows {
  CJCols c; int32_t user; int base; int32_t pidx; bool pool_ok; LJSel q; int32_t state;
  int64_t* jid; int64_t* stamp; int64_t* submit; int32_t* pi; uint8_t* ok;
  __device__ bool keep(int i) const { return c.user[i] == user; }
  template <class V> void outs(V&& v) { v(jid); v(stamp); v(submit); v(pi); v(ok); }
  __device__ void emit(int i, int d) const {
    d += base;
    const int64_t j = c.jid[i], s = c.submit[i];
    const uint8_t k = c.kind[i];
    jid[d] = j;
    stamp[d] = c.stamp[i];
    submit[d] = s;
    pi[d] = pidx;
    ok[d] = k != COOK_CJ_REOPENED && (state == COOK_LC_COMPLETED || k == state) && s >= q.start && s < q.end &&
            j >= q.lo && j < q.hi && (pool_ok || c.spool[i] == q.pool) && (q.all_exec || c.exec[i] == 0);
  }
};

// (job id, stamp descending, dense index descending): each job's latest record first
struct LessJobStamp {
  const int64_t* jid; const int64_t* stamp;
  __device__ bool operator()(int32_t a, int32_t b) const {
    if (jid[a] != jid[b]) return jid[a] < jid[b];
    if (stamp[a] != stamp[b]) return stamp[a] > stamp[b];
    return a > b;
  }
};

// The host columns of a seed or record batch, checked row by row: the rows kept (submit >= since), the executor as the
// stored byte.
struct CJBatch {
  std::vector<int64_t> jid, stamp, submit;
  std::vector<int32_t> user, spool;
  std::vector<int8_t> exec;
  std::vector<uint8_t> kind;
};

int32_t cj_batch(cook_pool* pool, const char* who, int n, int64_t since, bool skip, const int64_t* job_id,
                 const int64_t* stamp, const int32_t* user, const int64_t* submit_ms, const int32_t* submit_pool,
                 const int32_t* custom_executor, const uint8_t* kind, CJBatch* b) {
  if (n < 0) return set_err(pool, COOK_E_BADARG, "%s: n < 0", who);
  if (n && (!job_id || !stamp || !user || !submit_ms || !submit_pool || !custom_executor || !kind))
    return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  std::unordered_set<int64_t> seen;
  seen.reserve((size_t)n);
  for (int i = 0; i < n; i++) {
    if (submit_ms[i] < since && !skip) return set_err(pool, COOK_E_BADARG, "%s: a row submitted before since_ms", who);
    if (user[i] < 0 || stamp[i] < 0) return set_err(pool, COOK_E_BADARG, "%s: a negative user or stamp", who);
    if (kind[i] < COOK_CJ_SUCCESS || kind[i] > COOK_CJ_REOPENED) return set_err(pool, COOK_E_BADARG, "%s: an unknown kind", who);
    if (custom_executor[i] < -1 || custom_executor[i] > 1)
      return set_err(pool, COOK_E_BADARG, "%s: a custom_executor outside {-1, 0, 1}", who);
    if (submit_pool[i] < -1) return set_err(pool, COOK_E_BADARG, "%s: a submit pool code below -1", who);
    if (!seen.insert(job_id[i]).second) return set_err(pool, COOK_E_BADARG, "%s: job id twice", who);
  }
  for (int i = 0; i < n; i++) {
    if (submit_ms[i] < since) continue;
    b->jid.push_back(job_id[i]); b->stamp.push_back(stamp[i]); b->submit.push_back(submit_ms[i]);
    b->user.push_back(user[i]); b->spool.push_back(submit_pool[i]); b->exec.push_back((int8_t)custom_executor[i]);
    b->kind.push_back(kind[i]);
  }
  return COOK_OK;
}

// the batch's rows appended at the log's tail, straight into its columns
int32_t cj_append(cook_pool* pool, PoolState* S, const CJBatch& b, const char* who) {
  Completed& L = S->cj;
  const int64_t k = (int64_t)b.jid.size();
  if (L.tail + k > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 log rows", who);
  CK(pool, L.grow(L.tail + k, pool->stream));
  const int64_t t = L.tail;
  StateWrite w(pool, S);
  if (int32_t rc = w.direct([&](Carve& c) {
    if (!k) return;
    L.c.copy(c, t, k, {b.jid.data(), b.stamp.data(), b.submit.data(), b.user.data(), b.spool.data(), b.exec.data(),
                       b.kind.data()});
  }))
    return rc;
  if (int32_t rc = w.end()) return rc;
  L.tail += k;
  L.h_user.insert(L.h_user.end(), b.user.begin(), b.user.end());
  L.h_submit.insert(L.h_submit.end(), b.submit.begin(), b.submit.end());
  for (int32_t u : b.user) L.users[u]++;
  return COOK_OK;
}

int32_t completed_seed(cook_pool* pool, PoolState* S, const char* who, int64_t since_ms, int n, const int64_t* job_id,
                       const int64_t* stamp, const int32_t* user, const int64_t* submit_ms, const int32_t* submit_pool,
                       const int32_t* custom_executor, const uint8_t* kind) {
  CJBatch b;
  if (int32_t rc = cj_batch(pool, who, n, since_ms, false, job_id, stamp, user, submit_ms, submit_pool, custom_executor,
                            kind, &b))
    return rc;
  Completed& L = S->cj;
  L.clear_rows();
  L.since = since_ms;
  L.on = true;
  return cj_append(pool, S, b, who);
}

int32_t completed_record(cook_pool* pool, PoolState* S, const char* who, int n, const int64_t* job_id,
                         const int64_t* stamp, const int32_t* user, const int64_t* submit_ms, const int32_t* submit_pool,
                         const int32_t* custom_executor, const uint8_t* kind) {
  if (!S->cj.on) return set_err(pool, COOK_E_BADARG, "%s: the log is off", who);
  CJBatch b;
  if (int32_t rc = cj_batch(pool, who, n, S->cj.since, true, job_id, stamp, user, submit_ms, submit_pool,
                            custom_executor, kind, &b))
    return rc;
  return cj_append(pool, S, b, who);
}

// the horizon raised to since_ms: the rows submitted before it leave in one compaction into new columns, and from the
// host's rows
int32_t completed_advance(cook_pool* pool, PoolState* S, const char* who, int64_t since_ms) {
  Completed& L = S->cj;
  if (!L.on) return set_err(pool, COOK_E_BADARG, "%s: the log is off", who);
  if (since_ms < L.since) return set_err(pool, COOK_E_BADARG, "%s: since_ms below the horizon", who);
  int32_t* blk = nullptr;
  const int T = (int)L.tail;
  const bool move = T && since_ms > L.since;
  StateWrite w(pool, S);
  if (int32_t rc = w.up(S->scratch, [&](Carve& c) {
    if (move) blk = c.take<int32_t>((size_t)T / CP_BLOCK + 2);
  }))
    return rc;
  if (move)
    if (int32_t rc = log_advance(pool, S, w, L, CJ_SUBMIT, since_ms, blk)) return rc;
  if (int32_t rc = w.end()) return rc;
  if (move) {   // the host's rows, by the same rule and in the same order
    int64_t w = 0;
    for (int64_t i = 0; i < T; i++) {
      if (L.h_submit[i] >= since_ms) {
        L.h_user[w] = L.h_user[i];
        L.h_submit[w++] = L.h_submit[i];
      } else if (--L.users[L.h_user[i]] == 0) {
        L.users.erase(L.h_user[i]);
      }
    }
    L.h_user.resize(w);
    L.h_submit.resize(w);
    if (L.tail != w) return set_err(pool, COOK_E_CUDA, "%s: the device kept %lld rows, the host %lld", who,
                                    (long long)L.tail, (long long)w);
  }
  L.since = since_ms;
  return COOK_OK;
}

int32_t list_completed(cook_pool* const* pools, int n, int32_t user, int32_t state, const LJSel& q,
                       const int32_t* handle_pool, int32_t limit, int32_t cap, int64_t* o_jid, int64_t* o_submit,
                       int32_t* o_pool, int32_t* o_n, cook_phase_stats* out_stats) {
  const char* who = "cook_state_list_completed";
  // ---- every check before any device work or output
  if (int32_t rc = check_handle_set(pools, n, who, true)) return rc;
  cook_pool* pool = pools[0];
  if (state != COOK_LC_SUCCESS && state != COOK_LC_FAILED && state != COOK_LC_COMPLETED)
    return set_err(pool, COOK_E_BADARG, "%s: an unknown state", who);
  if (int32_t rc = check_list_args(pool, who, user, q, handle_pool, limit, cap)) return rc;
  if (!o_jid || !o_submit || !o_pool || !o_n) return set_err(pool, COOK_E_BADARG, "%s: null argument", who);
  // the handles holding a record of the user, and the records (the host-side counts)
  struct Src { const Completed* l; int32_t k; int rows; };
  std::vector<Src> hs;
  int64_t C = 0;
  int tmax = 0;
  for (int k = 0; k < n; k++) {
    const PoolState* s = static_cast<const PoolState*>(pools[k]->state);
    if (!s || !s->cj.on) return set_err(pool, COOK_E_BADARG, "%s: a handle whose log is off", who);
    if (s->cj.since > q.start) return set_err(pool, COOK_E_BADARG, "%s: start_ms before a handle's horizon", who);
    auto it = s->cj.users.find(user);
    if (it == s->cj.users.end()) continue;
    hs.push_back({&s->cj, k, (int)it->second});
    C += it->second;
    tmax = std::max(tmax, (int)s->cj.tail);
  }
  if (C > INT32_MAX) return set_err(pool, COOK_E_TOO_LARGE, "%s: more than 2^31 - 1 records of the user", who);
  if (C == 0) {   // no record to read: empty results without device work
    *o_n = 0;
    return no_rows(out_stats);
  }
  ReadCall r(pool);
  if (int32_t rc = r.open(who)) return rc;
  cudaStream_t st = r.st;
  // ---- one carve: the records, their order, the entries, the counts
  const int Cn = (int)C, On = std::min(Cn, limit);
  int64_t *jid = nullptr, *stamp = nullptr, *submit = nullptr, *e_jid = nullptr, *e_submit = nullptr;
  int32_t *pi = nullptr, *ord = nullptr, *tmp = nullptr, *e_pi = nullptr, *cnt = nullptr, *blk = nullptr;
  uint8_t* ok = nullptr;
  if (int32_t rc = r.scratch([&](Carve& c) {
    cnt = c.take<int32_t>(2);   // [0] the entries, [1] the record compactions' own
    blk = c.take<int32_t>((size_t)std::max(tmax, Cn) / CP_BLOCK + 2);
    jid = c.take<int64_t>(Cn); stamp = c.take<int64_t>(Cn); submit = c.take<int64_t>(Cn);
    pi = c.take<int32_t>(Cn); ok = c.take<uint8_t>(Cn); ord = c.take<int32_t>(Cn); tmp = c.take<int32_t>(Cn);
    e_jid = c.take<int64_t>(On); e_submit = c.take<int64_t>(On); e_pi = c.take<int32_t>(On);
  }))
    return rc;
  int& nl = r.nl;
  int64_t& d2h = r.d2h;
  int base = 0;
  Gather g(pool);
  for (const Src& h : hs) {
    const bool pool_ok = q.pool == -1 || handle_pool[h.k] == q.pool;   // on the host: no array crosses devices
    CK(pool, g.rows(pools[h.k], CJRows{h.l->cols(), user, base, h.k, pool_ok, q, state, jid, stamp, submit, pi, ok},
                    (int)h.l->tail, h.rows, blk, cnt + 1, &nl));
    base += h.rows;
  }
  CK(pool, csort::sort_indices(ord, tmp, Cn, LessJobStamp{jid, stamp}, st, &nl));
  compact(JobPick<false>{ord, jid, pi, submit, ok, e_jid, e_submit, e_pi}, Cn, nullptr, blk, cnt, limit, st, &nl);
  CK(pool, cudaGetLastError());
  CK(pool, cudaEventRecord(pool->ev[22], st));
  int32_t got = 0;
  CK(pool, download(&got, cnt, 1, st, &d2h));
  CK(pool, cudaStreamSynchronize(st));
  if (got > cap) {
    *o_n = got;
    return set_err(pool, COOK_E_TOO_LARGE, "%s: more entries than cap: %d", who, got);
  }
  if (got) CK(pool, download_entries(o_jid, o_submit, o_pool, e_jid, e_submit, e_pi, got, st, &d2h));
  if (int32_t rc = r.close(out_stats)) return rc;
  *o_n = got;
  return COOK_OK;
}

}  // namespace

extern "C" int32_t cook_state_list_facts(cook_pool* pool, int32_t n, const int64_t* job_id, const int64_t* submit_ms,
                                         const int32_t* submit_pool, const int32_t* custom_executor) {
  const char* who = "cook_state_list_facts";
  return on_state(pool, who, [&](PoolState* S) {
    return list_facts(pool, S, who, n, job_id, submit_ms, submit_pool, custom_executor);
  });
}

extern "C" int32_t cook_state_list_jobs(cook_pool* const* pools, int32_t n_pools, int32_t user, int32_t states,
                                        int64_t start_ms, int64_t end_ms, int64_t job_id_lo, int64_t job_id_hi,
                                        int32_t pool_code, const int32_t* handle_pool, int32_t include_custom_executor,
                                        int32_t limit, int32_t cap, int32_t* out_state, int64_t* out_job_id,
                                        int64_t* out_submit_ms, int32_t* out_pool, int32_t* out_n,
                                        int32_t* out_n_missing, cook_phase_stats* out_stats) {
  const LJSel q{start_ms, end_ms, job_id_lo, job_id_hi, pool_code, include_custom_executor};
  return list_jobs(pools, n_pools, user, states, q, handle_pool, limit, cap, out_state, out_job_id, out_submit_ms,
                   out_pool, out_n, out_n_missing, out_stats);
}

extern "C" int32_t cook_state_completed_seed(cook_pool* pool, int64_t since_ms, int32_t n, const int64_t* job_id,
                                             const int64_t* stamp, const int32_t* user, const int64_t* submit_ms,
                                             const int32_t* submit_pool, const int32_t* custom_executor,
                                             const uint8_t* kind) {
  const char* who = "cook_state_completed_seed";
  return on_state(pool, who, [&](PoolState* S) {
    return completed_seed(pool, S, who, since_ms, n, job_id, stamp, user, submit_ms, submit_pool, custom_executor, kind);
  });
}

extern "C" int32_t cook_state_completed_record(cook_pool* pool, int32_t n, const int64_t* job_id, const int64_t* stamp,
                                               const int32_t* user, const int64_t* submit_ms, const int32_t* submit_pool,
                                               const int32_t* custom_executor, const uint8_t* kind) {
  const char* who = "cook_state_completed_record";
  return on_state(pool, who, [&](PoolState* S) {
    return completed_record(pool, S, who, n, job_id, stamp, user, submit_ms, submit_pool, custom_executor, kind);
  });
}

extern "C" int32_t cook_state_completed_advance(cook_pool* pool, int64_t since_ms) {
  const char* who = "cook_state_completed_advance";
  return on_state(pool, who, [&](PoolState* S) { return completed_advance(pool, S, who, since_ms); });
}

extern "C" int32_t cook_state_list_completed(cook_pool* const* pools, int32_t n_pools, int32_t user, int32_t state,
                                             int64_t start_ms, int64_t end_ms, int64_t job_id_lo, int64_t job_id_hi,
                                             int32_t pool_code, const int32_t* handle_pool,
                                             int32_t include_custom_executor, int32_t limit, int32_t cap,
                                             int64_t* out_job_id, int64_t* out_submit_ms, int32_t* out_pool,
                                             int32_t* out_n, cook_phase_stats* out_stats) {
  const LJSel q{start_ms, end_ms, job_id_lo, job_id_hi, pool_code, include_custom_executor};
  return list_completed(pools, n_pools, user, state, q, handle_pool, limit, cap, out_job_id, out_submit_ms, out_pool,
                        out_n, out_stats);
}
