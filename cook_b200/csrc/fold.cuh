// fold.cuh — the f64 running sums of the path and the index plumbing around them.
//
// Every running sum is the reference's left fold (common.cuh, "Exact-grid fast path"): a parallel
// scan when grid_exact says every partial sum is exact, else the lane-serial chain below, which keeps
// the association.  Around them: segment bounds of a sorted order, the order-wide tile scan that
// replaces per-segment folds on the grid, and stable stream compaction.
#pragma once
#include "common.cuh"

namespace {   // one copy per translation unit, like the kernels that use it

constexpr unsigned FULL_MASK = 0xffffffffu;

// ---- warp left folds over K f64 columns; lane l holds slot l of a chunk of 32 slots.  `stage` is the
// calling warp's own K x 32 doubles of shared memory.
// The serial chain: the chunk is staged, lane k runs column k over the lanes of `mask` in lane order,
// carry[k] = carry[k] + x[k] of that lane, so the sum is ((carry + x_a) + x_b) + ... whatever the addends.
// Each lane of `mask` gets its inclusive value in mine[k].  One ld.shared / add / st.shared per slot on K
// lanes: cheaper than shuffling every slot to the whole warp when many warps fold at once.
template <int K>
__device__ __forceinline__ void warp_chain(const double (&x)[K], double (&carry)[K], double (&mine)[K], unsigned mask,
                                           double (*stage)[32]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < K; k++) stage[k][lane] = x[k];
  __syncwarp();
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < K; k++)
    if (lane == k) acc = carry[k];
  if (lane < K) {
    double* row = stage[lane];
    const int cnt = 32 - __clz(mask);
#pragma unroll 8
    for (int l = 0; l < cnt; l++) {
      if ((mask >> l) & 1u) acc = acc + row[l];
      row[l] = acc;
    }
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < K; k++) {
    mine[k] = stage[k][lane];
    carry[k] = __shfl_sync(FULL_MASK, acc, k);
  }
  __syncwarp();
}

// Inclusive prefix over the first `cnt` slots of a chunk: x[k] becomes carry[k] + x_0 + ... + x_lane and
// carry[k] moves past the chunk.  `exact`: the sums are association-free (grid_exact), so a parallel scan.
template <int K>
__device__ __forceinline__ void warp_fold_prefix(double (&x)[K], double (&carry)[K], int cnt, bool exact,
                                                 double (*stage)[32]) {
  const int lane = threadIdx.x & 31;
  if (exact) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      x[k] = carry[k] + warp_incl_scan(x[k], lane);
      carry[k] = __shfl_sync(FULL_MASK, x[k], cnt - 1);
    }
    return;
  }
  warp_chain(x, carry, x, cnt >= 32 ? FULL_MASK : (1u << cnt) - 1u, stage);
}

// The sum of items 0 .. n-1 added to carry (every lane gets it).  load(i, x) fills the addends of item i
// into the zeroed x and says whether the item takes part (one that does not must leave x zero); D
// chunks are loaded ahead.  `exact`: lane partial sums and a butterfly; else the chain over the items
// that take part.
template <int K, int D, class Load>
__device__ __forceinline__ void warp_fold_sum(double (&carry)[K], int n, bool exact, const Load& load,
                                              double (*stage)[32]) {
  const int lane = threadIdx.x & 31;
  double part[K];
#pragma unroll
  for (int k = 0; k < K; k++) part[k] = 0.0;
  for (int base = 0; base < n; base += 32 * D) {
    double x[D][K];
    bool on[D];
#pragma unroll
    for (int q = 0; q < D; q++) {
      const int i = base + 32 * q + lane;
#pragma unroll
      for (int k = 0; k < K; k++) x[q][k] = 0.0;
      on[q] = i < n && load(i, x[q]);
    }
#pragma unroll
    for (int q = 0; q < D; q++) {
      if (exact) {
#pragma unroll
        for (int k = 0; k < K; k++) part[k] += x[q][k];
      } else {
        double mine[K];
        warp_chain(x[q], carry, mine, __ballot_sync(FULL_MASK, on[q]), stage);
      }
    }
  }
  if (exact) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      for (int o = 16; o > 0; o >>= 1) part[k] += __shfl_xor_sync(FULL_MASK, part[k], o);
      carry[k] = carry[k] + part[k];
    }
  }
}

// ---- segment bounds of a sorted order: key(p) is the segment (user, host) of position p of n;
// seg_start[k] / seg_end[k] get the first position of segment k and one past its last
template <class Key>
__device__ __forceinline__ int mark_segment(int p, int n, const Key& key, int32_t* seg_start, int32_t* seg_end) {
  const int k = key(p);
  if (p == 0 || key(p - 1) != k) seg_start[k] = p;
  if (p == n - 1 || key(p + 1) != k) seg_end[k] = p + 1;
  return k;
}
struct SortedKey {   // key[ord[p]], or key[map[ord[p]]]
  const int32_t* ord; const int32_t* map; const int32_t* key;
  __device__ int operator()(int p) const {
    int i = ord[p];
    if (map) i = map[i];
    return key[i];
  }
};

// tools.clj:614-641 compare of feature vectors, prefixed by the user's name
// rank so that one global sort yields all per-user lists, users in name order.
struct LessUserTask {
  const int32_t* user; const int32_t* prio; const int64_t* start; const int64_t* tid; const int64_t* jid;
  const int32_t* name_rank;
  __device__ bool operator()(int32_t a, int32_t b) const {
    int ua = name_rank[user[a]], ub = name_rank[user[b]];
    if (ua != ub) return ua < ub;
    int pa = -prio[a], pb = -prio[b];
    if (pa != pb) return pa < pb;
    if (start[a] != start[b]) return start[a] < start[b];
    if (tid[a] != tid[b]) return tid[a] < tid[b];
    if (jid[a] != jid[b]) return jid[a] < jid[b];
    return a < b;
  }
};

// key_at (may be null): the segment of every position
__global__ void seg_bounds_kernel(SortedKey key, int n, int32_t* seg_start, int32_t* seg_end, int32_t* key_at) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int k = mark_segment(p, n, key, seg_start, seg_end);
  if (key_at) key_at[p] = k;
}

// ---- order-wide scan, exact grid only: a running sum over one segment of a sorted order is ONE
// inclusive scan over the whole order minus the scan just before the segment's first position, so no
// segment, however long, sits on one warp.  Two launches: tile scans, then one warp turns the tile
// totals into exclusive offsets.  Both do nothing unless grid_exact(gf, n).
constexpr int OS_TB = 256, OS_IPT = 8, OS_TILE = OS_TB * OS_IPT;

template <class T, int K>
struct OrderScan {
  T* part[K];   // [n] inclusive sums inside the tile
  T* tile[K];   // [tiles] tile totals, then exclusive offsets
  __device__ T at(int k, int p) const { return part[k][p] + tile[k][p / OS_TILE]; }
  // column k summed over the positions s .. p
  __device__ T segment_sum(int k, int p, int s) const {
    T v = at(k, p);
    if (s > 0) v = v - at(k, s - 1);
    return v;
  }
};

// load(p, x) fills the zeroed addends of position p
template <class T, int K, class Load>
__global__ void __launch_bounds__(OS_TB) order_scan_tiles(OrderScan<T, K> os, Load load, int n, const GridFlag* gf) {
  if (!grid_exact(gf, n)) return;
  __shared__ T s_w[K][OS_TB / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int p0 = blockIdx.x * OS_TILE + threadIdx.x * OS_IPT;
  T x[OS_IPT][K];
#pragma unroll
  for (int j = 0; j < OS_IPT; j++) {
#pragma unroll
    for (int k = 0; k < K; k++) x[j][k] = T(0);
    if (p0 + j < n) load(p0 + j, x[j]);
  }
#pragma unroll
  for (int j = 1; j < OS_IPT; j++)
#pragma unroll
    for (int k = 0; k < K; k++) x[j][k] = x[j - 1][k] + x[j][k];
  T off[K];
#pragma unroll
  for (int k = 0; k < K; k++) {
    const T i = warp_incl_scan(x[OS_IPT - 1][k], lane);
    if (lane == 31) s_w[k][warp] = i;
    off[k] = i - x[OS_IPT - 1][k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; k++)
    for (int w = 0; w < warp; w++) off[k] = off[k] + s_w[k][w];
#pragma unroll
  for (int j = 0; j < OS_IPT; j++)
    if (p0 + j < n)
#pragma unroll
      for (int k = 0; k < K; k++) os.part[k][p0 + j] = off[k] + x[j][k];
  if (threadIdx.x == OS_TB - 1)
#pragma unroll
    for (int k = 0; k < K; k++) os.tile[k][blockIdx.x] = off[k] + x[OS_IPT - 1][k];
}

template <class T, int K>
__global__ void order_scan_totals(OrderScan<T, K> os, int nb, int n, const GridFlag* gf) {
  if (!grid_exact(gf, n)) return;
  const int lane = threadIdx.x;
  T carry[K];
#pragma unroll
  for (int k = 0; k < K; k++) carry[k] = T(0);
  for (int base = 0; base < nb; base += 32) {
    const int b = base + lane;
#pragma unroll
    for (int k = 0; k < K; k++) {
      const T x = b < nb ? os.tile[k][b] : T(0);
      const T i = carry[k] + warp_incl_scan(x, lane);
      if (b < nb) os.tile[k][b] = i - x;
      carry[k] = __shfl_sync(FULL_MASK, i, 31);
    }
  }
}

template <class T, int K, class Load>
inline void order_scan(const OrderScan<T, K>& os, const Load& load, int n, const GridFlag* gf, cudaStream_t st) {
  const int nb = (n + OS_TILE - 1) / OS_TILE;
  order_scan_tiles<<<nb, OS_TB, 0, st>>>(os, load, n, gf);
  order_scan_totals<<<1, 32, 0, st>>>(os, nb, n, gf);
}

// ---- stable stream compaction: the items i < n with f.keep(i) go, in order, to slots 0, 1, ... through
// f.emit(i, slot) for the slots below cap, and *out_n = min(count, cap).  n is *n_dev when that is given
// (a count only the device knows), at most n_max, which sizes the grid and blk[n_max / CP_BLOCK + 1].
// Three launches: per-block counts, one warp turns them into exclusive offsets, scatter.
constexpr int CP_TB = 256, CP_ITEMS = 4, CP_BLOCK = CP_TB * CP_ITEMS;

__device__ __forceinline__ int compact_n(const int32_t* n_dev, int n_max) { return n_dev ? min(*n_dev, n_max) : n_max; }

template <class F>
__global__ void __launch_bounds__(CP_TB) compact_count_kernel(F f, const int32_t* n_dev, int n_max, int32_t* blk) {
  __shared__ int warp_sums[CP_TB / 32];
  const int n = compact_n(n_dev, n_max);
  const int base = (blockIdx.x * CP_TB + threadIdx.x) * CP_ITEMS;
  int c = 0;
#pragma unroll
  for (int q = 0; q < CP_ITEMS; q++) c += (base + q < n && f.keep(base + q)) ? 1 : 0;
  c = __reduce_add_sync(FULL_MASK, c);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < CP_TB / 32; w++) t += warp_sums[w];
    blk[blockIdx.x] = t;
  }
}

__global__ void compact_scan_kernel(int32_t* blk, const int32_t* n_dev, int n_max, int32_t* out_n, int cap) {
  const int lane = threadIdx.x;
  const int nblk = (compact_n(n_dev, n_max) + CP_BLOCK - 1) / CP_BLOCK;
  int carry = 0;
  for (int base = 0; base < nblk; base += 32) {
    const int b = base + lane;
    const int v = b < nblk ? blk[b] : 0;
    const int incl = carry + warp_incl_scan(v, lane);
    if (b < nblk) blk[b] = incl - v;
    carry = __shfl_sync(FULL_MASK, incl, 31);
  }
  if (lane == 0) *out_n = min(carry, cap);
}

template <class F>
__global__ void __launch_bounds__(CP_TB) compact_scatter_kernel(F f, const int32_t* n_dev, int n_max, const int32_t* blk,
                                                               int cap) {
  __shared__ int warp_off[CP_TB / 32];
  const int n = compact_n(n_dev, n_max);
  const int base = (blockIdx.x * CP_TB + threadIdx.x) * CP_ITEMS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  bool on[CP_ITEMS];
  int c = 0;
#pragma unroll
  for (int q = 0; q < CP_ITEMS; q++) { on[q] = base + q < n && f.keep(base + q); c += on[q] ? 1 : 0; }
  const int incl = warp_incl_scan(c, lane);
  if (lane == 31) warp_off[warp] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < CP_TB / 32; w++) { const int x = warp_off[w]; warp_off[w] = t; t += x; }
  }
  __syncthreads();
  int slot = blk[blockIdx.x] + warp_off[warp] + incl - c;
#pragma unroll
  for (int q = 0; q < CP_ITEMS; q++)
    if (on[q]) {
      if (slot < cap) f.emit(base + q, slot);
      slot++;
    }
}

template <class F>
inline void compact(const F& f, int n_max, const int32_t* n_dev, int32_t* blk, int32_t* out_n, int cap, cudaStream_t st) {
  const int nb = (n_max + CP_BLOCK - 1) / CP_BLOCK;
  compact_count_kernel<<<nb, CP_TB, 0, st>>>(f, n_dev, n_max, blk);
  compact_scan_kernel<<<1, 32, 0, st>>>(blk, n_dev, n_max, out_n, cap);
  compact_scatter_kernel<<<nb, CP_TB, 0, st>>>(f, n_dev, n_max, blk, cap);
}

}  // namespace
