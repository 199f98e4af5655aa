// fold_probe.cu — test-only harness: drives each primitive of cook_b200/csrc/fold.cuh with host inputs.
//
// Built by __graft_entry__.build() into tests/libfoldprobe.so with the product's nvcc flags and loaded by
// tests/test_fold_primitives.py.  Every entry point copies its host inputs to the device, runs the
// primitive exactly as the product kernels do, copies the outputs back and returns a cudaError_t
// (0 = success).  Device buffers are sized from the host arguments, so no call reads or writes past them.
#include "../cook_b200/csrc/fold.cuh"

namespace {

constexpr int PB_WARPS = 4;   // warps per block; one warp per segment

struct Bufs {   // device allocations of one call, freed on every return path
  std::vector<void*> p;
  cudaError_t err = cudaSuccess;
  template <class T>
  T* alloc(size_t n) {
    void* d = nullptr;
    if (err == cudaSuccess) err = cudaMalloc(&d, (n ? n : 1) * sizeof(T));
    if (d) p.push_back(d);
    return static_cast<T*>(d);
  }
  template <class T>
  T* upload(const T* h, size_t n) {
    T* d = alloc<T>(n);
    if (err == cudaSuccess && n) err = cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice);
    return d;
  }
  template <class T>
  void download(T* h, const T* d, size_t n) {
    if (err == cudaSuccess && n) err = cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost);
  }
  cudaError_t finish() {
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    return err;
  }
  ~Bufs() {
    for (void* d : p) cudaFree(d);
  }
};

// ---- warp_fold_prefix<K>: segment g is x[off[g] .. off[g+1]) of every column, folded in chunks of 32
// from start[g][k].  Lanes at or past a chunk's count hold `pad` (the primitive must ignore them).
template <int K>
__global__ void prefix_kernel(const double* x, int n, const int* off, int nseg, const double* start, bool exact,
                              double pad, double* out, double* carry_out) {
  __shared__ double stage[PB_WARPS][K][32];
  const int g = blockIdx.x * PB_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (g >= nseg) return;
  const int s = off[g], e = off[g + 1];
  double carry[K];
#pragma unroll
  for (int k = 0; k < K; k++) carry[k] = start[g * K + k];
  for (int base = s; base < e; base += 32) {
    const int i = base + lane, cnt = min(32, e - base);
    double v[K];
#pragma unroll
    for (int k = 0; k < K; k++) v[k] = i < e ? x[(size_t)k * n + i] : pad;
    warp_fold_prefix(v, carry, cnt, exact, stage[threadIdx.x >> 5]);
    if (i < e)
#pragma unroll
      for (int k = 0; k < K; k++) out[(size_t)k * n + i] = v[k];
  }
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; k++) carry_out[g * K + k] = carry[k];
}

// ---- warp_fold_sum<K, D>: items off[g] .. off[g+1] of segment g; item i takes part when on[i], and one
// that does not leaves its addends zero
template <int K, int D>
__global__ void sum_kernel(const double* x, int n, const uint8_t* on, const int* off, int nseg, const double* start,
                           bool exact, double* carry_out) {
  __shared__ double stage[PB_WARPS][K][32];
  const int g = blockIdx.x * PB_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (g >= nseg) return;
  const int s = off[g], e = off[g + 1];
  double carry[K];
#pragma unroll
  for (int k = 0; k < K; k++) carry[k] = start[g * K + k];
  warp_fold_sum<K, D>(carry, e - s, exact, [&](int i, double (&v)[K]) {
    if (!on[s + i]) return false;
#pragma unroll
    for (int k = 0; k < K; k++) v[k] = x[(size_t)k * n + s + i];
    return true;
  }, stage[threadIdx.x >> 5]);
  // every lane must hold the total: lane l writes its own copy
#pragma unroll
  for (int k = 0; k < K; k++) carry_out[((size_t)g * K + k) * 32 + lane] = carry[k];
}

// ---- order_scan
template <class T, int K>
struct LoadCols {
  const T* x; int n;
  __device__ void operator()(int p, T (&v)[K]) const {
#pragma unroll
    for (int k = 0; k < K; k++) v[k] = x[(size_t)k * n + p];
  }
};

template <class T, int K>
__global__ void scan_read_kernel(OrderScan<T, K> os, int n, const int* qp, const int* qs, int nq, T* at, T* seg) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
#pragma unroll
    for (int k = 0; k < K; k++) at[(size_t)k * n + i] = os.at(k, i);
  if (i < nq)
#pragma unroll
    for (int k = 0; k < K; k++) seg[(size_t)k * nq + i] = os.segment_sum(k, qp[i], qs[i]);
}

// part / tile come in pre-filled (a sentinel survives when the grid gate is closed); at / seg are read
// back only when `read` is set, since at() of a closed gate adds sentinels.
template <class T, int K>
cudaError_t run_order_scan(const T* x, int n, int bad, unsigned long long max_bits, const int* qp, const int* qs, int nq,
                           int read, T* part, T* tile, T* at, T* seg) {
  Bufs b;
  const int nb = (n + OS_TILE - 1) / OS_TILE;
  const T* d_x = b.upload(x, (size_t)K * n);
  T* d_part = b.upload(part, (size_t)K * n);
  T* d_tile = b.upload(tile, (size_t)K * nb);
  const GridFlag hf{bad, max_bits};
  const GridFlag* d_gf = b.upload(&hf, 1);
  const int* d_qp = b.upload(qp, nq);
  const int* d_qs = b.upload(qs, nq);
  T* d_at = b.alloc<T>((size_t)K * n);
  T* d_seg = b.alloc<T>((size_t)K * nq);
  if (b.err != cudaSuccess) return b.err;
  OrderScan<T, K> os;
  for (int k = 0; k < K; k++) {
    os.part[k] = d_part + (size_t)k * n;
    os.tile[k] = d_tile + (size_t)k * nb;
  }
  order_scan(os, LoadCols<T, K>{d_x, n}, n, d_gf, 0);
  if (read) {
    const int m = max(n, nq);
    scan_read_kernel<<<(m + 255) / 256, 256>>>(os, n, d_qp, d_qs, nq, d_at, d_seg);
  }
  b.download(part, d_part, (size_t)K * n);
  b.download(tile, d_tile, (size_t)K * nb);
  if (read) {
    b.download(at, d_at, (size_t)K * n);
    b.download(seg, d_seg, (size_t)K * nq);
  }
  return b.finish();
}

__global__ void grid_query_kernel(const GridFlag* f, const long long* qn, const double* qstart, int nq, uint8_t* ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq) ok[i] = grid_exact(f, qn[i], qstart[i]) ? 1 : 0;
}

__global__ void value_ok_kernel(const double* x, int n, uint8_t* ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ok[i] = grid_value_ok(x[i]) ? 1 : 0;
}

// ---- compact: keep[i] from the host, emit writes item i to slot
struct KeepEmit {
  const uint8_t* flag; int32_t* out;
  __device__ bool keep(int i) const { return flag[i] != 0; }
  __device__ void emit(int i, int slot) const { out[slot] = i; }
};

}  // namespace

extern "C" {

// x: [K][n] column-major by column; off: [nseg + 1]; start, carry_out: [nseg][K]; out: [K][n]
int fp_warp_fold_prefix(int K, const double* x, int n, const int* off, int nseg, const double* start, int exact,
                        double pad, double* out, double* carry_out) {
  if (K < 1 || K > 4 || nseg < 1) return (int)cudaErrorInvalidValue;
  Bufs b;
  const double* d_x = b.upload(x, (size_t)K * n);
  const int* d_off = b.upload(off, nseg + 1);
  const double* d_start = b.upload(start, (size_t)nseg * K);
  double* d_out = b.upload(out, (size_t)K * n);
  double* d_carry = b.alloc<double>((size_t)nseg * K);
  if (b.err != cudaSuccess) return b.err;
  const int grid = (nseg + PB_WARPS - 1) / PB_WARPS, tb = 32 * PB_WARPS;
  switch (K) {
    case 1: prefix_kernel<1><<<grid, tb>>>(d_x, n, d_off, nseg, d_start, exact != 0, pad, d_out, d_carry); break;
    case 2: prefix_kernel<2><<<grid, tb>>>(d_x, n, d_off, nseg, d_start, exact != 0, pad, d_out, d_carry); break;
    case 3: prefix_kernel<3><<<grid, tb>>>(d_x, n, d_off, nseg, d_start, exact != 0, pad, d_out, d_carry); break;
    case 4: prefix_kernel<4><<<grid, tb>>>(d_x, n, d_off, nseg, d_start, exact != 0, pad, d_out, d_carry); break;
  }
  b.download(out, d_out, (size_t)K * n);
  b.download(carry_out, d_carry, (size_t)nseg * K);
  return b.finish();
}

// on: [n] participation; carry_out: [nseg][K][32], the total as every lane of the warp holds it
int fp_warp_fold_sum(int K, int D, const double* x, const uint8_t* on, int n, const int* off, int nseg,
                     const double* start, int exact, double* carry_out) {
  if (K < 1 || K > 4 || (D != 1 && D != 4) || nseg < 1) return (int)cudaErrorInvalidValue;
  Bufs b;
  const double* d_x = b.upload(x, (size_t)K * n);
  const uint8_t* d_on = b.upload(on, n);
  const int* d_off = b.upload(off, nseg + 1);
  const double* d_start = b.upload(start, (size_t)nseg * K);
  double* d_carry = b.alloc<double>((size_t)nseg * K * 32);
  if (b.err != cudaSuccess) return b.err;
  const int grid = (nseg + PB_WARPS - 1) / PB_WARPS, tb = 32 * PB_WARPS;
  const bool ex = exact != 0;
#define FP_SUM(KK, DD) sum_kernel<KK, DD><<<grid, tb>>>(d_x, n, d_on, d_off, nseg, d_start, ex, d_carry)
  switch (K * 10 + D) {
    case 11: FP_SUM(1, 1); break;
    case 14: FP_SUM(1, 4); break;
    case 21: FP_SUM(2, 1); break;
    case 24: FP_SUM(2, 4); break;
    case 31: FP_SUM(3, 1); break;
    case 34: FP_SUM(3, 4); break;
    case 41: FP_SUM(4, 1); break;
    case 44: FP_SUM(4, 4); break;
  }
#undef FP_SUM
  b.download(carry_out, d_carry, (size_t)nseg * K * 32);
  return b.finish();
}

// order_scan<double, 3>: x, part, at: [3][n]; tile: [3][tiles]; seg: [3][nq] = segment_sum(k, qp, qs)
int fp_order_scan_f64(const double* x, int n, int bad, unsigned long long max_bits, const int* qp, const int* qs,
                      int nq, int read, double* part, double* tile, double* at, double* seg) {
  if (n < 1) return (int)cudaErrorInvalidValue;
  return run_order_scan<double, 3>(x, n, bad, max_bits, qp, qs, nq, read, part, tile, at, seg);
}

// order_scan<int, 1>
int fp_order_scan_i32(const int* x, int n, int bad, unsigned long long max_bits, const int* qp, const int* qs, int nq,
                      int read, int* part, int* tile, int* at, int* seg) {
  if (n < 1) return (int)cudaErrorInvalidValue;
  return run_order_scan<int, 1>(x, n, bad, max_bits, qp, qs, nq, read, part, tile, at, seg);
}

int fp_order_scan_tile() { return OS_TILE; }
int fp_compact_block() { return CP_BLOCK; }

// grid_check_kernel over columns a, b, c (each may be NULL) into a zeroed flag, then grid_exact(flag, qn, qstart)
int fp_grid_check(const double* a, const double* b_, const double* c, int n, const long long* qn, const double* qstart,
                  int nq, int* bad_out, unsigned long long* max_bits_out, uint8_t* ok_out) {
  Bufs b;
  const double* d_a = a ? b.upload(a, n) : nullptr;
  const double* d_b = b_ ? b.upload(b_, n) : nullptr;
  const double* d_c = c ? b.upload(c, n) : nullptr;
  const GridFlag zero{0, 0ull};
  GridFlag* d_gf = b.upload(&zero, 1);
  const long long* d_qn = b.upload(qn, nq);
  const double* d_qs = b.upload(qstart, nq);
  uint8_t* d_ok = b.alloc<uint8_t>(nq);
  if (b.err != cudaSuccess) return b.err;
  if (n > 0) grid_check_kernel<<<(n + 255) / 256, 256>>>(d_a, d_b, d_c, n, d_gf);
  if (nq > 0) grid_query_kernel<<<(nq + 255) / 256, 256>>>(d_gf, d_qn, d_qs, nq, d_ok);
  GridFlag hf{};
  b.download(&hf, d_gf, 1);
  b.download(ok_out, d_ok, nq);
  const cudaError_t e = b.finish();
  *bad_out = hf.bad;
  *max_bits_out = hf.max_bits;
  return e;
}

int fp_grid_value_ok(const double* x, int n, uint8_t* ok_out) {
  if (n < 1) return (int)cudaErrorInvalidValue;
  Bufs b;
  const double* d_x = b.upload(x, n);
  uint8_t* d_ok = b.alloc<uint8_t>(n);
  if (b.err != cudaSuccess) return b.err;
  value_ok_kernel<<<(n + 255) / 256, 256>>>(d_x, n, d_ok);
  b.download(ok_out, d_ok, n);
  return b.finish();
}

// seg_bounds_kernel over key[map[ord[p]]] (map may be NULL); seg_start / seg_end come in pre-filled with
// a sentinel and are [nseg]; every key must lie in [0, nseg)
int fp_seg_bounds(const int* ord, const int* map, int n_map, const int* key, int n_key, int n, int nseg,
                  int* seg_start, int* seg_end, int* key_at) {
  if (n < 1 || nseg < 1) return (int)cudaErrorInvalidValue;
  Bufs b;
  const int* d_ord = b.upload(ord, n);
  const int* d_map = map ? b.upload(map, n_map) : nullptr;
  const int* d_key = b.upload(key, n_key);
  int* d_s = b.upload(seg_start, nseg);
  int* d_e = b.upload(seg_end, nseg);
  int* d_at = b.alloc<int>(n);
  if (b.err != cudaSuccess) return b.err;
  seg_bounds_kernel<<<(n + 255) / 256, 256>>>(SortedKey{d_ord, d_map, d_key}, n, d_s, d_e, d_at);
  b.download(seg_start, d_s, nseg);
  b.download(seg_end, d_e, nseg);
  b.download(key_at, d_at, n);
  return b.finish();
}

// compact over keep[0 .. n_max), n read from the device when n_dev >= 0; out: [out_len] pre-filled with a
// sentinel, out_len >= cap (slots past cap must survive)
int fp_compact(const uint8_t* keep, int n_max, int n_dev, int cap, int* out, int out_len, int* out_n) {
  if (n_max < 1 || cap < 0 || out_len < cap) return (int)cudaErrorInvalidValue;
  Bufs b;
  const uint8_t* d_keep = b.upload(keep, n_max);
  int* d_out = b.upload(out, out_len);
  const int* d_n = n_dev >= 0 ? b.upload(&n_dev, 1) : nullptr;
  int* d_blk = b.alloc<int>(n_max / CP_BLOCK + 1);
  int* d_outn = b.alloc<int>(1);
  if (b.err != cudaSuccess) return b.err;
  compact(KeepEmit{d_keep, d_out}, n_max, d_n, d_blk, d_outn, cap, 0);
  b.download(out, d_out, out_len);
  b.download(out_n, d_outn, 1);
  return b.finish();
}

}  // extern "C"
