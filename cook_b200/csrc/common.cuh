// common.cuh — handles, error plumbing and the device arena of libcookgpu.so.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
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
// upload.  Adds the uploaded bytes to *h2d.
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
  *h2d += c.h2d;
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
  cudaEvent_t ev[20] = {};
  cook_phase_stats phase[4] = {};        // last rank / match / rebalance / exchange call
  double* xchg = nullptr;                // exchange buffers: [n_pad] local + [world * n_pad] gathered
  size_t xchg_cap = 0;
  Arena arena;
  void* match_plan = nullptr;            // MatchPlan (match.cu), resident inputs
  void (*match_plan_free)(void*) = nullptr;
  char err[512] = {0};
};

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
