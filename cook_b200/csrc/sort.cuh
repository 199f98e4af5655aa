// sort.cuh — comparator-driven index sort (hand-written; no CUB).
//
// Sorts an array of int32 indices under an arbitrary strict-weak `Less`
// functor evaluated on the device.  Used for (a) the per-user task order
// (tools.clj:614-641 feature-vector compare) and (b) the global DRU order with
// the dynamic k-way-merge tie rule (dru.clj:82-104), neither of which maps to a
// fixed-width radix key.
//
//   1. tile sort : one CTA bitonic-sorts TILE indices in shared memory
//   2. merge     : log2(n/TILE) passes; every thread finds its merge-path
//                  split by binary search and emits ITEMS outputs (stable:
//                  left run wins ties).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace csort {

constexpr int TILE = 2048;        // indices per CTA in the tile sort
constexpr int TILE_THREADS = 512; // 4 per thread
constexpr int ITEMS = 8;          // outputs per thread in a merge pass

template <class Less>
__global__ void __launch_bounds__(TILE_THREADS) tile_sort_kernel(int32_t* __restrict__ idx, int n,
                                                                  Less less) {
  __shared__ int32_t s[TILE];
  const int base = blockIdx.x * TILE;
  for (int i = threadIdx.x; i < TILE; i += TILE_THREADS) {
    int g = base + i;
    s[i] = g < n ? g : -1;  // the identity; -1 = +inf padding
  }
  __syncthreads();
  auto lt = [&](int32_t a, int32_t b) {
    if (a < 0) return false;
    if (b < 0) return true;
    return less(a, b);
  };
  for (int k = 2; k <= TILE; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < TILE / 2; t += TILE_THREADS) {
        int i = 2 * t - (t & (j - 1));  // lower index of the pair
        int p = i + j;
        bool up = ((i & k) == 0);
        int32_t a = s[i], b = s[p];
        bool swap = up ? lt(b, a) : lt(a, b);
        if (swap) { s[i] = b; s[p] = a; }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < TILE; i += TILE_THREADS) {
    int g = base + i;
    if (g < n) idx[g] = s[i];
  }
}

// Merge pass: runs of `width` from src are merged pairwise into dst.
template <class Less>
__global__ void merge_pass_kernel(const int32_t* __restrict__ src, int32_t* __restrict__ dst,
                                  int n, int width, Less less) {
  const long long out0 = (long long)(blockIdx.x * (long long)blockDim.x + threadIdx.x) * ITEMS;
  if (out0 >= n) return;
  const long long pair = out0 / (2LL * width);
  const int a0 = (int)(pair * 2LL * width);
  const int a1 = min(a0 + width, n);
  const int b0 = a1;
  const int b1 = min(a0 + 2 * width, n);
  const int la = a1 - a0, lb = b1 - b0;
  const int diag = (int)(out0 - a0);  // outputs of this pair before mine
  // merge path: find i in [max(0,diag-lb), min(diag,la)] s.t. A[i-1] <= B[diag-i] and B[diag-i-1] < A[i]
  int lo = max(0, diag - lb), hi = min(diag, la);
  while (lo < hi) {
    int i = (lo + hi) >> 1;
    int j = diag - i;
    // if B[j-1] < A[i] is false (A[i] <= B[j-1]) we need more from A
    if (!less(src[b0 + j - 1], src[a0 + i]))
      lo = i + 1;
    else
      hi = i;
  }
  int i = lo, j = diag - lo;
  const int cnt = min(ITEMS, (int)(min((long long)n, (long long)a0 + la + lb) - out0));
  for (int k = 0; k < cnt; k++) {
    bool takeA;
    if (i >= la) takeA = false;
    else if (j >= lb) takeA = true;
    else takeA = !less(src[b0 + j], src[a0 + i]);  // stable: A wins ties
    dst[out0 + k] = takeA ? src[a0 + i++] : src[b0 + j++];
  }
}

// Sorts the indices 0..n-1 into idx[0..n); tmp must hold n int32.  Adds its kernel launches to *launches.
template <class Less>
inline cudaError_t sort_indices(int32_t* idx, int32_t* tmp, int n, Less less, cudaStream_t st, int* launches) {
  if (n <= 0) return cudaSuccess;
  int tiles = (n + TILE - 1) / TILE;
  tile_sort_kernel<Less><<<tiles, TILE_THREADS, 0, st>>>(idx, n, less);
  ++*launches;
  int32_t* src = idx;
  int32_t* dst = tmp;
  for (long long width = TILE; width < n; width <<= 1) {
    long long threads = ((long long)n + ITEMS - 1) / ITEMS;
    int blocks = (int)((threads + 255) / 256);
    merge_pass_kernel<Less><<<blocks, 256, 0, st>>>(src, dst, n, (int)width, less);
    ++*launches;
    int32_t* t = src; src = dst; dst = t;
  }
  if (src != idx)
    return cudaMemcpyAsync(idx, src, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToDevice, st);
  return cudaGetLastError();
}

}  // namespace csort
