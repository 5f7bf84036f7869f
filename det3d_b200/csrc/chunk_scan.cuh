// Block-wide scans shared by the order-preserving compactions of ingest.cu and frustum.cu: the clamp of a device offset
// table into a monotone prefix, and the one-CTA exclusive scan of per-chunk counts (count -> scan -> emit).
#pragma once
#include <climits>

#include "common.cuh"

namespace d3b {

// Inclusive block-wide scan of one value per thread (sum, or max with kMax); `total` = the whole block's.  Every thread
// of the block calls it; `buf` is 32 ints of shared memory, free again on return.
template <bool kMax>
__device__ __forceinline__ int block_scan(int v, int* buf, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v = kMax ? max(v, t) : v + t;
  }
  if (lane == 31) buf[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int w = lane < (int)(blockDim.x >> 5) ? buf[lane] : (kMax ? INT_MIN : 0);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w = kMax ? max(w, t) : w + t;
    }
    buf[lane] = w;
  }
  __syncthreads();
  if (warp > 0) v = kMax ? max(v, buf[warp - 1]) : v + buf[warp - 1];
  total = buf[31];
  __syncthreads();
  return v;
}

// dst[i] = min(max(0, raw(1..i)), cap) for i in [0, n] (dst[0] = 0): a table clamped into 0 = dst[0] <= ... <= dst[n]
// <= cap.  With `chunks`, also chunks[i] = sum over j in [1, i] of ceil((dst[j] - dst[j-1]) / kChunk).  Returns
// (per thread) whether an entry it handled changed.
template <int kChunk, class Raw>
__device__ __forceinline__ bool clamp_table(Raw raw, int n, int cap, int* dst, int* chunks, int* buf) {
  int run_max = 0, run_chunks = 0;
  bool bad = false;
  for (int base = 0; base <= n; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int r = i <= n ? raw(i) : 0;
    int total;
    const int m = max(block_scan<true>(i == 0 ? 0 : (i <= n ? r : INT_MIN), buf, total), run_max);
    run_max = max(run_max, total);
    const int c = min(m, cap);
    bad |= i <= n && c != r;
    if (i <= n) dst[i] = c;
    if (chunks != nullptr) {
      __syncthreads();
      const int k = (i == 0 || i > n) ? 0 : (c - dst[i - 1] + kChunk - 1) / kChunk;
      const int incl = block_scan<false>(k, buf, total) + run_chunks;
      run_chunks += total;
      if (i <= n) chunks[i] = incl;
    }
  }
  return bad;
}

// One CTA: chunk_base[g] = exclusive prefix of chunk_cnt[0..n_chunks) for every g; returns the total to every thread.
// `warp_sums` is 32 ints and `running` one int of shared memory.
__device__ __forceinline__ int scan_chunk_counts(const int* __restrict__ chunk_cnt, int n_chunks, int* chunk_base,
                                                 int* warp_sums, int& running) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  for (int base = 0; base < n_chunks; base += blockDim.x) {
    const int g = base + threadIdx.x;
    const int v = g < n_chunks ? chunk_cnt[g] : 0;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = warp_sums[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += t;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    if (g < n_chunks) chunk_base[g] = running + (warp == 0 ? 0 : warp_sums[warp - 1]) + incl - v;
    const int total = warp_sums[31];
    __syncthreads();
    if (threadIdx.x == 0) running += total;
    __syncthreads();
  }
  return running;
}

}  // namespace d3b
