// Ordered compaction of one sample's result rows by one CTA, shared by the result-row kernels (kitti_results.cu,
// nusc_results.cu).  The CTA walks rows [0, D) in chunks of kThreads; row_fn(i, row) fills row[0, kCols) and returns
// whether row i is kept.  Kept rows are written to out in input order (ballot, per-warp counts in shared memory, a
// prefix over the warps), rows past the kept count are written as zeros, and the kept count is returned, the same in
// every thread.  warp_cnt is kThreads / 32 ints of shared memory.
#pragma once

namespace d3b {

template <int kThreads, int kCols, class RowFn>
__device__ __forceinline__ int compact_rows(int D, double* __restrict__ out, int* warp_cnt, RowFn row_fn) {
  static_assert(kThreads % 32 == 0, "whole warps");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int count = 0;                                    // kept rows so far, the same in every thread
  for (int base = 0; base < D; base += kThreads) {
    const int i = base + threadIdx.x;
    double row[kCols];
    const bool keep = i < D && row_fn(i, row);
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      const int n = warp_cnt[w];
      before += w < warp ? n : 0;
      total += n;
    }
    if (keep) {
      double* o = out + (size_t)(count + before + __popc(bal & ((1u << lane) - 1u))) * kCols;
#pragma unroll
      for (int j = 0; j < kCols; ++j) o[j] = row[j];
    }
    count += total;
    __syncthreads();                                // warp_cnt is rewritten by the next chunk
  }
  for (size_t j = (size_t)count * kCols + threadIdx.x; j < (size_t)D * kCols; j += kThreads) out[j] = 0.0;
  return count;
}

}  // namespace d3b
