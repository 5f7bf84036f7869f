// Shared helpers for the det3d_b200 CUDA translation units (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <stdint.h>
#include <stdio.h>

#include "det3d_b200.h"

namespace d3b {

// ---- error plumbing --------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define D3B_REQUIRE(cond, ...)          \
  do {                                  \
    if (!(cond)) {                      \
      d3b::set_error(__VA_ARGS__);      \
      return D3B_ERR_INVALID_ARG;       \
    }                                   \
  } while (0)

#define D3B_CUDA(call)                                                              \
  do {                                                                              \
    cudaError_t e__ = (call);                                                       \
    if (e__ != cudaSuccess) {                                                       \
      d3b::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call,                   \
                     cudaGetErrorString(e__));                                      \
      return D3B_ERR_CUDA;                                                          \
    }                                                                               \
  } while (0)

#define D3B_LAUNCH_CHECK()                                                          \
  do {                                                                              \
    d3b::count_launch();                                                            \
    cudaError_t e__ = cudaGetLastError();                                           \
    if (e__ != cudaSuccess) {                                                       \
      d3b::set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__,               \
                     cudaGetErrorString(e__));                                      \
      return D3B_ERR_CUDA;                                                          \
    }                                                                               \
  } while (0)

// ---- > 48 KB dynamic shared memory opt-in ----------------------------------------
// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE function attribute: the opt-in is cached per device id
// (atomics: setting it twice from two threads is benign), never in a process-wide flag.
constexpr int kMaxDevices = 64;
struct SmemOptIn {
  std::atomic<int> bytes[kMaxDevices];
};
template <typename Kernel>
static inline cudaError_t ensure_dynamic_smem(Kernel kernel, size_t bytes, SmemOptIn& cache) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const bool cached = dev >= 0 && dev < kMaxDevices;
  if (cached && cache.bytes[dev].load(std::memory_order_acquire) >= (int)bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess && cached) cache.bytes[dev].store((int)bytes, std::memory_order_release);
  return e;
}

// nms.cu: `batch` box sets of one capacity in two launches (the detector's per-sample NMS); fmt_kernel 0 xyxyr (iou3d),
// 1 xywlr (rotate_nms_cc), 2 axis-aligned, 3 axis-aligned "+1", 4 RRPN.
int nms_batched(int fmt_kernel, const float* boxes, int n_cap, const int* n_dev, float thresh, int max_keep,
                long long* keep_idx, int* keep_count, void* workspace, size_t workspace_bytes, int batch, cudaStream_t stream);

// ---- programmatic dependent launch --------------------------------------------------------------------------------
// The convolution kernels run back to back on one stream.  Launched with programmatic stream serialisation, kernel N+1 is
// scheduled as soon as every CTA of kernel N has executed `griddepcontrol.launch_dependents` (they do so on entry): its
// launch latency and its prologue (barrier init, rulebook staging -- nothing that reads kernel N's
// output) overlap kernel N's tail; `griddepcontrol.wait` (executed by every thread before it touches activations) then
// blocks until kernel N has completed and its writes are visible.  Inside a captured CUDA graph the edge becomes a
// programmatic dependency.  d3b_set_pdl(0) turns it off (plain stream order).
bool pdl_enabled();
// bevconv16_sm90.cu: 0 = pixel-stationary tiles (two 128-pixel halves) everywhere, 2 = automatic = the pipelined kernel
// (16 x 8 pixel tiles, two partials in flight) for the 3x3 stride-1 128-channel-block layers and pixel-stationary for
// the rest, the fastest choice on the H100 (d3b_set_bev_variant)
int bev_variant();
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_maybe_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                           Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait_prior_grid() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- device constants --------------------------------------------------------
constexpr int kNumSMs = 132;  // H100 SXM

static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Grid for a grid-stride kernel over `n` items: enough CTAs to cover n but
// never more than `waves` full waves of the 132 SMs at `ctas_per_sm`.
static inline int grid_for(long long n, int block, int ctas_per_sm = 8) {
  long long want = (n + block - 1) / block;
  long long cap = (long long)kNumSMs * ctas_per_sm;
  if (want < 1) want = 1;
  return (int)(want < cap ? want : cap);
}

// 64-bit mix (splitmix64 finaliser) for the open-addressing tables.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebULL;
  x ^= x >> 31;
  return x;
}

constexpr unsigned long long kEmptyKey = ~0ULL;  // memset 0xff
constexpr int kSentinelMin = 0x7f000000;         // memset 0x7f -> 0x7f7f7f7f == "empty"

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

}  // namespace d3b
