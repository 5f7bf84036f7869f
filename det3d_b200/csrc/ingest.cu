// nuScenes-style multi-sweep ingest on the device (SURVEY 8f.4): the raw sweeps of a sample -> one cloud
// [N, n_feat + 1] = (x, y, z, intensity.., time lag), ready for d3b_voxelize.
//
// Reference semantics, det3d/datasets/pipelines/loading.py:
//   read_file   :17-31   raw file = float32 [n, 5], the first n_feat (4) columns are kept
//   remove_close:34-43   sweeps only: drop points with |x| < radius AND |y| < radius (in the sweep's own frame)
//   read_sweep  :46-64   xyz <- (transform_matrix . [x y z 1]^T)[:3] -- float64 matrix times float64-promoted
//                         points, rounded once into the float32 array; time column = time_lag
//   __call__    :98-124  key frame first (no filter, no transform, time 0), then the chosen sweeps in order;
//                         np.concatenate keeps every sweep's point order
// The order-preserving compaction is a chunked scan (1024-point chunks: count -> scan of chunk counts -> emit).
//
// Sweep tables: d3b_ingest_sweeps takes one sample's table on the host (in the by-value params), d3b_ingest_sweeps_dev
// takes a batch of samples' tables from device memory, so one captured CUDA graph serves sweeps of any size up to a raw
// capacity.  Both run the same three kernels.  Every CTA first copies the sweep offsets, the samples' sweep ranges and
// the chunk prefix of the sweeps into shared memory (load_table); device tables are clamped there, the same way in every
// CTA, before any point index is formed.  Chunks never straddle a sweep, so a CTA stages its sweep's transform once, and
// one scan over the whole batch gives both the output rows and the per-sample cloud offsets.
//
// d3b_ingest_sweeps_gather adds one device array, sweep_src: the raw row where each sweep starts, so sweeps can be read
// from wherever they sit (a ring of history slots) while sweep_offsets stays the logical prefix that drives the chunks,
// the scan and the cloud offsets.  Without it the start of sweep s is its offset, which is the other two entry points.
#include <climits>

#include "common.cuh"

namespace d3b {
namespace {

constexpr int kIngestChunk = 1024;
constexpr int kIngestMaxBatch = 64;
constexpr int kIngestMaxTable = kIngestMaxBatch * D3B_INGEST_MAX_SWEEPS;   // sweeps of one device table
constexpr unsigned kHasTransform = 1u, kFilterClose = 2u;                   // device table flags

struct IngestParams {
  int n_sweeps;                                 // host table: the sample's sweeps; device table: its capacity
  int batch;                                    // samples (1 for the host table)
  int raw_stride, n_feat;
  int raw_cap;                                  // sweep offsets are clamped to this many raw rows
  float radius;
  // host table (d3b_ingest_sweeps)
  int off[D3B_INGEST_MAX_SWEEPS + 1];           // raw point offsets of the sweeps
  double m[D3B_INGEST_MAX_SWEEPS][12];          // rows 0..2 of the 4x4 transform
  float time_lag[D3B_INGEST_MAX_SWEEPS];
  unsigned char flags[D3B_INGEST_MAX_SWEEPS];   // kHasTransform | kFilterClose
  // device table (d3b_ingest_sweeps_dev), else nullptr
  const int* off_dev;
  const int* sample_dev;
  const int* src_dev;                           // d3b_ingest_sweeps_gather only: raw row where each sweep starts
  const double* m_dev;                          // [n_sweeps][16]
  const float* lag_dev;
  const unsigned char* flags_dev;
};

// Per-CTA copy of the clamped table.
struct IngestTable {
  int off[kIngestMaxTable + 1];                 // logical prefix of the sweeps' lengths
  int src[kIngestMaxTable];                     // raw row where each sweep starts (off[s] unless gathered)
  int chunk_off[kIngestMaxTable + 1];           // prefix of the sweeps' chunk counts
  int sample[kIngestMaxBatch + 1];              // sample b owns sweeps [sample[b], sample[b + 1])
  int buf[32];                                  // block-scan scratch
};

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
// <= cap.  With `chunks`, also chunks[i] = sum over j in [1, i] of ceil((dst[j] - dst[j-1]) / kIngestChunk).  Returns
// (per thread) whether an entry it handled changed.
template <class Raw>
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
      const int k = (i == 0 || i > n) ? 0 : (c - dst[i - 1] + kIngestChunk - 1) / kIngestChunk;
      const int incl = block_scan<false>(k, buf, total) + run_chunks;
      run_chunks += total;
      if (i <= n) chunks[i] = incl;
    }
  }
  return bad;
}

constexpr int kClampedTable = 1, kClampedSrc = 2;   // status bits

// Fills `t` from the params (host table) or from device memory (device table, clamped).  Returns, to every thread after
// the barrier, which clamps changed anything (kClampedTable | kClampedSrc).
__device__ __forceinline__ int load_table(const IngestParams& p, IngestTable& t) {
  bool bad = clamp_table([&](int i) { return p.off_dev != nullptr ? __ldg(p.off_dev + i) : p.off[i]; },
                         p.n_sweeps, p.raw_cap, t.off, t.chunk_off, t.buf);
  bad |= clamp_table([&](int b) { return p.sample_dev != nullptr ? __ldg(p.sample_dev + b) : (b == 0 ? 0 : p.n_sweeps); },
                     p.batch, p.n_sweeps, t.sample, nullptr, t.buf);
  // t.off is complete here (the scans above passed barriers after writing it).  A gathered start is clamped into
  // [0, raw_cap - len]; without sweep_src the start is the offset itself, which is always inside.
  bool bad_src = false;
  for (int s = threadIdx.x; s < p.n_sweeps; s += blockDim.x) {
    const int off = t.off[s];
    if (p.src_dev != nullptr) {
      const int r = __ldg(p.src_dev + s), c = min(max(r, 0), p.raw_cap - (t.off[s + 1] - off));
      bad_src |= c != r;
      t.src[s] = c;
    } else {
      t.src[s] = off;
    }
  }
  const int clamped = __syncthreads_or(bad) != 0 ? kClampedTable : 0;
  return clamped | (__syncthreads_or(bad_src) != 0 ? kClampedSrc : 0);
}

// Chunks of the live sweeps (those of samples 0..batch-1); the rest of a capacity-sized grid returns.
__device__ __forceinline__ int live_chunks(const IngestParams& p, const IngestTable& t) {
  return t.chunk_off[t.sample[p.batch]];
}

// The sweep that owns chunk g < live_chunks: the last s with chunk_off[s] <= g (so never an empty sweep).
__device__ __forceinline__ int sweep_of_chunk(const IngestParams& p, const IngestTable& t, int g) {
  int lo = 0, hi = p.n_sweeps - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.chunk_off[mid] <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ unsigned sweep_flags(const IngestParams& p, int s) {
  return p.flags_dev != nullptr ? __ldg(p.flags_dev + s) : p.flags[s];
}

// ---- the per-point work, shared by both entry points -------------------------------------------------------------
__device__ __forceinline__ bool keeps(const float* __restrict__ q, bool filter_close, float radius) {
  return !(filter_close && fabsf(q[0]) < radius && fabsf(q[1]) < radius);                      // :39-41
}

__device__ __forceinline__ void ingest_point(const float* __restrict__ q, float* __restrict__ o, bool has_transform,
                                             const double* m, float lag, int n_feat) {
  if (has_transform) {
    // float64 row . [x y z 1], terms added in index order like a plain dot product, one rounding to fp32 (:55-58)
    const double x = (double)q[0], y = (double)q[1], z = (double)q[2];
#pragma unroll
    for (int c = 0; c < 3; ++c)
      o[c] = (float)(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[4 * c], x), __dmul_rn(m[4 * c + 1], y)),
                                          __dmul_rn(m[4 * c + 2], z)), m[4 * c + 3]));
  } else {
    o[0] = q[0]; o[1] = q[1]; o[2] = q[2];
  }
  for (int c = 3; c < n_feat; ++c) o[c] = q[c];
  o[n_feat] = lag;
}

// ---- count -> scan -> emit -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ingest_count(const IngestParams p, const float* __restrict__ raw, int* __restrict__ chunk_cnt) {
  __shared__ IngestTable t;
  load_table(p, t);
  const int g = blockIdx.x;
  if (g >= live_chunks(p, t)) return;           // d3b_ingest_sweeps_dev: grid sized for the capacity
  const int s = sweep_of_chunk(p, t, g);
  const bool filter = (sweep_flags(p, s) & kFilterClose) != 0;
  const int i0 = t.src[s] + (g - t.chunk_off[s]) * kIngestChunk + threadIdx.x * 4, end = t.src[s] + t.off[s + 1] - t.off[s];
  int local = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (i0 + j < end) local += keeps(raw + (size_t)(i0 + j) * p.raw_stride, filter, p.radius) ? 1 : 0;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) local += __shfl_xor_sync(0xffffffffu, local, d);
  if ((threadIdx.x & 31) == 0) t.buf[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    int n = 0;
    for (int w = 0; w < 8; ++w) n += t.buf[w];
    chunk_cnt[g] = n;
  }
}

// One CTA: exclusive scan of the live chunk counts -> chunk_base; then the kept total (n_out, host table) or the
// per-sample cloud offsets (device table: sample b starts at the base of its first sweep's first chunk).
__global__ void __launch_bounds__(1024)
ingest_scan(const IngestParams p, const int* __restrict__ chunk_cnt, int* chunk_base, int* __restrict__ n_out,
            int out_cap, int* __restrict__ cloud_offsets, int* __restrict__ status) {
  __shared__ IngestTable t;
  __shared__ int running;
  const int clamped = load_table(p, t);
  const int n_chunks = live_chunks(p, t);
  int* warp_sums = t.buf;
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
  if (threadIdx.x == 0) {
    if (n_out != nullptr) *n_out = running < out_cap ? running : out_cap;
    if (status != nullptr) *status = clamped;
  }
  if (cloud_offsets != nullptr)
    for (int b = threadIdx.x; b <= p.batch; b += blockDim.x) {
      const int g = t.chunk_off[t.sample[b]];
      cloud_offsets[b] = g < n_chunks ? chunk_base[g] : running;
    }
}

__global__ void __launch_bounds__(256)
ingest_emit(const IngestParams p, const float* __restrict__ raw, const int* __restrict__ chunk_base,
            float* __restrict__ out, int out_cap) {
  __shared__ IngestTable t;
  __shared__ double m[12];
  load_table(p, t);
  const int g = blockIdx.x;
  if (g >= live_chunks(p, t)) return;           // d3b_ingest_sweeps_dev: grid sized for the capacity
  const int s = sweep_of_chunk(p, t, g);
  if (threadIdx.x < 12)
    m[threadIdx.x] = p.m_dev != nullptr ? __ldg(p.m_dev + (size_t)s * 16 + threadIdx.x) : p.m[s][threadIdx.x];
  const unsigned flags = sweep_flags(p, s);
  const float lag = p.lag_dev != nullptr ? __ldg(p.lag_dev + s) : p.time_lag[s];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i0 = t.src[s] + (g - t.chunk_off[s]) * kIngestChunk + threadIdx.x * 4, end = t.src[s] + t.off[s + 1] - t.off[s];
  unsigned int kept = 0u;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (i0 + j < end && keeps(raw + (size_t)(i0 + j) * p.raw_stride, (flags & kFilterClose) != 0, p.radius))
      kept |= 1u << j;
  const int local = __popc(kept);
  int incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) t.buf[warp] = incl;
  __syncthreads();                              // also publishes m
  int warp_off = 0;
  for (int w = 0; w < warp; ++w) warp_off += t.buf[w];
  int r = chunk_base[g] + warp_off + incl - local;
  const int width = p.n_feat + 1;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (!((kept >> j) & 1u)) continue;
    if (r < out_cap)
      ingest_point(raw + (size_t)(i0 + j) * p.raw_stride, out + (size_t)r * width, (flags & kHasTransform) != 0, m, lag,
                   p.n_feat);
    ++r;
  }
}

IngestParams params_of(int n_sweeps, int batch, int raw_stride, int n_feat, float radius) {
  IngestParams p = {};
  p.n_sweeps = n_sweeps; p.batch = batch; p.raw_stride = raw_stride; p.n_feat = n_feat; p.radius = radius;
  return p;
}

int launch_ingest(const IngestParams& p, const float* raw, int n_chunks, float* out, int out_cap, int* n_out,
                  int* cloud_offsets, int* status, int* chunk_cnt, int* chunk_base, cudaStream_t stream) {
  ingest_count<<<n_chunks, 256, 0, stream>>>(p, raw, chunk_cnt);
  D3B_LAUNCH_CHECK();
  ingest_scan<<<1, 1024, 0, stream>>>(p, chunk_cnt, chunk_base, n_out, out_cap, cloud_offsets, status);
  D3B_LAUNCH_CHECK();
  ingest_emit<<<n_chunks, 256, 0, stream>>>(p, raw, chunk_base, out, out_cap);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

}  // namespace
}  // namespace d3b

using namespace d3b;

// Chunks never straddle a sweep: at most n / kIngestChunk + (sweeps) of them.
extern "C" size_t d3b_ingest_workspace_bytes(int32_t n_points_total) {
  if (n_points_total < 0) return 0;
  return align_up(((size_t)n_points_total / kIngestChunk + D3B_INGEST_MAX_SWEEPS + 1) * 4) * 2;
}

extern "C" size_t d3b_ingest_dev_workspace_bytes(int32_t raw_capacity, int32_t sweep_capacity) {
  if (raw_capacity < 0 || sweep_capacity < 1) return 0;
  return align_up(((size_t)div_up(raw_capacity, kIngestChunk) + sweep_capacity) * 4) * 2;
}

extern "C" int d3b_ingest_sweeps(const float* raw, const int32_t* sweep_offsets, int32_t n_sweeps, int32_t raw_stride,
                                 int32_t n_feat, const double* transforms, const uint8_t* has_transform,
                                 const float* time_lag, const uint8_t* filter_close, float radius, float* out,
                                 int32_t out_cap, int32_t* n_out, void* workspace, size_t workspace_bytes,
                                 void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(sweep_offsets && n_out && has_transform && time_lag && filter_close, "d3b_ingest_sweeps: null argument");
  D3B_REQUIRE(n_sweeps >= 1 && n_sweeps <= D3B_INGEST_MAX_SWEEPS, "d3b_ingest_sweeps: %d sweeps outside [1, %d]", n_sweeps,
              D3B_INGEST_MAX_SWEEPS);
  D3B_REQUIRE(n_feat >= 3 && raw_stride >= n_feat && out_cap >= 0, "d3b_ingest_sweeps: bad layout (n_feat %d, stride %d)",
              n_feat, raw_stride);
  IngestParams p = params_of(n_sweeps, 1, raw_stride, n_feat, radius);
  int n_chunks = 0;
  for (int s = 0; s <= n_sweeps; ++s) {
    p.off[s] = sweep_offsets[s];
    D3B_REQUIRE(s == 0 ? p.off[s] == 0 : p.off[s] >= p.off[s - 1], "d3b_ingest_sweeps: sweep_offsets not monotone");
    if (s > 0) n_chunks += div_up(p.off[s] - p.off[s - 1], kIngestChunk);
  }
  for (int s = 0; s < n_sweeps; ++s) {
    const bool has = has_transform[s] != 0;
    p.flags[s] = (has ? kHasTransform : 0u) | (filter_close[s] ? kFilterClose : 0u);
    p.time_lag[s] = time_lag[s];
    D3B_REQUIRE(!has || transforms, "d3b_ingest_sweeps: transforms missing");
    for (int c = 0; c < 12; ++c) p.m[s][c] = has ? transforms[(size_t)s * 16 + c] : 0.0;
  }
  const int n = p.off[n_sweeps];
  p.raw_cap = n;
  if (n == 0) {
    D3B_CUDA(cudaMemsetAsync(n_out, 0, 4, stream));
    return D3B_OK;
  }
  D3B_REQUIRE(raw && out && workspace, "d3b_ingest_sweeps: null buffer");
  const size_t need = d3b_ingest_workspace_bytes(n);
  if (need > workspace_bytes) {
    set_error("d3b_ingest_sweeps: workspace %zu < %zu", workspace_bytes, need);
    return D3B_ERR_WORKSPACE;
  }
  return launch_ingest(p, raw, n_chunks, out, out_cap, n_out, nullptr, nullptr, (int*)workspace,
                       (int*)((char*)workspace + need / 2), stream);
}

namespace {

// d3b_ingest_sweeps_dev and d3b_ingest_sweeps_gather: the same checks and launches, sweep_src = nullptr for the former.
int ingest_dev(const char* name, const float* raw, int32_t raw_capacity, int32_t raw_stride, int32_t n_feat,
               const int32_t* sweep_offsets, const int32_t* sweep_src, const int32_t* sample_sweeps,
               const double* transforms, const float* time_lag, const uint8_t* flags, int32_t sweep_capacity,
               int32_t batch, float radius, float* out, int32_t* cloud_offsets, int32_t* status, void* workspace,
               size_t workspace_bytes, cudaStream_t stream) {
  D3B_REQUIRE(sweep_offsets && sample_sweeps && transforms && time_lag && flags && cloud_offsets && workspace,
              "%s: null argument", name);
  D3B_REQUIRE(batch >= 1 && batch <= kIngestMaxBatch, "%s: batch %d outside [1, %d]", name, batch, kIngestMaxBatch);
  D3B_REQUIRE(sweep_capacity >= 1 && sweep_capacity <= D3B_INGEST_MAX_SWEEPS * batch,
              "%s: sweep_capacity %d outside [1, %d * batch]", name, sweep_capacity, D3B_INGEST_MAX_SWEEPS);
  D3B_REQUIRE(raw_capacity >= 0 && raw_capacity <= (1 << 30), "%s: raw_capacity %d outside [0, 2^30]", name,
              raw_capacity);
  D3B_REQUIRE(n_feat >= 3 && raw_stride >= n_feat, "%s: bad layout (n_feat %d, stride %d)", name, n_feat, raw_stride);
  D3B_REQUIRE(raw_capacity == 0 || (raw && out), "%s: null buffer", name);
  const size_t need = d3b_ingest_dev_workspace_bytes(raw_capacity, sweep_capacity);
  if (need > workspace_bytes) {
    set_error("%s: workspace %zu < %zu", name, workspace_bytes, need);
    return D3B_ERR_WORKSPACE;
  }
  IngestParams p = params_of(sweep_capacity, batch, raw_stride, n_feat, radius);
  p.raw_cap = raw_capacity;
  p.off_dev = sweep_offsets; p.src_dev = sweep_src; p.sample_dev = sample_sweeps; p.m_dev = transforms;
  p.lag_dev = time_lag; p.flags_dev = flags;
  return launch_ingest(p, raw, div_up(raw_capacity, kIngestChunk) + sweep_capacity, out, raw_capacity, nullptr,
                       cloud_offsets, status, (int*)workspace, (int*)((char*)workspace + need / 2), stream);
}

}  // namespace

extern "C" int d3b_ingest_sweeps_dev(const float* raw, int32_t raw_capacity, int32_t raw_stride, int32_t n_feat,
                                     const int32_t* sweep_offsets, const int32_t* sample_sweeps, const double* transforms,
                                     const float* time_lag, const uint8_t* flags, int32_t sweep_capacity, int32_t batch,
                                     float radius, float* out, int32_t* cloud_offsets, int32_t* status, void* workspace,
                                     size_t workspace_bytes, void* stream_) {
  return ingest_dev("d3b_ingest_sweeps_dev", raw, raw_capacity, raw_stride, n_feat, sweep_offsets, nullptr,
                    sample_sweeps, transforms, time_lag, flags, sweep_capacity, batch, radius, out, cloud_offsets, status,
                    workspace, workspace_bytes, (cudaStream_t)stream_);
}

extern "C" size_t d3b_ingest_gather_workspace_bytes(int32_t raw_capacity, int32_t sweep_capacity) {
  return d3b_ingest_dev_workspace_bytes(raw_capacity, sweep_capacity);
}

extern "C" int d3b_ingest_sweeps_gather(const float* raw, int32_t raw_capacity, int32_t raw_stride, int32_t n_feat,
                                        const int32_t* sweep_offsets, const int32_t* sweep_src,
                                        const int32_t* sample_sweeps, const double* transforms, const float* time_lag,
                                        const uint8_t* flags, int32_t sweep_capacity, int32_t batch, float radius,
                                        float* out, int32_t* cloud_offsets, int32_t* status, void* workspace,
                                        size_t workspace_bytes, void* stream_) {
  D3B_REQUIRE(sweep_src, "d3b_ingest_sweeps_gather: null argument (sweep_src)");
  return ingest_dev("d3b_ingest_sweeps_gather", raw, raw_capacity, raw_stride, n_feat, sweep_offsets, sweep_src,
                    sample_sweeps, transforms, time_lag, flags, sweep_capacity, batch, radius, out, cloud_offsets, status,
                    workspace, workspace_bytes, (cudaStream_t)stream_);
}
