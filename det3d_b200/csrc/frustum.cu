// KITTI camera-frustum crop on the device: a batch of raw LiDAR scans -> the points that fall inside each scan's camera
// frustum, every column, input order kept, in the form d3b_voxelize_dev takes.
//
// Reference semantics, det3d/core/bbox/box_np_ops.py:941-952 (remove_outside_points) with
// det3d/core/bbox/geometry.py:241-276 (_points_in_convex_polygon_3d_jit): for each point and each of the frustum's 6
// planes in order, s = x*n0 + y*n1 + z*n2 + d with the f32 coordinates promoted to f64 and the sum taken left to right;
// the point is outside as soon as s >= 0 (a NaN coordinate never satisfies it, so such a point is kept).  The planes
// (n0, n1, n2, d) come from the calibration and are computed once per calibration on the host
// (det3d_b200.core.bbox.box_np_ops.camera_frustum_planes); only the test and the compaction run per point.
//
// The compaction is the ingest's (csrc/ingest.cu): 1024-point chunks that never straddle a cloud, count -> one-CTA scan
// of the chunk counts -> emit.  Every CTA first clamps the device cloud offsets (prefix max, then min with the capacity)
// into shared memory, identically in every CTA, before any point index is formed; a count / emit CTA then stages its
// cloud's 24 doubles in shared memory.
#include "chunk_scan.cuh"

namespace d3b {
namespace {

constexpr int kCropChunk = 1024;
constexpr int kCropThreads = 256;                  // 4 consecutive points per thread
constexpr int kCropMaxBatch = 64;
constexpr int kCropMinDim = 3, kCropMaxDim = 16;

struct CropParams {
  const int* off_dev;                              // [batch + 1] raw cloud offsets
  const double* planes;                            // [batch][6][4] (n0, n1, n2, d)
  int batch, ndim, cap;
};

// Per-CTA copy of the clamped offsets.
struct CropTable {
  int off[kCropMaxBatch + 1];                      // raw rows of cloud b: [off[b], off[b + 1])
  int chunk_off[kCropMaxBatch + 1];                // prefix of the clouds' chunk counts
  int buf[32];                                     // block-scan scratch
};

// Returns, to every thread after the barrier, whether the clamp changed anything.
__device__ __forceinline__ bool load_offsets(const CropParams& p, CropTable& t) {
  const bool bad = clamp_table<kCropChunk>([&](int i) { return __ldg(p.off_dev + i); }, p.batch, p.cap, t.off,
                                           t.chunk_off, t.buf);
  return __syncthreads_or(bad) != 0;
}

// The cloud that owns chunk g < chunk_off[batch]: the last b with chunk_off[b] <= g (so never an empty cloud).
__device__ __forceinline__ int cloud_of_chunk(const CropParams& p, const CropTable& t, int g) {
  int lo = 0, hi = p.batch - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.chunk_off[mid] <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The reference's plane test: every product and sum rounded on its own, in its order (no FMA contraction).
__device__ __forceinline__ bool in_frustum(const float* __restrict__ q, const double* pl) {
  const double x = (double)q[0], y = (double)q[1], z = (double)q[2];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const double* n = pl + 4 * k;
    const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, n[0]), __dmul_rn(y, n[1])), __dmul_rn(z, n[2])), n[3]);
    if (s >= 0.0) return false;
  }
  return true;
}

// The chunk's cloud and its planes (staged in `pl`), its first row i0 for this thread, its end row; false when the CTA
// is past the live chunks (the grid is sized for the capacity).  Every thread calls it.
__device__ __forceinline__ bool chunk_of_cta(const CropParams& p, CropTable& t, double* pl, int& i0, int& end) {
  load_offsets(p, t);
  const int g = blockIdx.x;
  if (g >= t.chunk_off[p.batch]) return false;
  const int b = cloud_of_chunk(p, t, g);
  if (threadIdx.x < 24) pl[threadIdx.x] = __ldg(p.planes + (size_t)b * 24 + threadIdx.x);
  i0 = t.off[b] + (g - t.chunk_off[b]) * kCropChunk + threadIdx.x * 4;
  end = t.off[b + 1];
  __syncthreads();
  return true;
}

__device__ __forceinline__ unsigned kept_bits(const CropParams& p, const float* __restrict__ points, const double* pl,
                                              int i0, int end) {
  unsigned kept = 0u;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (i0 + j < end && in_frustum(points + (size_t)(i0 + j) * p.ndim, pl)) kept |= 1u << j;
  return kept;
}

__global__ void __launch_bounds__(kCropThreads)
crop_count(const CropParams p, const float* __restrict__ points, int* __restrict__ chunk_cnt) {
  __shared__ CropTable t;
  __shared__ double pl[24];
  int i0, end;
  if (!chunk_of_cta(p, t, pl, i0, end)) return;
  int local = __popc(kept_bits(p, points, pl, i0, end));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) local += __shfl_xor_sync(0xffffffffu, local, d);
  if ((threadIdx.x & 31) == 0) t.buf[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    int n = 0;
    for (int w = 0; w < kCropThreads / 32; ++w) n += t.buf[w];
    chunk_cnt[blockIdx.x] = n;
  }
}

// One CTA: exclusive scan of the live chunk counts -> chunk_base, then cloud_offsets_out[b] = the base of cloud b's
// first chunk (the kept total for an empty cloud at the end) and the clamp flag.
__global__ void __launch_bounds__(1024)
crop_scan(const CropParams p, const int* __restrict__ chunk_cnt, int* chunk_base, int* __restrict__ cloud_offsets,
          int* __restrict__ status) {
  __shared__ CropTable t;
  __shared__ int running;
  const bool clamped = load_offsets(p, t);
  const int n_chunks = t.chunk_off[p.batch];
  const int total = scan_chunk_counts(chunk_cnt, n_chunks, chunk_base, t.buf, running);
  if (threadIdx.x == 0 && status != nullptr) *status = clamped ? 1 : 0;
  for (int b = threadIdx.x; b <= p.batch; b += blockDim.x) {
    const int g = t.chunk_off[b];
    cloud_offsets[b] = g < n_chunks ? chunk_base[g] : total;
  }
}

__global__ void __launch_bounds__(kCropThreads)
crop_emit(const CropParams p, const float* __restrict__ points, const int* __restrict__ chunk_base,
          float* __restrict__ out) {
  __shared__ CropTable t;
  __shared__ double pl[24];
  int i0, end;
  if (!chunk_of_cta(p, t, pl, i0, end)) return;
  const unsigned kept = kept_bits(p, points, pl, i0, end);
  const int local = __popc(kept), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) t.buf[warp] = incl;
  __syncthreads();
  int warp_off = 0;
  for (int w = 0; w < warp; ++w) warp_off += t.buf[w];
  int r = chunk_base[blockIdx.x] + warp_off + incl - local;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (!((kept >> j) & 1u)) continue;
    if (r < p.cap) {
      const float* __restrict__ q = points + (size_t)(i0 + j) * p.ndim;
      float* __restrict__ o = out + (size_t)r * p.ndim;
      for (int c = 0; c < p.ndim; ++c) o[c] = q[c];
    }
    ++r;
  }
}

int max_chunks(int point_capacity, int batch) { return div_up(point_capacity, kCropChunk) + batch; }

}  // namespace
}  // namespace d3b

using namespace d3b;

// Chunks never straddle a cloud: at most capacity / 1024 + batch of them; two int arrays (counts, bases).
extern "C" size_t d3b_frustum_crop_workspace_bytes(int32_t point_capacity, int32_t batch) {
  if (point_capacity < 0 || point_capacity > (1 << 30) || batch < 1 || batch > kCropMaxBatch) return 0;
  return align_up((size_t)max_chunks(point_capacity, batch) * 4) * 2;
}

extern "C" int d3b_frustum_crop_dev(const float* points, int32_t point_capacity, int32_t ndim,
                                    const int32_t* cloud_offsets_in, const double* planes, int32_t batch, float* out,
                                    int32_t* cloud_offsets_out, int32_t* status, void* workspace,
                                    size_t workspace_bytes, void* stream_) {
  static const char* name = "d3b_frustum_crop_dev";
  D3B_REQUIRE(cloud_offsets_in && planes && cloud_offsets_out && workspace, "%s: null argument", name);
  D3B_REQUIRE(batch >= 1 && batch <= kCropMaxBatch, "%s: batch %d outside [1, %d]", name, batch, kCropMaxBatch);
  D3B_REQUIRE(point_capacity >= 0 && point_capacity <= (1 << 30), "%s: point_capacity %d outside [0, 2^30]", name,
              point_capacity);
  if (ndim < kCropMinDim || ndim > kCropMaxDim) {
    set_error("%s: ndim %d not built (%d <= ndim <= %d)", name, ndim, kCropMinDim, kCropMaxDim);
    return D3B_ERR_UNSUPPORTED;
  }
  D3B_REQUIRE(point_capacity == 0 || (points && out), "%s: null buffer", name);
  const size_t need = d3b_frustum_crop_workspace_bytes(point_capacity, batch);
  if (need > workspace_bytes) {
    set_error("%s: workspace %zu < %zu", name, workspace_bytes, need);
    return D3B_ERR_WORKSPACE;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  CropParams p = {};
  p.off_dev = cloud_offsets_in; p.planes = planes; p.batch = batch; p.ndim = ndim; p.cap = point_capacity;
  int* chunk_cnt = (int*)workspace;
  int* chunk_base = (int*)((char*)workspace + need / 2);
  const int n_chunks = max_chunks(point_capacity, batch);
  crop_count<<<n_chunks, kCropThreads, 0, stream>>>(p, points, chunk_cnt);
  D3B_LAUNCH_CHECK();
  crop_scan<<<1, 1024, 0, stream>>>(p, chunk_cnt, chunk_base, cloud_offsets_out, status);
  D3B_LAUNCH_CHECK();
  crop_emit<<<n_chunks, kCropThreads, 0, stream>>>(p, points, chunk_base, out);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}
