// Order-exact GPU voxelizer.
//
// Reproduces, bit for bit, the sequential first-come semantics of the
// reference CPU voxelizer (det3d/ops/point_cloud/point_cloud_ops.py:7-55):
//   * voxel id      = rank of the voxel's FIRST point in input order,
//   * slot of point = rank of the point among its voxel's points in input
//                     order, truncated at max_points,
//   * `break` at the first point that would open voxel #max_voxels+1
//     (point_cloud_ops.py:46-47): every later point is dropped, including
//     points of already-open voxels,
//   * cell = floorf((p - lo) / vs) in IEEE fp32 (true division, :36),
//     range test on the float before the int cast (:37-39).
//
// Four kernels, no sort:
//   A  vox_insert : cell -> open-addressing hash slot, atomicMin(first point)
//   B  vox_chunk_count / vox_chunk_scan / vox_assign : scan of the "is first point" flags in input
//                   order -> voxel ids, the cut-off point i*, voxel count
//   C  vox_lists  : every surviving point cascades its index through the
//                   voxel's max_points-long sorted list with atomicMin
//                   (a systolic insertion: each step keeps the smaller index
//                   and carries the larger one on) -> the max_points smallest
//                   indices, in order, without any sort or per-voxel lock
//   D  vox_emit   : gathers points into voxels[M,max_points,ndim], writes
//                   coors (b,z,y,x), num_points and the per-voxel mean
//                   (VoxelFeatureExtractorV3, voxel_encoder.py:206-211).
//
// HBM traffic per cloud = N*ndim*4 (points, read twice: A and D, the second
// time from L2) + M*(max_points*ndim*4 + 16 + 4 + ndim*4) written once.
//
// Cloud offsets: d3b_voxelize_dev reads them from device memory, so one
// captured CUDA graph serves clouds of any size up to a point capacity.  Every
// CTA that needs them first copies them, clamped, and their 1024-point chunk
// prefix into shared memory (load_offsets).  Grids, hash and workspace are
// sized from the capacity; voxel ids are first-point ranks, not hash slots, so
// the outputs do not depend on the capacity.
#include "common.cuh"

namespace d3b {

constexpr int kMaxBatch = 64;

constexpr int kRankChunk = 1024;          // points per rank chunk = 256 threads x 4 consecutive points

struct VoxParams {
  float vs[3];
  float lo[3];
  int grid[3];
  int ndim, max_points, max_voxels, batch;
  const int* off_dev;             // device cloud offsets [batch + 1]
  int point_cap;                  // rows of `points`
};

// Per-CTA copy of the cloud offsets and of their chunk prefix.
struct VoxOffsets {
  int off[kMaxBatch + 1];
  int chunk_off[kMaxBatch + 1];
};

// Fills `s` from p.off_dev, clamped into
// 0 = off[0] <= ... <= off[batch] <= point_cap as off[b] = min(max(0, raw[1..b]), point_cap) -- the same values in every
// CTA, before any point index is formed.  Returns (to every thread, after the barrier) whether the clamp changed anything.
__device__ __forceinline__ bool load_offsets(const VoxParams& p, VoxOffsets& s) {
  __shared__ int s_bad;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    int run_max = 0, run_off = 0, run_chunks = 0;
    bool bad = false;
#pragma unroll 1                                            // unrolled, it raises every kernel's register count
    for (int base = 0; base <= p.batch; base += 32) {
      const int b = base + lane;
      const int raw = b <= p.batch ? __ldg(p.off_dev + b) : 0;
      int m = b == 0 ? 0 : raw;                             // rows past `batch` repeat the last offset: 0 chunks
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {                    // inclusive prefix max
        const int t = __shfl_up_sync(0xffffffffu, m, d);
        if (lane >= d) m = max(m, t);
      }
      m = max(m, run_max);
      const int c = min(m, p.point_cap);
      bad |= b <= p.batch && c != raw;
      int prev = __shfl_up_sync(0xffffffffu, c, 1);
      if (lane == 0) prev = run_off;
      int n = b == 0 ? 0 : (c - prev + kRankChunk - 1) / kRankChunk;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {                    // inclusive prefix sum of the chunk counts
        const int t = __shfl_up_sync(0xffffffffu, n, d);
        if (lane >= d) n += t;
      }
      n += run_chunks;
      if (b <= p.batch) { s.off[b] = c; s.chunk_off[b] = n; }
      run_max = __shfl_sync(0xffffffffu, m, 31);
      run_off = __shfl_sync(0xffffffffu, c, 31);
      run_chunks = __shfl_sync(0xffffffffu, n, 31);
    }
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) s_bad = bad;
  }
  __syncthreads();
  return s_bad != 0;
}

__device__ __forceinline__ int cloud_of(const VoxParams& p, const VoxOffsets& s, int i) {
  int b = 0;
  while (b + 1 < p.batch && i >= s.off[b + 1]) ++b;
  return b;
}

// ---- A: hash insert ---------------------------------------------------------
__global__ void __launch_bounds__(256)
vox_insert(const VoxParams p, const float* __restrict__ points, unsigned long long* keys,
           int* first, int* __restrict__ pslot, unsigned int cap_mask) {
  __shared__ VoxOffsets s;
  load_offsets(p, s);
  const int n_total = s.off[p.batch];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += gridDim.x * blockDim.x) {
    const float* pt = points + (size_t)i * p.ndim;
    int c[3];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      // IEEE fp32: sub, true division, floor.  No reciprocal, no FMA.
      float f = floorf(__fdiv_rn(__fsub_rn(pt[j], p.lo[j]), p.vs[j]));
      // NaN fails both comparisons below -> dropped (reference: undefined).
      if (!(f >= 0.0f && f < (float)p.grid[j])) { ok = false; break; }
      c[j] = (int)f;
    }
    if (!ok) { pslot[i] = -1; continue; }
    const int b = cloud_of(p, s, i);
    const unsigned long long key =
        (((unsigned long long)b * p.grid[2] + c[2]) * p.grid[1] + c[1]) * p.grid[0] + c[0];
    unsigned int slot = (unsigned int)mix64(key) & cap_mask;
    while (true) {
      unsigned long long prev = atomicCAS(&keys[slot], kEmptyKey, key);
      if (prev == kEmptyKey || prev == key) break;
      slot = (slot + 1) & cap_mask;
    }
    atomicMin(&first[slot], i);
    pslot[i] = (int)slot;
  }
}

// ---- B: rank voxels by first point ------------------------------------------------
// voxel id = number of "first points" that precede the voxel's own first point in input order: an exclusive scan
// of the is-first flags over the cloud.  One CTA per cloud is bound by a single SM's load/store path (measured
// 28 us for 20k points), so the scan is split the classic way: per-1024-point chunk counts (grid) -> scan of the
// chunk counts (one CTA per cloud, a few dozen values) -> chunk-local scan + offset (grid).
__device__ __forceinline__ int chunk_cloud(const VoxParams& p, const VoxOffsets& s, int g) {
  int b = 0;
  while (b + 1 < p.batch && g >= s.chunk_off[b + 1]) ++b;
  return b;
}

// is-first flags of the 4 points owned by this thread (bit j) and their hash slots
__device__ __forceinline__ unsigned int rank_flags(const VoxParams& p, const int* __restrict__ first,
                                                   const int* __restrict__ pslot, int i0, int end, int (&slot)[4]) {
  int fst[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) slot[j] = (i0 + j < end) ? pslot[i0 + j] : -1;
#pragma unroll
  for (int j = 0; j < 4; ++j) fst[j] = slot[j] >= 0 ? first[slot[j]] : -1;
  unsigned int flags = 0u;
#pragma unroll
  for (int j = 0; j < 4; ++j) flags |= (unsigned int)(slot[j] >= 0 && fst[j] == i0 + j) << j;
  return flags;
}

__global__ void __launch_bounds__(256)
vox_chunk_count(const VoxParams p, const int* __restrict__ first, const int* __restrict__ pslot,
                int* __restrict__ chunk_cnt) {
  __shared__ int warp_sums[8];
  __shared__ VoxOffsets s;
  load_offsets(p, s);
  const int g = blockIdx.x;
  if (g >= s.chunk_off[p.batch]) return;   // the grid is sized for the capacity
  const int b = chunk_cloud(p, s, g);
  const int i0 = s.off[b] + (g - s.chunk_off[b]) * kRankChunk + threadIdx.x * 4;
  int slot[4];
  int local = __popc(rank_flags(p, first, pslot, i0, s.off[b + 1], slot));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) local += __shfl_xor_sync(0xffffffffu, local, d);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < 8; ++w) t += warp_sums[w];
    chunk_cnt[g] = t;
  }
}

// one CTA per cloud: exclusive scan of its chunk counts, voxel count, default cut-off
__global__ void __launch_bounds__(1024)
vox_chunk_scan(const VoxParams p, const int* __restrict__ chunk_cnt, int* __restrict__ chunk_base,
               int* __restrict__ cut, int* __restrict__ counts, int* __restrict__ status) {
  __shared__ int warp_sums[32];
  __shared__ int running;
  __shared__ VoxOffsets s;
  const bool clamped = load_offsets(p, s);
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (status != nullptr && b == 0 && threadIdx.x == 0) *status = clamped ? 1 : 0;
  const int g0 = s.chunk_off[b], g1 = s.chunk_off[b + 1];
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  for (int base = g0; base < g1; base += blockDim.x) {
    const int g = base + threadIdx.x;
    const int v = g < g1 ? chunk_cnt[g] : 0;
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
    if (g < g1) chunk_base[g] = running + (warp == 0 ? 0 : warp_sums[warp - 1]) + incl - v;
    const int total = warp_sums[31];
    __syncthreads();
    if (threadIdx.x == 0) running += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counts[b] = running < p.max_voxels ? running : p.max_voxels;
    cut[b] = s.off[b + 1];               // vox_assign lowers it to the point where the reference `break` fires
  }
}

__global__ void __launch_bounds__(256)
vox_assign(const VoxParams p, const int* __restrict__ first, const int* __restrict__ pslot,
           const int* __restrict__ chunk_base, int* __restrict__ vid, int* __restrict__ vslot, int* __restrict__ cut) {
  __shared__ int warp_sums[8];
  __shared__ VoxOffsets s;
  load_offsets(p, s);
  const int g = blockIdx.x;
  if (g >= s.chunk_off[p.batch]) return;   // the grid is sized for the capacity
  const int b = chunk_cloud(p, s, g);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i0 = s.off[b] + (g - s.chunk_off[b]) * kRankChunk + threadIdx.x * 4;
  int slot[4];
  const unsigned int flags = rank_flags(p, first, pslot, i0, s.off[b + 1], slot);
  const int local = __popc(flags);
  int incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  int warp_off = 0;
  for (int w = 0; w < warp; ++w) warp_off += warp_sums[w];
  int r = chunk_base[g] + warp_off + incl - local;   // exclusive rank of this thread's first flagged point
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (!((flags >> j) & 1u)) continue;
    if (r < p.max_voxels) {
      vid[slot[j]] = r;
      vslot[b * p.max_voxels + r] = slot[j];
    } else {
      vid[slot[j]] = -1;
      if (r == p.max_voxels) cut[b] = i0 + j;   // the reference `break` fires here
    }
    ++r;
  }
}

// ---- C: per-voxel sorted index lists --------------------------------------------
__global__ void __launch_bounds__(256)
vox_lists(const VoxParams p, const int* __restrict__ pslot, const int* __restrict__ vid,
          const int* __restrict__ cut, int* lists) {
  __shared__ VoxOffsets s;
  load_offsets(p, s);
  const int n_total = s.off[p.batch];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += gridDim.x * blockDim.x) {
    const int slot = pslot[i];
    if (slot < 0) continue;
    const int b = cloud_of(p, s, i);
    if (i >= cut[b]) continue;
    const int v = vid[slot];
    if (v < 0) continue;
    int* L = lists + ((size_t)b * p.max_voxels + v) * p.max_points;
    // Entries only ever decrease, so a (possibly stale) tail already below i
    // proves the list is full of smaller indices.
    if (*(volatile int*)&L[p.max_points - 1] < i) continue;
    int x = i;
    for (int r = 0; r < p.max_points; ++r) {
      const int old = atomicMin(&L[r], x);
      if (old >= kSentinelMin) break;  // took an empty slot
      if (old > x) x = old;            // displaced a larger index: carry it on
    }
  }
}

// ---- D: emit ------------------------------------------------------------------
__global__ void __launch_bounds__(256)
vox_emit(const VoxParams p, const float* __restrict__ points,
         const unsigned long long* __restrict__ keys, const int* __restrict__ vslot,
         const int* __restrict__ lists, int* __restrict__ counts, float* __restrict__ voxels,
         int* __restrict__ coors, int* __restrict__ num_points, float* __restrict__ mean_feats) {
  __shared__ int pref[kMaxBatch + 1];
  if (threadIdx.x == 0) {
    int s = 0;
    for (int b = 0; b < p.batch; ++b) { pref[b] = s; s += counts[b]; }
    pref[p.batch] = s;
    if (blockIdx.x == 0) counts[p.batch] = s;
  }
  __syncthreads();
  // without the [M, max_points, ndim] output only slot 0's threads have work (mean / coors / counts): shrink the index space
  const int per_voxel = (voxels != nullptr ? p.max_points : 1) * p.ndim;
  const long long total = (long long)pref[p.batch] * per_voxel;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(e / per_voxel);
    const int rc = (int)(e - (long long)g * per_voxel);
    const int r = rc / p.ndim, c = rc - r * p.ndim;
    int b = 0;
    while (b + 1 < p.batch && g >= pref[b + 1]) ++b;
    const int v = g - pref[b];
    const int* L = lists + ((size_t)b * p.max_voxels + v) * p.max_points;
    if (voxels != nullptr) {
      const int idx = L[r];
      voxels[e] = idx < kSentinelMin ? points[(size_t)idx * p.ndim + c] : 0.0f;
    }
    if (r == 0) {
      int num = 0;
      float sum = 0.0f;
      for (int q = 0; q < p.max_points; ++q) {
        const int idx = L[q];
        if (idx >= kSentinelMin) break;
        sum = __fadd_rn(sum, points[(size_t)idx * p.ndim + c]);
        ++num;
      }
      if (mean_feats != nullptr) mean_feats[(size_t)g * p.ndim + c] = __fdiv_rn(sum, (float)num);
      if (c == 0) {
        num_points[g] = num;
        unsigned long long key = keys[vslot[b * p.max_voxels + v]];
        const int cx = (int)(key % p.grid[0]); key /= p.grid[0];
        const int cy = (int)(key % p.grid[1]); key /= p.grid[1];
        const int cz = (int)(key % p.grid[2]);
        int4 o = make_int4(b, cz, cy, cx);
        *reinterpret_cast<int4*>(coors + (size_t)g * 4) = o;
      }
    }
  }
}

// ---- workspace carve-up ----------------------------------------------------------
struct VoxWorkspace {
  unsigned long long* keys;
  int* first;   // [cap]          \ one 0x7f memset
  int* lists;   // [B*MV*MP]      /
  int* vid;     // [cap]
  int* pslot;   // [n_total]
  int* vslot;   // [B*MV]
  int* cut;     // [B]
  int* chunk_cnt;   // [chunks] is-first points per 1024-point chunk
  int* chunk_base;  // [chunks] exclusive scan of the above within the cloud
  size_t cap, bytes, sentinel_bytes;
};

static VoxWorkspace carve(const d3b_voxel_cfg* cfg, int n_total, int batch, char* base) {
  VoxWorkspace w;
  size_t cap = 1024;
  while (cap < 2 * (size_t)(n_total > 0 ? n_total : 1)) cap <<= 1;
  w.cap = cap;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return base ? base + o : (char*)nullptr; };
  w.keys = (unsigned long long*)take(cap * 8);
  const size_t first_bytes = align_up(cap * 4);
  const size_t lists_bytes = align_up((size_t)batch * cfg->max_voxels * cfg->max_points * 4);
  w.first = (int*)take(first_bytes);
  w.lists = (int*)take(lists_bytes);
  w.sentinel_bytes = first_bytes + lists_bytes;
  w.vid = (int*)take(cap * 4);
  w.pslot = (int*)take((size_t)(n_total > 0 ? n_total : 1) * 4);
  w.vslot = (int*)take((size_t)batch * cfg->max_voxels * 4);
  w.cut = (int*)take((size_t)batch * 4);
  w.chunk_cnt = (int*)take(((size_t)n_total / 1024 + batch + 1) * 4);
  w.chunk_base = (int*)take(((size_t)n_total / 1024 + batch + 1) * 4);
  w.bytes = off;
  return w;
}

}  // namespace d3b

using namespace d3b;

extern "C" size_t d3b_voxelize_workspace_bytes(const d3b_voxel_cfg* cfg, int32_t n_points_total,
                                               int32_t batch) {
  if (!cfg || batch < 1 || n_points_total < 0) return 0;
  return carve(cfg, n_points_total, batch, nullptr).bytes;
}

extern "C" const int32_t* d3b_voxelize_point_lists(const d3b_voxel_cfg* cfg, int32_t n_points_total, int32_t batch,
                                                   void* workspace) {
  if (!cfg || batch < 1 || n_points_total < 0 || !workspace) return nullptr;
  return carve(cfg, n_points_total, batch, (char*)workspace).lists;
}

// The grid-stride kernels are sized for the capacity's rows and the rank-chunk grids for its chunks plus one partial
// chunk per cloud; the kernels stop at the live counts they read from the offsets.
static int launch_voxelize(const VoxParams& p, const d3b_voxel_cfg* cfg, const float* points, float* voxels,
                           int32_t* coors, int32_t* num_points, float* mean_feats, int32_t* voxel_counts,
                           int32_t* status, const VoxWorkspace& w, cudaStream_t stream) {
  const int n_rows = p.point_cap, n_chunks = div_up(p.point_cap, kRankChunk) + p.batch;
  D3B_CUDA(cudaMemsetAsync(w.keys, 0xff, w.cap * 8, stream));
  D3B_CUDA(cudaMemsetAsync(w.first, 0x7f, w.sentinel_bytes, stream));
  if (n_rows > 0) {
    vox_insert<<<grid_for(n_rows, 256), 256, 0, stream>>>(p, points, w.keys, w.first, w.pslot,
                                                           (unsigned int)(w.cap - 1));
    D3B_LAUNCH_CHECK();
  }
  vox_chunk_count<<<n_chunks, 256, 0, stream>>>(p, w.first, w.pslot, w.chunk_cnt);
  D3B_LAUNCH_CHECK();
  vox_chunk_scan<<<p.batch, 1024, 0, stream>>>(p, w.chunk_cnt, w.chunk_base, w.cut, voxel_counts, status);
  D3B_LAUNCH_CHECK();
  vox_assign<<<n_chunks, 256, 0, stream>>>(p, w.first, w.pslot, w.chunk_base, w.vid, w.vslot, w.cut);
  D3B_LAUNCH_CHECK();
  if (n_rows > 0) {
    vox_lists<<<grid_for(n_rows, 256), 256, 0, stream>>>(p, w.pslot, w.vid, w.cut, w.lists);
    D3B_LAUNCH_CHECK();
  }
  const long long cap_elems = (long long)p.batch * cfg->max_voxels * (voxels != nullptr ? cfg->max_points : 1) * cfg->ndim;
  vox_emit<<<grid_for(cap_elems, 256), 256, 0, stream>>>(p, points, w.keys, w.vslot, w.lists,
                                                          voxel_counts, voxels, coors, num_points,
                                                          mean_feats);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_voxelize_dev(const d3b_voxel_cfg* cfg, const float* points, int32_t point_capacity,
                                const int32_t* cloud_offsets_dev, int32_t batch, float* voxels, int32_t* coors,
                                int32_t* num_points, float* mean_feats, int32_t* voxel_counts, int32_t* status,
                                void* workspace, size_t workspace_bytes, void* stream_) {
  D3B_REQUIRE(cfg && cloud_offsets_dev && coors && num_points && voxel_counts && workspace,
              "d3b_voxelize_dev: null argument");
  D3B_REQUIRE(batch >= 1 && batch <= kMaxBatch, "d3b_voxelize_dev: batch %d outside [1,%d]", batch, kMaxBatch);
  D3B_REQUIRE(cfg->ndim >= 3 && cfg->max_points >= 1 && cfg->max_voxels >= 1,
              "d3b_voxelize_dev: bad cfg (ndim %d, max_points %d, max_voxels %d)", cfg->ndim, cfg->max_points,
              cfg->max_voxels);
  for (int j = 0; j < 3; ++j)
    D3B_REQUIRE(cfg->grid[j] >= 1 && cfg->voxel_size[j] > 0.0f, "d3b_voxelize_dev: bad grid/voxel_size");
  D3B_REQUIRE((double)cfg->grid[0] * cfg->grid[1] * cfg->grid[2] * batch < 9.0e18, "d3b_voxelize_dev: grid too large");
  D3B_REQUIRE(point_capacity >= 0 && point_capacity <= (1 << 30), "d3b_voxelize_dev: point_capacity %d outside [0, 2^30]",
              point_capacity);
  D3B_REQUIRE(point_capacity == 0 || points, "d3b_voxelize_dev: null points");
  VoxParams p;
  for (int j = 0; j < 3; ++j) { p.vs[j] = cfg->voxel_size[j]; p.lo[j] = cfg->range_min[j]; p.grid[j] = cfg->grid[j]; }
  p.ndim = cfg->ndim; p.max_points = cfg->max_points; p.max_voxels = cfg->max_voxels; p.batch = batch;
  p.off_dev = cloud_offsets_dev;
  p.point_cap = point_capacity;
  VoxWorkspace w = carve(cfg, point_capacity, batch, (char*)workspace);
  if (w.bytes > workspace_bytes) {
    set_error("d3b_voxelize_dev: workspace %zu < %zu", workspace_bytes, w.bytes);
    return D3B_ERR_WORKSPACE;
  }
  return launch_voxelize(p, cfg, points, voxels, coors, num_points, mean_feats, voxel_counts, status, w,
                         (cudaStream_t)stream_);
}
