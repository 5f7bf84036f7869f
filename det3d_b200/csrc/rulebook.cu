// Rulebook construction for submanifold and strided sparse 3-D convolution.
//
// Semantics follow spconv v1.x `get_indice_pairs` as used by
// det3d/models/backbones/scn.py:106-157 (SubMConv3d / SparseConv3d):
//   input site p feeds output site o through kernel offset k = (kz,ky,kx) iff
//       p = o * stride - padding + k          (dilation 1)
//   SubMConv3d : outputs == inputs (same rows, same order), padding = k/2
//   SparseConv3d: outputs = every in-bounds o reachable from an active p,
//                 numbered by ascending linear index ((b*D+z)*H+y)*W+x.
// Row rule, the same in every kernel here and in the scatters: a row whose batch index or coordinate lies outside its
// grid is ignored (it is no neighbour, marks no output and gets -1 for every offset), and among rows that share a
// cell the lowest row index is the one every lookup returns.
//
// The map is stored output-stationary (nbr[k][o] = input row or -1) so the
// convolution kernel owns its output rows: no scatter-add, no atomics,
// deterministic accumulation order.
//
// Site lookup structures:
//   level 0      : open-addressing hash  key(lin) -> row       (rows keep the
//                  caller's order)
//   strided level: occupancy bitmap over the output grid + exclusive popcount
//                  prefix per 32-bit word; row(o) = prefix[w] + popc(bits below).
//                  The popcount scan IS the ascending-order numbering: no sort.
//
// HBM bytes per build ~= N_in*16 (coords) + K*N_out*4 (map) + N_out*16 + bitmap.
#include "common.cuh"

namespace d3b {

struct SiteIndexDev {
  int D, H, W, B;
  const unsigned long long* hkeys;
  const int* hvals;
  unsigned int hmask;
  const unsigned int* bitmap;
  const int* prefix;
  int row_cap;  // bitmap mode: ranks >= row_cap are treated as absent
};

static SiteIndexDev to_dev(const d3b_site_index* s, int row_cap) {
  SiteIndexDev d;
  d.D = s->spatial[0]; d.H = s->spatial[1]; d.W = s->spatial[2]; d.B = s->batch;
  d.hkeys = (const unsigned long long*)s->hash_keys;
  d.hvals = s->hash_vals;
  d.hmask = (unsigned int)(s->hash_cap - 1);
  d.bitmap = s->bitmap;
  d.prefix = s->word_prefix;
  d.row_cap = row_cap;
  return d;
}

__device__ __forceinline__ unsigned long long lin_index(const SiteIndexDev& s, int b, int z, int y,
                                                        int x) {
  return (((unsigned long long)b * s.D + z) * s.H + y) * s.W + x;
}

__device__ __forceinline__ bool in_grid(const SiteIndexDev& s, int4 c) {
  return (unsigned)c.x < (unsigned)s.B && (unsigned)c.y < (unsigned)s.D && (unsigned)c.z < (unsigned)s.H &&
         (unsigned)c.w < (unsigned)s.W;
}

__device__ __forceinline__ int site_lookup(const SiteIndexDev& s, int b, int z, int y, int x) {
  if ((unsigned)z >= (unsigned)s.D || (unsigned)y >= (unsigned)s.H || (unsigned)x >= (unsigned)s.W)
    return -1;
  const unsigned long long lin = lin_index(s, b, z, y, x);
  if (s.hkeys != nullptr) {
    unsigned int slot = (unsigned int)mix64(lin) & s.hmask;
    while (true) {
      const unsigned long long k = s.hkeys[slot];
      if (k == lin) return s.hvals[slot];
      if (k == kEmptyKey) return -1;
      slot = (slot + 1) & s.hmask;
    }
  }
  const unsigned long long w = lin >> 5;
  const unsigned int bit = (unsigned int)(lin & 31);
  const unsigned int word = s.bitmap[w];
  if (!((word >> bit) & 1u)) return -1;
  const int r = s.prefix[w] + __popc(word & ((1u << bit) - 1u));
  return r < s.row_cap ? r : -1;
}

struct KernelGeom {
  int k[3], s[3], p[3];
  int kvol;
};

// ---- level-0 hash build --------------------------------------------------------
// vals must hold a value above every row index on entry (0x7f memset): duplicates of a cell keep the lowest row, so
// the map does not depend on which thread wins the key.
__global__ void __launch_bounds__(256)
rb_hash_insert(const int* __restrict__ coors, const int* __restrict__ n_rows, int row_cap,
               SiteIndexDev s, unsigned long long* keys, int* vals) {
  const int n = min(*n_rows, row_cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int4 c = *reinterpret_cast<const int4*>(coors + (size_t)i * 4);
    if (!in_grid(s, c)) continue;  // out-of-grid rows are never found by any lookup
    const unsigned long long lin = lin_index(s, c.x, c.y, c.z, c.w);
    unsigned int slot = (unsigned int)mix64(lin) & s.hmask;
    while (true) {
      const unsigned long long prev = atomicCAS(&keys[slot], kEmptyKey, lin);
      if (prev == kEmptyKey || prev == lin) break;
      slot = (slot + 1) & s.hmask;
    }
    atomicMin(&vals[slot], i);
  }
}

// ---- neighbour map (shared by SubM and strided) -----------------------------------
// One thread per (k, o); consecutive threads walk consecutive o for one k so
// both the coordinate reads and the nbr writes are coalesced.
__global__ void __launch_bounds__(256)
rb_neighbours(const int* __restrict__ out_coors, const int* __restrict__ n_out, int out_cap,
              SiteIndexDev out_grid, SiteIndexDev in_index, KernelGeom g, int* __restrict__ nbr,
              unsigned int* __restrict__ tile_mask) {
  const int n = min(*n_out, out_cap);
  const long long total = (long long)n * g.kvol;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(e / n);
    const int o = (int)(e - (long long)k * n);
    const int4 c = *reinterpret_cast<const int4*>(out_coors + (size_t)o * 4);
    const int kx = k % g.k[2];
    const int ky = (k / g.k[2]) % g.k[1];
    const int kz = k / (g.k[2] * g.k[1]);
    const int z = c.y * g.s[0] - g.p[0] + kz;
    const int y = c.z * g.s[1] - g.p[1] + ky;
    const int x = c.w * g.s[2] - g.p[2] + kx;
    const int r = in_grid(out_grid, c) ? site_lookup(in_index, c.x, z, y, x) : -1;
    nbr[(size_t)k * out_cap + o] = r;
    if (r >= 0) {
      // one atomic per (tile, k) group present in this warp
      const int tag = (o >> 7) * 32 + k;
      const unsigned int peers = __match_any_sync(__activemask(), tag);
      if ((int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicOr(&tile_mask[o >> 7], 1u << k);
    }
  }
}

// ---- strided conv: mark reachable output sites --------------------------------------
__global__ void __launch_bounds__(256)
rb_mark_outputs(const int* __restrict__ in_coors, const int* __restrict__ n_in, int in_cap,
                SiteIndexDev in_dims, SiteIndexDev out, KernelGeom g, unsigned int* bitmap) {
  const int n = min(*n_in, in_cap);
  const long long total = (long long)n * g.kvol;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / g.kvol);
    const int k = (int)(e - (long long)i * g.kvol);
    const int4 c = *reinterpret_cast<const int4*>(in_coors + (size_t)i * 4);
    if (!in_grid(in_dims, c)) continue;
    const int kx = k % g.k[2];
    const int ky = (k / g.k[2]) % g.k[1];
    const int kz = k / (g.k[2] * g.k[1]);
    const int tz = c.y + g.p[0] - kz, ty = c.z + g.p[1] - ky, tx = c.w + g.p[2] - kx;
    if (tz < 0 || ty < 0 || tx < 0) continue;
    if (tz % g.s[0] || ty % g.s[1] || tx % g.s[2]) continue;
    const int oz = tz / g.s[0], oy = ty / g.s[1], ox = tx / g.s[2];
    if (oz >= out.D || oy >= out.H || ox >= out.W) continue;
    const unsigned long long lin = lin_index(out, c.x, oz, oy, ox);
    atomicOr(&bitmap[lin >> 5], 1u << (unsigned int)(lin & 31));
  }
}

// ---- popcount scan over the bitmap -----------------------------------------------------
constexpr int kScanThreads = 1024;
constexpr int kScanWordsPerThread = 4;
constexpr int kScanWordsPerBlock = kScanThreads * kScanWordsPerThread;

__device__ __forceinline__ int block_exclusive_scan(int v, int* smem /*[32]*/, int& block_total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = lane < (int)(blockDim.x >> 5) ? smem[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += t;
    }
    smem[lane] = w;
  }
  __syncthreads();
  const int off = warp == 0 ? 0 : smem[warp - 1];
  block_total = smem[(blockDim.x >> 5) - 1];
  __syncthreads();
  return off + incl - v;
}

// Exclusive popcount scan of the bitmap in ONE launch (decoupled look-back): a block counts its 4096 words, publishes the
// total, sums its
// predecessors' totals as they appear (they were dispatched earlier, so they are running or done), writes the word
// prefixes; the last block writes the row count.  block_sums must hold -1 ("not published") on entry (0xff memset).
__global__ void __launch_bounds__(kScanThreads)
rb_scan_fused(const unsigned int* __restrict__ bitmap, long long n_words, int* block_sums, int out_cap,
              int* __restrict__ n_out, int* __restrict__ word_prefix) {
  __shared__ int smem[32];
  __shared__ int s_offset;
  const long long base = (long long)blockIdx.x * kScanWordsPerBlock + threadIdx.x * kScanWordsPerThread;
  unsigned int w[kScanWordsPerThread];
  int cnt = 0;
  if (base + 3 < n_words) {
    const uint4 v = *reinterpret_cast<const uint4*>(bitmap + base);
    w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
  } else {
#pragma unroll
    for (int j = 0; j < kScanWordsPerThread; ++j) w[j] = base + j < n_words ? bitmap[base + j] : 0u;
  }
#pragma unroll
  for (int j = 0; j < kScanWordsPerThread; ++j) cnt += __popc(w[j]);
  int total;
  const int ex = block_exclusive_scan(cnt, smem, total);
  if (threadIdx.x == 0) {
    __threadfence();
    atomicExch(&block_sums[blockIdx.x], total);          // publish
  }
  if (threadIdx.x < 32) {
    int sum = 0;
    for (int j = threadIdx.x; j < (int)blockIdx.x; j += 32) {
      int v;
      do { v = *reinterpret_cast<volatile int*>(&block_sums[j]); } while (v < 0);
      sum += v;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    if (threadIdx.x == 0) s_offset = sum;
  }
  __syncthreads();
  int rank = s_offset + ex;
#pragma unroll
  for (int j = 0; j < kScanWordsPerThread; ++j) {
    if (base + j >= n_words) break;
    word_prefix[base + j] = rank;
    rank += __popc(w[j]);
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    const int all = s_offset + total;
    n_out[0] = all < out_cap ? all : out_cap;
    n_out[1] = all;
  }
}

// emit pass: a warp takes 32 bitmap words at a time; each lane decomposes ITS word's first cell once
// (the only 64-bit divisions), then the warp expands the non-zero words one by one, lane = bit, with
// carry arithmetic instead of divisions.
__global__ void __launch_bounds__(256)
rb_emit_coors(const unsigned int* __restrict__ bitmap, const int* __restrict__ word_prefix, long long n_words,
              SiteIndexDev out, int out_cap, int* __restrict__ out_coors) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long chunk = warp0; chunk * 32 < n_words; chunk += n_warps) {
    const long long wi = chunk * 32 + lane;
    const unsigned int mine = wi < n_words ? bitmap[wi] : 0u;
    int x0 = 0, y0 = 0, z0 = 0, b0 = 0, pref = 0;
    if (mine != 0u) {
      unsigned long long lin = (unsigned long long)wi << 5;
      x0 = (int)(lin % out.W); lin /= out.W;
      y0 = (int)(lin % out.H); lin /= out.H;
      z0 = (int)(lin % out.D);
      b0 = (int)(lin / out.D);
      pref = word_prefix[wi];
    }
    unsigned int nz = __ballot_sync(0xffffffffu, mine != 0u);
    while (nz) {
      const int src = __ffs(nz) - 1;
      nz &= nz - 1;
      const unsigned int bits = __shfl_sync(0xffffffffu, mine, src);
      int x = __shfl_sync(0xffffffffu, x0, src) + lane;
      int y = __shfl_sync(0xffffffffu, y0, src);
      int z = __shfl_sync(0xffffffffu, z0, src);
      int bb = __shfl_sync(0xffffffffu, b0, src);
      const int base_rank = __shfl_sync(0xffffffffu, pref, src);
      if ((bits >> lane) & 1u) {
        const int rank = base_rank + __popc(bits & ((1u << lane) - 1u));
        if (rank < out_cap) {
          while (x >= out.W) {
            x -= out.W;
            if (++y >= out.H) { y = 0; if (++z >= out.D) { z = 0; ++bb; } }
          }
          *reinterpret_cast<int4*>(out_coors + (size_t)rank * 4) = make_int4(bb, z, y, x);
        }
      }
    }
  }
}

static int check_geom(const int32_t ksize[3], KernelGeom* g) {
  g->kvol = ksize[0] * ksize[1] * ksize[2];
  for (int j = 0; j < 3; ++j) g->k[j] = ksize[j];
  return (g->kvol >= 1 && g->kvol <= 32 && ksize[0] >= 1 && ksize[1] >= 1 && ksize[2] >= 1) ? 0 : 1;
}

}  // namespace d3b

using namespace d3b;

extern "C" size_t d3b_rulebook_workspace_bytes(int64_t n_words) {
  if (n_words < 0) return 0;
  const long long n_blocks = (n_words + kScanWordsPerBlock - 1) / kScanWordsPerBlock;
  return align_up((size_t)(n_blocks + 1) * 4);
}

extern "C" int d3b_index_build_hash(const int32_t* coors, const int32_t* n_rows, int32_t row_cap,
                                    d3b_site_index* index, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(coors && n_rows && index && index->hash_keys && index->hash_vals,
              "d3b_index_build_hash: null argument");
  D3B_REQUIRE(index->hash_cap >= 2 && (index->hash_cap & (index->hash_cap - 1)) == 0 &&
                  index->hash_cap >= 2 * (long long)row_cap,
              "d3b_index_build_hash: hash_cap %d must be a power of two >= 2*row_cap (%d)",
              index->hash_cap, row_cap);
  D3B_CUDA(cudaMemsetAsync(index->hash_keys, 0xff, (size_t)index->hash_cap * 8, stream));
  D3B_CUDA(cudaMemsetAsync(index->hash_vals, 0x7f, (size_t)index->hash_cap * 4, stream));  // > any row (atomicMin)
  SiteIndexDev s = to_dev(index, row_cap);
  rb_hash_insert<<<grid_for(row_cap, 256), 256, 0, stream>>>(
      coors, n_rows, row_cap, s, (unsigned long long*)index->hash_keys, index->hash_vals);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_rulebook_subm(const int32_t* coors, const int32_t* n_rows, int32_t row_cap,
                                 const d3b_site_index* index, const int32_t ksize[3], int32_t* nbr,
                                 uint32_t* tile_mask, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(coors && n_rows && index && ksize && nbr && tile_mask, "d3b_rulebook_subm: null argument");
  KernelGeom g;
  D3B_REQUIRE(check_geom(ksize, &g) == 0, "d3b_rulebook_subm: kernel volume must be in [1,32]");
  for (int j = 0; j < 3; ++j) {
    D3B_REQUIRE(ksize[j] % 2 == 1, "d3b_rulebook_subm: kernel size must be odd");
    g.s[j] = 1;
    g.p[j] = ksize[j] / 2;
  }
  D3B_CUDA(cudaMemsetAsync(tile_mask, 0, (size_t)div_up(row_cap, 128) * 4, stream));
  const SiteIndexDev s = to_dev(index, row_cap);
  rb_neighbours<<<grid_for((long long)row_cap * g.kvol, 256), 256, 0, stream>>>(coors, n_rows, row_cap, s, s, g, nbr,
                                                                               tile_mask);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_rulebook_conv(const int32_t* in_coors, const int32_t* n_in, int32_t in_cap,
                                 const d3b_site_index* in_index, const int32_t ksize[3],
                                 const int32_t stride[3], const int32_t padding[3],
                                 d3b_site_index* out_index, int32_t* out_coors, int32_t* n_out,
                                 int32_t out_cap, int32_t* nbr, uint32_t* tile_mask, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(in_coors && n_in && in_index && ksize && stride && padding && out_index &&
                  out_coors && n_out && nbr && tile_mask && workspace,
              "d3b_rulebook_conv: null argument");
  D3B_REQUIRE(out_index->bitmap && out_index->word_prefix, "d3b_rulebook_conv: out_index needs bitmap storage");
  KernelGeom g;
  D3B_REQUIRE(check_geom(ksize, &g) == 0, "d3b_rulebook_conv: kernel volume must be in [1,32]");
  for (int j = 0; j < 3; ++j) {
    D3B_REQUIRE(stride[j] >= 1 && padding[j] >= 0, "d3b_rulebook_conv: bad stride/padding");
    D3B_REQUIRE(in_index->spatial[j] + 2 * padding[j] >= ksize[j],
                "d3b_rulebook_conv: kernel %d wider than the padded input %d + 2*%d along axis %d", ksize[j],
                in_index->spatial[j], padding[j], j);
    g.s[j] = stride[j];
    g.p[j] = padding[j];
    const int expect = (in_index->spatial[j] + 2 * padding[j] - (ksize[j] - 1) - 1) / stride[j] + 1;
    D3B_REQUIRE(out_index->spatial[j] == expect, "d3b_rulebook_conv: out spatial[%d]=%d, expected %d",
                j, out_index->spatial[j], expect);
  }
  D3B_REQUIRE(out_index->batch == in_index->batch, "d3b_rulebook_conv: batch mismatch");
  const long long cells = (long long)out_index->batch * out_index->spatial[0] * out_index->spatial[1] *
                          out_index->spatial[2];
  const long long n_words = (cells + 31) / 32;
  D3B_REQUIRE(out_index->n_words >= n_words, "d3b_rulebook_conv: bitmap has %lld words, need %lld",
              (long long)out_index->n_words, n_words);
  if (d3b_rulebook_workspace_bytes(n_words) > workspace_bytes) {
    set_error("d3b_rulebook_conv: workspace too small");
    return D3B_ERR_WORKSPACE;
  }
  int* block_sums = (int*)workspace;
  const int n_blocks = div_up(n_words, kScanWordsPerBlock);
  SiteIndexDev out = to_dev(out_index, out_cap);
  out.hkeys = nullptr;

  D3B_CUDA(cudaMemsetAsync(out_index->bitmap, 0, (size_t)n_words * 4, stream));
  D3B_CUDA(cudaMemsetAsync(tile_mask, 0, (size_t)div_up(out_cap, 128) * 4, stream));
  rb_mark_outputs<<<grid_for((long long)in_cap * g.kvol, 256), 256, 0, stream>>>(
      in_coors, n_in, in_cap, to_dev(in_index, in_cap), out, g, out_index->bitmap);
  D3B_LAUNCH_CHECK();
  D3B_CUDA(cudaMemsetAsync(block_sums, 0xff, (size_t)n_blocks * 4, stream));       // -1 = "not published yet"
  rb_scan_fused<<<n_blocks, kScanThreads, 0, stream>>>(out_index->bitmap, n_words, block_sums, out_cap, n_out,
                                                       out_index->word_prefix);
  D3B_LAUNCH_CHECK();
  rb_emit_coors<<<grid_for(n_words, 256), 256, 0, stream>>>(out_index->bitmap, out_index->word_prefix, n_words, out,
                                                           out_cap, out_coors);
  D3B_LAUNCH_CHECK();
  rb_neighbours<<<grid_for((long long)out_cap * g.kvol, 256), 256, 0, stream>>>(
      out_coors, n_out, out_cap, out, to_dev(in_index, in_cap), g, nbr, tile_mask);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}
