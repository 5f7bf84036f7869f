// Output-stationary sparse convolution, fp32 FFMA variant, + dense scatter.
//
//   out[o,:] = act((sum_k in[nbr[k][o],:] . W[k] + bias) * scale + shift + residual[o,:])
//
// replaces spconv v1.x indice_conv (per offset: gather rows -> torch.mm ->
// scatter-add) and the BatchNorm1d(eval)/ReLU/residual that follow every conv
// in det3d/models/backbones/scn.py:73-89,106-157.  One CTA owns 128 output
// rows, walks the kernel offsets that have at least one neighbour in the tile
// (tile_mask), gathers the input rows into shared memory and accumulates in
// registers; the epilogue is fused, nothing is scattered and no atomics are
// used, so the result is deterministic.
//
// This variant serves the layers the tensor-core kernel does not take (C_in
// not a multiple of 8, e.g. the 4/5-channel input layer) and is the
// in-library cross-check of the tensor-core kernel.
#include "common.cuh"

namespace d3b {

int sparse_conv_tc(const float* feat_in, const int32_t* nbr, const uint32_t* tile_mask,
                   const int32_t* n_out, int32_t out_cap, const d3b_conv_params* p,
                   float* feat_out, cudaStream_t stream);

constexpr int kTileM = 128;
constexpr int kSimtThreads = 256;
constexpr int kChunk = 16;  // input channels staged per step

template <int COUT>
__global__ void __launch_bounds__(kSimtThreads)
spconv_simt_kernel(const float* __restrict__ feat_in, const int* __restrict__ nbr,
                   const unsigned int* __restrict__ tile_mask, const int* __restrict__ n_out_p,
                   int out_cap, int c_in, int k_vol, const float* __restrict__ weight,
                   const float* __restrict__ bias, const float* __restrict__ scale,
                   const float* __restrict__ shift, const float* __restrict__ residual, int relu,
                   float* __restrict__ feat_out) {
  constexpr int CG = COUT / 4;             // column groups of 4
  constexpr int RG = kSimtThreads / CG;    // row groups
  constexpr int RPT = kTileM / RG;         // rows per thread
  __shared__ float As[kTileM][kChunk + 1];
  __shared__ __align__(16) float Ws[kChunk][COUT];
  __shared__ int nbr_s[kTileM];

  const int n_out = min(*n_out_p, out_cap);
  const int n_tiles = (n_out + kTileM - 1) / kTileM;
  const int cg = threadIdx.x % CG, rg = threadIdx.x / CG;

  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int row0 = tile * kTileM;
    float acc[RPT][4];
#pragma unroll
    for (int j = 0; j < RPT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0f;

    unsigned int mask = tile_mask[tile];
    while (mask) {
      const int k = __ffs(mask) - 1;
      mask &= mask - 1;
      __syncthreads();  // previous offset's readers are done with nbr_s / As / Ws
      if (threadIdx.x < kTileM) {
        const int o = row0 + threadIdx.x;
        nbr_s[threadIdx.x] = o < n_out ? nbr[(size_t)k * out_cap + o] : -1;
      }
      for (int c0 = 0; c0 < c_in; c0 += kChunk) {
        const int cw = min(kChunk, c_in - c0);
        __syncthreads();
        for (int idx = threadIdx.x; idx < kTileM * kChunk; idx += kSimtThreads) {
          const int r = idx / kChunk, c = idx % kChunk;
          const int src = nbr_s[r];
          As[r][c] = (src >= 0 && c < cw) ? feat_in[(size_t)src * c_in + c0 + c] : 0.0f;
        }
        for (int idx = threadIdx.x; idx < kChunk * COUT; idx += kSimtThreads) {
          const int c = idx / COUT, n = idx % COUT;
          Ws[c][n] = c < cw ? weight[((size_t)k * c_in + c0 + c) * COUT + n] : 0.0f;
        }
        __syncthreads();
#pragma unroll 4
        for (int c = 0; c < kChunk; ++c) {
          const float4 w = *reinterpret_cast<const float4*>(&Ws[c][cg * 4]);
#pragma unroll
          for (int j = 0; j < RPT; ++j) {
            const float a = As[rg + j * RG][c];
            acc[j][0] = fmaf(a, w.x, acc[j][0]);
            acc[j][1] = fmaf(a, w.y, acc[j][1]);
            acc[j][2] = fmaf(a, w.z, acc[j][2]);
            acc[j][3] = fmaf(a, w.w, acc[j][3]);
          }
        }
      }
    }
    // fused epilogue
    const int col = cg * 4;
    float4 b4 = bias ? *reinterpret_cast<const float4*>(bias + col) : make_float4(0, 0, 0, 0);
    float4 s4 = scale ? *reinterpret_cast<const float4*>(scale + col) : make_float4(1, 1, 1, 1);
    float4 t4 = shift ? *reinterpret_cast<const float4*>(shift + col) : make_float4(0, 0, 0, 0);
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const int o = row0 + rg + j * RG;
      if (o >= n_out) continue;
      float4 v;
      v.x = fmaf(acc[j][0] + b4.x, s4.x, t4.x);
      v.y = fmaf(acc[j][1] + b4.y, s4.y, t4.y);
      v.z = fmaf(acc[j][2] + b4.z, s4.z, t4.z);
      v.w = fmaf(acc[j][3] + b4.w, s4.w, t4.w);
      if (residual) {
        const float4 r = *reinterpret_cast<const float4*>(residual + (size_t)o * COUT + col);
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      if (relu) {
        v.x = fmaxf(v.x, 0.0f); v.y = fmaxf(v.y, 0.0f); v.z = fmaxf(v.z, 0.0f); v.w = fmaxf(v.w, 0.0f);
      }
      *reinterpret_cast<float4*>(feat_out + (size_t)o * COUT + col) = v;
    }
  }
}

template <int COUT>
static int launch_simt(const float* feat_in, const int32_t* nbr, const uint32_t* tile_mask,
                       const int32_t* n_out, int32_t out_cap, const d3b_conv_params* p,
                       float* feat_out, cudaStream_t stream) {
  const int n_tiles = div_up(out_cap, kTileM);
  const int grid = n_tiles < kNumSMs * 4 ? (n_tiles > 0 ? n_tiles : 1) : kNumSMs * 4;
  spconv_simt_kernel<COUT><<<grid, kSimtThreads, 0, stream>>>(
      feat_in, nbr, tile_mask, n_out, out_cap, p->c_in, p->k_vol, p->weight, p->bias, p->scale,
      p->shift, p->residual, p->relu, feat_out);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

// ---- dense scatter ----------------------------------------------------------------
// rows [n, C] -> out [B, C, D, H, W] (pre-zeroed).  Thread per (row, channel);
// a warp covers 32 channels of one row: coalesced reads, strided 4-byte writes
// (one per channel plane) -- the write pattern NCDHW imposes.
__global__ void __launch_bounds__(256)
sparse_to_dense_kernel(const float* __restrict__ feat, const int* __restrict__ coors,
                       const int* __restrict__ n_rows, int row_cap, int C, int D, int H, int W,
                       int B, float* __restrict__ out) {
  const int n = min(*n_rows, row_cap);
  const long long total = (long long)n * C;
  const size_t plane = (size_t)D * H * W;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / C), c = (int)(e - (long long)r * C);
    const int4 q = *reinterpret_cast<const int4*>(coors + (size_t)r * 4);
    if ((unsigned)q.x >= (unsigned)B || (unsigned)q.y >= (unsigned)D || (unsigned)q.z >= (unsigned)H ||
        (unsigned)q.w >= (unsigned)W)
      continue;
    out[((size_t)q.x * C + c) * plane + ((size_t)q.y * H + q.z) * W + q.w] = feat[e];
  }
}

// rows [n, C] -> channels-last BEV rows [B*H*W, C*D] (pre-zeroed), channel = c*D + z.
__global__ void __launch_bounds__(256)
sparse_to_bev_rows_kernel(const float* __restrict__ feat, const int* __restrict__ coors,
                          const int* __restrict__ n_rows, int row_cap, int C, int D, int H, int W, int B,
                          float* __restrict__ out) {
  const int n = min(*n_rows, row_cap);
  const long long total = (long long)n * C;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / C), c = (int)(e - (long long)r * C);
    const int4 q = *reinterpret_cast<const int4*>(coors + (size_t)r * 4);
    if ((unsigned)q.x >= (unsigned)B || (unsigned)q.y >= (unsigned)D || (unsigned)q.z >= (unsigned)H ||
        (unsigned)q.w >= (unsigned)W)
      continue;
    out[(((size_t)q.x * H + q.z) * W + q.w) * ((size_t)C * D) + (size_t)c * D + q.y] = feat[e];
  }
}

__global__ void __launch_bounds__(256)
dense2d_rulebook_kernel(int B, int H, int W, int kh, int kw, int ph, int pw, int* __restrict__ nbr,
                        unsigned int* __restrict__ tile_mask, int* __restrict__ n_rows) {
  const int n = B * H * W;
  const int kvol = kh * kw;
  if (blockIdx.x == 0 && threadIdx.x == 0) { n_rows[0] = n; n_rows[1] = n; }
  const long long total = (long long)n * kvol;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(e / n), row = (int)(e - (long long)k * n);
    const int x = row % W, y = (row / W) % H, b = row / (W * H);
    const int yy = y + k / kw - ph, xx = x + k % kw - pw;
    const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
    nbr[e] = ok ? (b * H + yy) * W + xx : -1;
  }
  const unsigned int full = kvol >= 32 ? 0xffffffffu : ((1u << kvol) - 1u);
  const int tiles = (n + kTileM - 1) / kTileM;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < tiles; t += gridDim.x * blockDim.x) tile_mask[t] = full;
}

}  // namespace d3b

using namespace d3b;

extern "C" int d3b_sparse_to_bev_rows(const float* feat, const int32_t* coors, const int32_t* n_rows,
                                      int32_t row_cap, int32_t channels, const int32_t spatial[3],
                                      int32_t batch, float* out_rows, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(feat && coors && n_rows && spatial && out_rows, "d3b_sparse_to_bev_rows: null argument");
  D3B_REQUIRE(channels >= 1 && batch >= 1 && row_cap >= 0, "d3b_sparse_to_bev_rows: bad shape");
  if (row_cap == 0) return D3B_OK;
  sparse_to_bev_rows_kernel<<<grid_for((long long)row_cap * channels, 256), 256, 0, stream>>>(
      feat, coors, n_rows, row_cap, channels, spatial[0], spatial[1], spatial[2], batch, out_rows);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_rulebook_dense2d(int32_t batch, int32_t height, int32_t width, const int32_t ksize[2],
                                    const int32_t padding[2], int32_t* nbr, uint32_t* tile_mask,
                                    int32_t* n_rows, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(ksize && padding && nbr && tile_mask && n_rows, "d3b_rulebook_dense2d: null argument");
  D3B_REQUIRE(batch >= 1 && height >= 1 && width >= 1 && ksize[0] >= 1 && ksize[1] >= 1 &&
                  ksize[0] * ksize[1] <= 32 && (long long)batch * height * width < (1ll << 31),
              "d3b_rulebook_dense2d: bad shape");
  const long long total = (long long)batch * height * width * ksize[0] * ksize[1];
  dense2d_rulebook_kernel<<<grid_for(total, 256), 256, 0, stream>>>(batch, height, width, ksize[0], ksize[1],
                                                                 padding[0], padding[1], nbr, tile_mask, n_rows);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_sparse_conv(const float* feat_in, const int32_t* nbr, const uint32_t* tile_mask,
                               const int32_t* n_out, int32_t out_cap, const d3b_conv_params* p,
                               float* feat_out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(feat_in && n_out && p && feat_out, "d3b_sparse_conv: null argument");
  D3B_REQUIRE(p->algo == D3B_ALGO_SIMT || p->algo == D3B_ALGO_TC, "d3b_sparse_conv: unknown algo %d", p->algo);
  D3B_REQUIRE(nbr && tile_mask, "d3b_sparse_conv: null rulebook");
  D3B_REQUIRE(p->c_in >= 1 && p->c_out >= 1 && p->k_vol >= 1 && p->k_vol <= 32 && out_cap >= 0,
              "d3b_sparse_conv: bad shape (c_in %d c_out %d k_vol %d)", p->c_in, p->c_out, p->k_vol);
  if (out_cap == 0) return D3B_OK;
  if (p->algo == D3B_ALGO_TC) return sparse_conv_tc(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
  D3B_REQUIRE(p->weight, "d3b_sparse_conv: null weight");
  switch (p->c_out) {
    case 16: return launch_simt<16>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
    case 32: return launch_simt<32>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
    case 64: return launch_simt<64>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
    case 128: return launch_simt<128>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
    default:
      set_error("d3b_sparse_conv: c_out %d not in {16,32,64,128}", p->c_out);
      return D3B_ERR_UNSUPPORTED;
  }
}

extern "C" int d3b_sparse_to_dense(const float* feat, const int32_t* coors, const int32_t* n_rows,
                                   int32_t row_cap, int32_t channels, const int32_t spatial[3],
                                   int32_t batch, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(feat && coors && n_rows && spatial && out, "d3b_sparse_to_dense: null argument");
  D3B_REQUIRE(channels >= 1 && batch >= 1 && row_cap >= 0, "d3b_sparse_to_dense: bad shape");
  if (row_cap == 0) return D3B_OK;
  sparse_to_dense_kernel<<<grid_for((long long)row_cap * channels, 256), 256, 0, stream>>>(
      feat, coors, n_rows, row_cap, channels, spatial[0], spatial[1], spatial[2], batch, out);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}
