// Dense BEV convolutions (RPN blocks, deblocks, task heads) as implicit GEMMs on the Hopper tensor cores, sm_90a.
//
// Reference: det3d/models/necks/rpn.py:82-159 (ZeroPad2d + Conv2d 3x3 [stride s] + BN + ReLU, n x (Conv2d 3x3 + BN +
// ReLU), deblock = Conv2d 1x1 / ConvTranspose2d(k = s, stride = s) + BN + ReLU, channel concat) and the 1x1 heads of
// det3d/models/bbox_heads/mg_head.py:198-230 -- fp32 cuDNN there.
//
//  * Activations are NHWC f16 planes (hi = f16(x), lo = f16(x - hi), see spconv16_sm90.cu), loaded by TMA with a 4-D
//    tensor map (C, W, H, B): box = 64 channels x 8 pixels x (16 + K - 1) rows, 128-byte swizzle, out-of-bounds
//    coordinates (the conv's zero padding, image borders, other samples) zero-filled by the TMA unit.  No thread
//    touches an activation on its way to the tensor core.
//  * Tile = 16 x 16 output pixels x C_out: two halves of 16 rows x 8 columns that share every weight stage, one
//    consumer warpgroup each, as two wgmma M = 64 blocks (8 rows x 8 columns).  In a patch, eight consecutive 128-byte
//    rows are one image row segment, so the matrix for kernel row ky is the SAME staged patch with the descriptor
//    start advanced by ky * 1024 bytes: one patch load per (kx, 64 channels) serves three (ky, kx) offsets.
//  * FP16x3: per k-step three MMAs (A_lo.B_hi, A_hi.B_lo, A_hi.B_hi) with fp32 accumulation in registers -- but only
//    across ONE kernel offset (<= 12 MMAs) into a fresh partial: the tensor core truncates on every accumulation, and
//    chaining all 216 MMAs of a 3x3x128 reduction into one accumulator shrinks the outputs in proportion to the chain
//    length, which 20 layers turn into > 1e-4.  The partial is scaled by 1 + n * 2^-26 (the mean truncation of its
//    n MMAs) and added into the running fp32 sums with round-to-nearest; at the end of the tile the epilogue applies
//    bias / BN / ReLU and writes the f16 planes.
//  * Warp roles: 8 consumer warps (wgmma + epilogue), 1 TMA warp; A ring of 2 stages (4 patches each), B ring of 2..4
//    stages, all mbarrier-driven; persistent grid.
//  * stride 2 (RPN down-sampling blocks): the box is loaded with elementStrides = 2, one load per (ky, kx).
//  * groups: several weight blocks over the same input in one launch -- C_out = 256 as two N = 128 passes, and
//    ConvTranspose2d(k = s, stride = s) as s*s 1x1 convolutions whose epilogues write pixel (y*s + dy, x*s + dx)
//    into a channel slice of the concat buffer.
//
// Bound: tensor pipe (f16).  fp32-equivalent flops per launch = 2 * B*H*W * K*K * C_in * C_out; the pipe
// executes 3x that.  Algorithmic bytes = B*H*W*(C_in + C_out)*4 + K*K*C_in*C_out*4.
#include <cuda.h>

#include "gmma.cuh"

namespace d3b {

struct BvEpi {          // same fields as spconv16_sm90.cu (kept local: the two kernels are separate TUs)
  const float* bias;
  const float* scale;
  const float* shift;
  float acc_scale;
  int relu;
};

constexpr int kBvTileY = 16, kBvTileX = 16;     // output pixels per tile
constexpr int kBvHalfX = 8;                     // one half = 16 rows x 8 columns = two wgmma M = 64 blocks
constexpr int kBvKc = 64;                       // channels per stage (128 bytes of f16)
constexpr int kBvMathWarps = 8;                 // warps 0..7: consumer warpgroup `half`
constexpr int kBvTmaWarp = kBvMathWarps;        // first warp of the producer warpgroup (warps 8..11)
constexpr int kBvThreads = 32 * (kBvMathWarps + 4);   // 384 (registers are allocated per warpgroup: 168 each)
constexpr int kBvAStages = 2;

template <int KS, int STRIDE, int COUT>
struct BvCfg {
  static constexpr int kPatchRows = STRIDE == 1 ? kBvTileY + KS - 1 : kBvTileY;      // rows in one staged patch
  static constexpr int kPatchBytes = kPatchRows * kBvHalfX * 128;
  static constexpr int kAStageBytes = 4 * kPatchBytes;                                // {half 0, half 1} x {hi, lo}
  static constexpr int kBBytes = 2 * COUT * 128;                                      // [B_hi rows | B_lo rows]
  static constexpr int kBStages = COUT >= 128 ? 2 : 4;
  static constexpr int kSmemBytes = kBvAStages * kAStageBytes + kBStages * kBBytes + 1024 + 256;
  // with stride 1 one A stage serves the KS kernel rows of a (kx, kb); with stride 2 every (ky, kx) has its own
  static constexpr int kRowsPerAStage = STRIDE == 1 ? KS : 1;
  // partials are computed in column passes of kPassN outputs (C_out = 128: two, so that sums + partial fit registers)
  static constexpr int kPassN = COUT >= 128 ? 64 : COUT;
};

struct BvGeom {
  int batch, h_out, w_out;        // conv output grid
  int c_in, n_kb;
  int pad;
  int tiles_y, tiles_x;           // per sample
  int groups, cgroups;            // weight blocks; cgroups of them tile the output channels, the rest are (uy, ux)
  int up;                         // output pixel = (y*up + uy, x*up + ux)
  int out_h, out_w;               // output tensor grid (h_out*up, w_out*up)
  int out_channels, out_c0;       // row length of the output tensor and first channel written
  int seq;                        // launch counter of this translation unit (development traces only)
};

__device__ __forceinline__ uint32_t bv_pack_half2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// mean truncation of one partial: three MMAs per k-step of one (kernel offset, 64-channel slice)
__device__ __forceinline__ float bv_trunc_fix(int n_ks) { return 1.f + 3.f * (float)n_ks * kTruncLossPerMma; }

template <int KS, int STRIDE, int COUT>
__global__ void __launch_bounds__(kBvThreads, 1)
bev_conv16_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, BvGeom g,
                  const __half* __restrict__ packed, BvEpi epi, __half* __restrict__ out_hi,
                  __half* __restrict__ out_lo, float* __restrict__ out_f32, int* __restrict__ overflow) {
  using Cfg = BvCfg<KS, STRIDE, COUT>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + kBvAStages * Cfg::kAStageBytes;
  const uint32_t bar_base = b_base + Cfg::kBStages * Cfg::kBBytes;
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (kBvAStages + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (2 * kBvAStages + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (2 * kBvAStages + Cfg::kBStages + s); };

  D3B_CTA_MARK(0, g.seq);
  pdl_launch_dependents();           // the next kernel of the stream may start its prologue behind this one's tail
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_group = g.batch * g.tiles_y * g.tiles_x;
  const int n_tiles = tiles_per_group * g.groups;
  const int k_vol = KS * KS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kBvAStages; ++s) { mbar_init(a_full(s), 1); mbar_init(a_empty(s), kBvMathWarps); }
    for (int s = 0; s < Cfg::kBStages; ++s) { mbar_init(b_full(s), 1); mbar_init(b_empty(s), kBvMathWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tm_hi);
    tma_prefetch_desc(&tm_lo);
  }
  __syncthreads();
  pdl_wait_prior_grid();             // everything below reads the previous layer's planes or writes buffers it may still read

  // tile -> (group, sample, y0, x0)
  auto decode = [&](int tile, int& grp, int& b, int& y0, int& x0) {
    grp = tile / tiles_per_group;
    int t = tile - grp * tiles_per_group;
    b = t / (g.tiles_y * g.tiles_x);
    t -= b * g.tiles_y * g.tiles_x;
    y0 = (t / g.tiles_x) * kBvTileY;
    x0 = (t % g.tiles_x) * kBvTileX;
  };

  if (warp >= kBvTmaWarp) {
    // ===================== TMA producer (one elected lane) =====================
    if (warp == kBvTmaWarp && lane == 0) {
      uint32_t a_it = 0, b_it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int grp, b, y0, x0;
        decode(tile, grp, b, y0, x0);
        const __half* wgrp = packed + (size_t)grp * k_vol * g.n_kb * (Cfg::kBBytes / 2);
        for (int kb = 0; kb < g.n_kb; ++kb) {
          for (int kx = 0; kx < KS; ++kx) {
            for (int ky0 = 0; ky0 < KS; ky0 += Cfg::kRowsPerAStage) {
              // ---- A stage: {half 0, half 1} x {hi, lo} patches ----
              const int sa = a_it % kBvAStages;
              D3B_STAMP(0, a_it);
              D3B_WAIT(a_empty(sa), ((a_it / kBvAStages) & 1u) ^ 1u, 1);
              mbar_arrive_expect_tx(a_full(sa), Cfg::kAStageBytes);
              const uint32_t dst = a_base + sa * Cfg::kAStageBytes;
              const int cy = STRIDE == 1 ? y0 - g.pad : y0 * STRIDE + ky0 - g.pad;
#pragma unroll
              for (int half = 0; half < 2; ++half) {
                const int cx = (x0 + half * kBvHalfX) * STRIDE + kx - g.pad;
                tma_load_4d(dst + (2 * half) * Cfg::kPatchBytes, &tm_hi, kb * kBvKc, cx, cy, b, a_full(sa));
                tma_load_4d(dst + (2 * half + 1) * Cfg::kPatchBytes, &tm_lo, kb * kBvKc, cx, cy, b, a_full(sa));
              }
              D3B_STAMP(1, a_it);
              ++a_it;
              // ---- B stages: one per kernel row served by this A stage ----
              for (int r = 0; r < Cfg::kRowsPerAStage; ++r) {
                const int ky = ky0 + r;
                const int sb = b_it % Cfg::kBStages;
                D3B_STAMP(2, b_it);
                D3B_WAIT(b_empty(sb), ((b_it / Cfg::kBStages) & 1u) ^ 1u, 2);
                mbar_arrive_expect_tx(b_full(sb), Cfg::kBBytes);
                tma_bulk_g2s(b_base + sb * Cfg::kBBytes,
                             wgrp + ((size_t)(ky * KS + kx) * g.n_kb + kb) * (Cfg::kBBytes / 2), Cfg::kBBytes, b_full(sb));
                D3B_STAMP(3, b_it);
                ++b_it;
              }
            }
          }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups: warps 0-3 -> half 0, warps 4-7 -> half 1 =====================
    const int half = warp >> 2, wq = warp & 3;
    bool ovf = false;
    uint32_t a_it = 0, b_it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      int grp, b, y0, x0;
      decode(tile, grp, b, y0, x0);
      float acc[2][COUT / 2];                   // wgmma M = 64 blocks: tile rows [0, 8) and [8, 16) of the half
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int q = 0; q < COUT / 2; ++q) acc[m][q] = 0.f;
      for (int kb = 0; kb < g.n_kb; ++kb) {
        const int n_ks = min(kBvKc / 16, (g.c_in - kb * kBvKc + 15) / 16);
        const float f_fix = bv_trunc_fix(n_ks);
        for (int kx = 0; kx < KS; ++kx) {
          for (int ky0 = 0; ky0 < KS; ky0 += Cfg::kRowsPerAStage) {
            const int sa = a_it % kBvAStages;
            if (warp == 0 && lane == 0) D3B_STAMP(4, a_it);
            D3B_WAIT(a_full(sa), (a_it / kBvAStages) & 1u, 4);
            if (warp == 0 && lane == 0) D3B_STAMP(5, a_it);
            for (int r = 0; r < Cfg::kRowsPerAStage; ++r, ++b_it) {
              const int sb = b_it % Cfg::kBStages;
              D3B_WAIT(b_full(sb), (b_it / Cfg::kBStages) & 1u, 5);
              if (warp == 0 && lane == 0) D3B_STAMP(6, b_it);
              const uint32_t b_hi = b_base + sb * Cfg::kBBytes, b_lo = b_hi + COUT * 128;
              // stride 1: kernel row r of the staged patch = the same bytes 8 rows (1024 B) further down
              const uint32_t row_adv = STRIDE == 1 ? (uint32_t)(ky0 + r) * 1024u : 0u;
              const uint32_t ah = a_base + sa * Cfg::kAStageBytes + (2 * half) * Cfg::kPatchBytes + row_adv;
#pragma unroll
              for (int m = 0; m < 2; ++m) {
                const uint32_t a_hi = ah + m * 8192u, a_lo = a_hi + Cfg::kPatchBytes;
#pragma unroll
                for (int np = 0; np < COUT / Cfg::kPassN; ++np) {
                  const uint32_t nb = np * Cfg::kPassN * 128;     // first B row of this column pass
                  float part[Cfg::kPassN / 2];
                  gmma_fence();
                  // always the full 64 channels: past C_in the TMA box is zero-filled and the packed weights are zero, so
                  // those MMAs add exact zeros -- and a uniform batch keeps the wgmmas from being serialised
#pragma unroll
                  for (int ks = 0; ks < kBvKc / 16; ++ks) {
                    const uint32_t adv = ks * 32;     // 32 bytes along K
                    // small terms first, the dominant hi.hi product last
                    wgmma_f16<Cfg::kPassN>(part, gmma_desc_sw128(a_lo + adv), gmma_desc_sw128(b_hi + nb + adv), ks > 0 ? 1u : 0u);
                    wgmma_f16<Cfg::kPassN>(part, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_lo + nb + adv), 1u);
                    wgmma_f16<Cfg::kPassN>(part, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_hi + nb + adv), 1u);
                  }
                  gmma_commit();
                  gmma_wait();
                  gmma_fence_regs(part);
#pragma unroll
                  for (int q = 0; q < Cfg::kPassN / 2; ++q)
                    acc[m][np * Cfg::kPassN / 2 + q] = fmaf(part[q], f_fix, acc[m][np * Cfg::kPassN / 2 + q]);
                }
              }
              __syncwarp();
              if (lane == 0) mbar_arrive(b_empty(sb));
              if (warp == 0 && lane == 0) D3B_STAMP(7, b_it);
            }
            if (lane == 0) mbar_arrive(a_empty(sa));
            ++a_it;
          }
        }
      }
      const int cg = grp % g.cgroups, ug = grp / g.cgroups;
      const int pcol = grp * COUT;              // per-group epilogue parameters are laid out group-major
#pragma unroll
      for (int m = 0; m < 2; ++m) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int y = y0 + 8 * m + 2 * wq + h, x = x0 + half * kBvHalfX + (lane >> 2);
          if (!(y < g.h_out && x < g.w_out)) continue;
          const int oy = y * g.up + ug / g.up, ox = x * g.up + ug % g.up;
          const size_t row_off = (((size_t)b * g.out_h + oy) * g.out_w + ox) * (size_t)g.out_channels + g.out_c0 + cg * COUT;
#pragma unroll
          for (int jn = 0; jn < COUT / 8; ++jn) {
            const int col = jn * 8 + 2 * (lane & 3);
            float v0 = acc[m][4 * jn + 2 * h] * epi.acc_scale, v1 = acc[m][4 * jn + 2 * h + 1] * epi.acc_scale;
            if (epi.bias) {
              const float2 bb = __ldg(reinterpret_cast<const float2*>(epi.bias + pcol + col));
              v0 += bb.x; v1 += bb.y;
            }
            if (epi.scale) {
              const float2 sc = __ldg(reinterpret_cast<const float2*>(epi.scale + pcol + col));
              const float2 sh = __ldg(reinterpret_cast<const float2*>(epi.shift + pcol + col));
              v0 = fmaf(v0, sc.x, sh.x); v1 = fmaf(v1, sc.y, sh.y);
            }
            if (epi.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (out_hi) {
              __half h0, l0, h1, l1;
              split_f16(v0, h0, l0);
              split_f16(v1, h1, l1);
              *reinterpret_cast<uint32_t*>(out_hi + row_off + col) = bv_pack_half2(h0, h1);
              *reinterpret_cast<uint32_t*>(out_lo + row_off + col) = bv_pack_half2(l0, l1);
              ovf |= !(fabsf(v0) < 65504.f) | !(fabsf(v1) < 65504.f);
            }
            if (out_f32) *reinterpret_cast<float2*>(out_f32 + row_off + col) = make_float2(v0, v1);
          }
        }
      }
    }
    if (ovf && overflow) atomicOr(overflow, 1);
  }
  D3B_CTA_MARK(1, g.seq);
}

// ======================================================================================================================
// Variant "channel-stationary" (3x3, stride 1, C_out = 128 per group, C_in % 64 == 0, up = 1): the GEMM is transposed,
//     D^T[C_out = 128 (M), 256 pixels (N)] += W[C_out, K16] . Act[256 pixels, K16]^T
// so each consumer warpgroup covers 64 channels of the 16 x 16 pixel tile in four N = 64 column passes: the weights
// are the A operand and pixels the N dimension.  Same products, same order, same partials and truncation correction as
// the pixel-stationary kernel.
//  * Activations: one TMA box per plane = 64 channels x 16 pixels x 18 rows: an image row is 2048 B (two swizzle groups),
//    pixel (r, x) of the tile is operand row r * 16 + x, kernel row ky = descriptor start + ky * 2048.
//  * Weights: the packed [W_hi | W_lo] image is K-major SW128 with C_out rows -- byte for byte usable as the A operand.
//  * Accumulators: a thread holds 2 channels x 64 pixels, so bias / BN parameters are per-thread scalars.
constexpr int kBwThreads = 384;                                   // warps 0..7 consumers, 8 activation TMA, 9 weights, 10..11 idle
constexpr int kBwActWarp = 8;
constexpr int kBwWeightWarp = 9;
constexpr int kBwCout = 128;
constexpr int kBwPatchRows = kBvTileY + 2;                        // 18
constexpr int kBwRowBytes = kBvTileX * 128;                       // one image row of the patch: 16 pixels x 128 B
constexpr int kBwPatchBytes = kBwPatchRows * kBwRowBytes;         // 36864
constexpr int kBwAStageBytes = 2 * kBwPatchBytes;                 // hi, lo
constexpr int kBwBBytes = 2 * kBwCout * 128;                      // [W_hi rows | W_lo rows]
constexpr int kBwBStages = 2;
constexpr int kBwPixels = kBvTileY * kBvTileX;                    // 256 pixel columns per tile
constexpr int kBwSmemBytes = kBvAStages * kBwAStageBytes + kBwBStages * kBwBBytes + 1024 + 256;

__global__ void __launch_bounds__(kBwThreads, 1)
bev_conv16_cs_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, BvGeom g,
                     const __half* __restrict__ packed, BvEpi epi, __half* __restrict__ out_hi,
                     __half* __restrict__ out_lo, float* __restrict__ out_f32, int* __restrict__ overflow) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + kBvAStages * kBwAStageBytes;
  const uint32_t bar_base = b_base + kBwBStages * kBwBBytes;
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (2 + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (4 + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (6 + s); };

  D3B_CTA_MARK(0, g.seq);
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_group = g.batch * g.tiles_y * g.tiles_x;
  const int n_tiles = tiles_per_group * g.groups;

  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(a_full(s), 1); mbar_init(a_empty(s), kBvMathWarps);
      mbar_init(b_full(s), 1); mbar_init(b_empty(s), kBvMathWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tm_hi);
    tma_prefetch_desc(&tm_lo);
  }
  __syncthreads();
  // (griddepcontrol.wait is executed by the threads that touch the previous layer's planes or write outputs: the activation
  // producer and the consumers; weight staging runs ahead of the previous grid's tail)

  auto decode = [&](int tile, int& grp, int& b, int& y0, int& x0) {
    grp = tile / tiles_per_group;
    int t = tile - grp * tiles_per_group;
    b = t / (g.tiles_y * g.tiles_x);
    t -= b * g.tiles_y * g.tiles_x;
    y0 = (t / g.tiles_x) * kBvTileY;
    x0 = (t % g.tiles_x) * kBvTileX;
  };

  if (warp == kBwActWarp) {
    // ===================== activation producer (TMA tensor loads) =====================
    // (Weights have their own producer warp: with one thread feeding both rings, the next patch load would queue up
    // behind a wait for a free weight stage.)
    if (lane == 0) {
      pdl_wait_prior_grid();           // the planes are the previous layer's output
      uint32_t a_it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int grp, b, y0, x0;
        decode(tile, grp, b, y0, x0);
        for (int kb = 0; kb < g.n_kb; ++kb) {
          for (int kx = 0; kx < 3; ++kx, ++a_it) {
            const int sa = a_it & 1;
            D3B_STAMP(0, a_it);
            D3B_WAIT(a_empty(sa), ((a_it >> 1) & 1u) ^ 1u, 1);
            mbar_arrive_expect_tx(a_full(sa), kBwAStageBytes);
            const uint32_t dst = a_base + sa * kBwAStageBytes;
            tma_load_4d(dst, &tm_hi, kb * kBvKc, x0 + kx - g.pad, y0 - g.pad, b, a_full(sa));
            tma_load_4d(dst + kBwPatchBytes, &tm_lo, kb * kBvKc, x0 + kx - g.pad, y0 - g.pad, b, a_full(sa));
            D3B_STAMP(1, a_it);
          }
        }
      }
    }
  } else if (warp == kBwWeightWarp) {
    // ===================== weight producer (bulk copies; weights do not depend on the previous grid) =====================
    if (lane == 0) {
      uint32_t b_it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int grp = tile / tiles_per_group;
        const __half* wgrp = packed + (size_t)grp * 9 * g.n_kb * (kBwBBytes / 2);
        for (int kb = 0; kb < g.n_kb; ++kb) {
          for (int kx = 0; kx < 3; ++kx) {
            for (int ky = 0; ky < 3; ++ky, ++b_it) {
              const int sb = b_it & 1;
              D3B_STAMP(2, b_it);
              D3B_WAIT(b_empty(sb), ((b_it >> 1) & 1u) ^ 1u, 2);
              mbar_arrive_expect_tx(b_full(sb), kBwBBytes);
              tma_bulk_g2s(b_base + sb * kBwBBytes, wgrp + ((size_t)(ky * 3 + kx) * g.n_kb + kb) * (kBwBBytes / 2),
                           kBwBBytes, b_full(sb));
              D3B_STAMP(3, b_it);
            }
          }
        }
      }
    }
  } else if (warp < kBvMathWarps) {
    // ===================== consumer warpgroups: warpgroup wg -> output channels [64 wg, 64 wg + 64) =====================
    pdl_wait_prior_grid();                              // (output buffers may still be read by earlier kernels)
    const int wg = warp >> 2, wq = warp & 3;
    const float f_fix = bv_trunc_fix(kBvKc / 16);      // (C_in % 64 == 0: four k-steps per offset and slice)
    bool ovf = false;
    uint32_t a_it = 0, b_it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      int grp, b, y0, x0;
      decode(tile, grp, b, y0, x0);
      float acc[kBwPixels / 2];
#pragma unroll
      for (int q = 0; q < kBwPixels / 2; ++q) acc[q] = 0.f;
      for (int kb = 0; kb < g.n_kb; ++kb) {
        for (int kx = 0; kx < 3; ++kx, ++a_it) {
          const uint32_t sa = a_it & 1u;
          if (warp == 0 && lane == 0) D3B_STAMP(4, a_it);
          D3B_WAIT(a_full(sa), (a_it >> 1) & 1u, 4);
          if (warp == 0 && lane == 0) D3B_STAMP(5, a_it);
          for (int ky = 0; ky < 3; ++ky, ++b_it) {
            const uint32_t sb = b_it & 1u;
            D3B_WAIT(b_full(sb), (b_it >> 1) & 1u, 5);
            if (warp == 0 && lane == 0) D3B_STAMP(6, b_it);
            const uint32_t w_hi = b_base + sb * kBwBBytes + wg * 8192u, w_lo = w_hi + kBwCout * 128;
            const uint32_t x_hi = a_base + sa * kBwAStageBytes + (uint32_t)ky * kBwRowBytes, x_lo = x_hi + kBwPatchBytes;
#pragma unroll
            for (int nh = 0; nh < 4; ++nh) {            // pixels [64 nh, 64 nh + 64): tile rows [4 nh, 4 nh + 4)
              const uint32_t xo = nh * 64 * 128;
              float part[32];
              gmma_fence();
#pragma unroll
              for (int ks = 0; ks < kBvKc / 16; ++ks) {
                const uint32_t adv = ks * 32;
                // small terms first, the dominant hi.hi product last (the order of the pixel-stationary kernel)
                wgmma_f16<64>(part, gmma_desc_sw128(w_hi + adv), gmma_desc_sw128(x_lo + xo + adv), ks > 0 ? 1u : 0u);
                wgmma_f16<64>(part, gmma_desc_sw128(w_lo + adv), gmma_desc_sw128(x_hi + xo + adv), 1u);
                wgmma_f16<64>(part, gmma_desc_sw128(w_hi + adv), gmma_desc_sw128(x_hi + xo + adv), 1u);
              }
              gmma_commit();
              gmma_wait();
              gmma_fence_regs(part);
#pragma unroll
              for (int q = 0; q < 32; ++q) acc[nh * 32 + q] = fmaf(part[q], f_fix, acc[nh * 32 + q]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(b_empty(sb));
            if (warp == 0 && lane == 0) D3B_STAMP(7, b_it);
          }
          if (lane == 0) mbar_arrive(a_empty(sa));
        }
      }
      // ---- epilogue: per-channel scalars; a thread holds channels ch, ch + 8 of pixels 8 jn + 2 (lane % 4) + {0, 1} ----
      const int cg = grp % g.cgroups;
      const size_t chan0 = (size_t)g.out_c0 + (size_t)cg * kBwCout;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ch = wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        const int pcol = grp * kBwCout + ch;
        const float e_bias = epi.bias ? __ldg(epi.bias + pcol) : 0.f;
        const float e_scale = epi.scale ? __ldg(epi.scale + pcol) : 1.f;
        const float e_shift = epi.scale ? __ldg(epi.shift + pcol) : 0.f;
#pragma unroll
        for (int jn = 0; jn < kBwPixels / 8; ++jn) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int p = jn * 8 + 2 * (lane & 3) + c;
            const int y = y0 + (p >> 4), x = x0 + (p & 15);
            float v = acc[4 * jn + 2 * h + c] * epi.acc_scale;
            if (epi.bias) v += e_bias;
            if (epi.scale) v = fmaf(v, e_scale, e_shift);
            if (epi.relu) v = fmaxf(v, 0.f);
            if (!(y < g.h_out && x < g.w_out)) continue;
            const size_t off = (((size_t)b * g.out_h + y) * g.out_w + x) * (size_t)g.out_channels + chan0 + ch;
            if (out_hi) {
              __half hh, ll;
              split_f16(v, hh, ll);
              out_hi[off] = hh;
              out_lo[off] = ll;
              ovf |= !(fabsf(v) < 65504.f);
            }
            if (out_f32) out_f32[off] = v;
          }
        }
      }
    }
    if (ovf && overflow) atomicOr(overflow, 1);
  }
  D3B_CTA_MARK(1, g.seq);
}

// ---- host side: tensor maps through the driver entry point (libcuda is not linked: CPU hosts must dlopen us) ----------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
  static std::atomic<void*> cached{nullptr};
  void* fn = cached.load(std::memory_order_acquire);
  if (fn == nullptr) {
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    cached.store(fn, std::memory_order_release);
  }
  return (EncodeTiledFn)fn;
}

// planes [B, H, W, C] f16 -> map with box (64 channels, box_w pixels, box_h rows, 1 sample), 128B swizzle, zero OOB fill
static int make_map(CUtensorMap* map, const void* base, int batch, int h, int w, int c, int box_w, int box_h, int stride) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (enc == nullptr) {
    set_error("cuTensorMapEncodeTiled is not available from this driver");
    return D3B_ERR_CUDA;
  }
  const cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)batch};
  const cuuint64_t strides[3] = {(cuuint64_t)c * 2, (cuuint64_t)w * c * 2, (cuuint64_t)h * w * c * 2};
  // with a traversal stride s the box spans (n - 1) * s + 1 tensor elements to deliver n of them
  const cuuint32_t box[4] = {(cuuint32_t)kBvKc, (cuuint32_t)((box_w - 1) * stride + 1), (cuuint32_t)((box_h - 1) * stride + 1), 1u};
  const cuuint32_t estr[4] = {1u, (cuuint32_t)stride, (cuuint32_t)stride, 1u};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) for planes [%d,%d,%d,%d] box [%d,%d] stride %d", (int)r, batch, h, w, c,
              box_w, box_h, stride);
    return D3B_ERR_CUDA;
  }
  return D3B_OK;
}

template <int KS, int STRIDE, int COUT>
static int launch_bev(const d3b_bev16_params* p, const BvGeom& g, cudaStream_t stream) {
  using Cfg = BvCfg<KS, STRIDE, COUT>;
  static SmemOptIn optin;
  D3B_CUDA(ensure_dynamic_smem(bev_conv16_kernel<KS, STRIDE, COUT>, Cfg::kSmemBytes, optin));
  CUtensorMap tm_hi, tm_lo;
  int st = make_map(&tm_hi, p->in_hi, p->batch, p->h_in, p->w_in, p->c_in, kBvHalfX, Cfg::kPatchRows, STRIDE);
  if (st != D3B_OK) return st;
  st = make_map(&tm_lo, p->in_lo, p->batch, p->h_in, p->w_in, p->c_in, kBvHalfX, Cfg::kPatchRows, STRIDE);
  if (st != D3B_OK) return st;
  BvEpi e;
  e.bias = p->bias; e.scale = p->scale; e.shift = p->shift; e.acc_scale = p->acc_scale; e.relu = p->relu;
  const int n_tiles = g.batch * g.tiles_y * g.tiles_x * g.groups;
  const int grid = n_tiles < kNumSMs ? n_tiles : kNumSMs;
  D3B_CUDA(launch_maybe_pdl(bev_conv16_kernel<KS, STRIDE, COUT>, dim3(grid), dim3(kBvThreads), Cfg::kSmemBytes, stream, tm_hi,
                            tm_lo, g, (const __half*)p->weight_packed, e, (__half*)p->out_hi, (__half*)p->out_lo, p->out_f32,
                            (int*)p->overflow));
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

// channel-stationary variant: 3x3, stride 1, one or more output blocks of exactly 128 channels, no sub-pixel groups
static int launch_bev_cs(const d3b_bev16_params* p, const BvGeom& g, cudaStream_t stream) {
  static SmemOptIn optin;
  D3B_CUDA(ensure_dynamic_smem(bev_conv16_cs_kernel, kBwSmemBytes, optin));
  CUtensorMap tm_hi, tm_lo;
  int st = make_map(&tm_hi, p->in_hi, p->batch, p->h_in, p->w_in, p->c_in, kBvTileX, kBwPatchRows, 1);
  if (st != D3B_OK) return st;
  st = make_map(&tm_lo, p->in_lo, p->batch, p->h_in, p->w_in, p->c_in, kBvTileX, kBwPatchRows, 1);
  if (st != D3B_OK) return st;
  BvEpi e;
  e.bias = p->bias; e.scale = p->scale; e.shift = p->shift; e.acc_scale = p->acc_scale; e.relu = p->relu;
  const int n_tiles = g.batch * g.tiles_y * g.tiles_x * g.groups;
  const int grid = n_tiles < kNumSMs ? n_tiles : kNumSMs;
  D3B_CUDA(launch_maybe_pdl(bev_conv16_cs_kernel, dim3(grid), dim3(kBwThreads), kBwSmemBytes, stream, tm_hi, tm_lo, g,
                            (const __half*)p->weight_packed, e, (__half*)p->out_hi, (__half*)p->out_lo, p->out_f32,
                            (int*)p->overflow));
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

}  // namespace d3b

using namespace d3b;

extern "C" int d3b_bev_conv16(const d3b_bev16_params* p, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(p && p->in_hi && p->in_lo && p->weight_packed, "d3b_bev_conv16: null argument");
  D3B_REQUIRE(p->batch >= 1 && p->h_in >= 1 && p->w_in >= 1 && p->c_in >= 16 && p->c_in % 16 == 0,
              "d3b_bev_conv16: bad input shape [%d,%d,%d,%d] (C_in must be a multiple of 16)", p->batch, p->h_in, p->w_in, p->c_in);
  D3B_REQUIRE((p->ksize == 1 || p->ksize == 3) && (p->stride == 1 || p->stride == 2) && !(p->ksize == 1 && p->stride != 1),
              "d3b_bev_conv16: ksize %d stride %d not built (3x3 s1/s2, 1x1 s1)", p->ksize, p->stride);
  D3B_REQUIRE(p->pad >= 0 && p->pad <= p->ksize / 2 + 1, "d3b_bev_conv16: pad %d", p->pad);
  D3B_REQUIRE(p->up >= 1 && p->up <= 4 && p->cgroups >= 1 && p->groups == p->cgroups * p->up * p->up,
              "d3b_bev_conv16: groups %d != cgroups %d * up^2 (up %d)", p->groups, p->cgroups, p->up);
  D3B_REQUIRE((p->out_hi != nullptr) == (p->out_lo != nullptr) && (p->out_hi || p->out_f32),
              "d3b_bev_conv16: give out_hi + out_lo and/or out_f32");
  D3B_REQUIRE((p->scale == nullptr) == (p->shift == nullptr), "d3b_bev_conv16: scale and shift go together");
  D3B_REQUIRE(p->out_channels % 8 == 0 && p->out_c0 % 8 == 0 && p->out_c0 + p->cgroups * p->c_out <= p->out_channels,
              "d3b_bev_conv16: output channel slice [%d, %d) does not fit rows of %d", p->out_c0,
              p->out_c0 + p->cgroups * p->c_out, p->out_channels);
  BvGeom g;
  g.batch = p->batch;
  g.h_out = (p->h_in + 2 * p->pad - p->ksize) / p->stride + 1;
  g.w_out = (p->w_in + 2 * p->pad - p->ksize) / p->stride + 1;
  D3B_REQUIRE(g.h_out >= 1 && g.w_out >= 1, "d3b_bev_conv16: empty output grid");
  g.c_in = p->c_in;
  g.n_kb = (p->c_in + kBvKc - 1) / kBvKc;
  g.pad = p->pad;
  g.tiles_y = div_up(g.h_out, kBvTileY);
  g.tiles_x = div_up(g.w_out, kBvTileX);
  g.groups = p->groups; g.cgroups = p->cgroups; g.up = p->up;
  g.out_h = g.h_out * p->up; g.out_w = g.w_out * p->up;
  g.out_channels = p->out_channels; g.out_c0 = p->out_c0;
  static std::atomic<int> launch_seq{0};
  g.seq = launch_seq.fetch_add(1, std::memory_order_relaxed);
  // Automatic (variant 2) = pixel-stationary: on the H100 it is the faster schedule (H100 80GB HBM3 at a 700 W limit,
  // PointPillars, B = 1, 20k points: dense 3x3 layers 4.0 ms/step pixel-stationary vs 5.4 ms channel-stationary; CBGS,
  // whose launches have fewer tiles than SMs, measured the same either way).  The channel-stationary kernel stays selectable (variant 1) and gives the same bits.
  const int variant = bev_variant();
  if (variant == 1 && p->ksize == 3 && p->stride == 1 && p->c_out == kBwCout &&
      p->c_in % kBvKc == 0 && p->up == 1 && p->out_channels % 4 == 0)
    return launch_bev_cs(p, g, stream);
#define D3B_BEV_CASE(KS, ST)                                                   \
  if (p->ksize == KS && p->stride == ST) {                                     \
    switch (p->c_out) {                                                        \
      case 32: return launch_bev<KS, ST, 32>(p, g, stream);                    \
      case 64: return launch_bev<KS, ST, 64>(p, g, stream);                    \
      case 128: return launch_bev<KS, ST, 128>(p, g, stream);                  \
      default: break;                                                          \
    }                                                                          \
  }
  D3B_BEV_CASE(3, 1)
  D3B_BEV_CASE(3, 2)
  D3B_BEV_CASE(1, 1)
#undef D3B_BEV_CASE
  set_error("d3b_bev_conv16: C_out per group %d not in {32, 64, 128}", p->c_out);
  return D3B_ERR_UNSUPPORTED;
}

#ifdef D3B_SOFT_TIMEOUT
extern "C" int d3b_debug_fault_bevconv16(unsigned int* host8) {
  cudaError_t e = cudaMemcpyFromSymbol(host8, d3b::g_d3b_fault, 32);
  unsigned int zeros[8] = {0};
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(d3b::g_d3b_fault, zeros, 32);
  return (int)e;
}
extern "C" int d3b_debug_cta_ns_bevconv16(unsigned long long* host4096) {
  return (int)cudaMemcpyFromSymbol(host4096, d3b::g_d3b_cta_ns, sizeof(unsigned long long) * 4096);
}
extern "C" int d3b_debug_cta_clk_bevconv16(long long* host4096) {
  return (int)cudaMemcpyFromSymbol(host4096, d3b::g_d3b_cta_clk, sizeof(long long) * 4096);
}
extern "C" int d3b_debug_trace_bevconv16(long long* host, int clear) {
  cudaError_t e = cudaMemcpyFromSymbol(host, d3b::g_d3b_trace, sizeof(long long) * 16 * 512);
  if (e == cudaSuccess && clear) {
    static long long zeros[16 * 512];
    e = cudaMemcpyToSymbol(d3b::g_d3b_trace, zeros, sizeof(zeros));
  }
  return (int)e;
}
#endif
