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
//    length, which 20 layers turn into > 1e-4.  The partial is added into the running fp32 sums with round-to-nearest;
//    at the end of the tile the epilogue scales the sums by 1 + n * 2^-26 (the mean truncation of n MMAs, gmma.cuh),
//    applies bias / BN / ReLU and writes the f16 planes.
//  * Warp roles: 8 consumer warps (wgmma + epilogue), 1 TMA warp; A ring of 2 stages (4 patches each), B ring of 2..4
//    stages, all mbarrier-driven; persistent grid.
//  * stride 2 (RPN down-sampling blocks): the box is loaded with elementStrides = 2, one load per (ky, kx).
//  * Conv2d(kernel = stride = s, pad 0), s in {2, 3, 4} (the deblock rpn.py builds for an up-sampling stride 1/s):
//    the same strided loads with elementStrides = s -- box (8-1)*s+1 columns x (16-1)*s+1 rows, at most 29 x 61 --
//    one A stage per (64 channels, kx, ky).  Output rows / columns past floor(H / s) are not formed, as in torch.
//  * groups: several weight blocks over the same input in one launch -- C_out = 256 as two N = 128 passes, and
//    ConvTranspose2d(k = s, stride = s) as s*s 1x1 convolutions whose epilogues write pixel (y*s + dy, x*s + dx)
//    into a channel slice of the concat buffer.
//
// Bound: tensor pipe (f16).  fp32-equivalent flops per launch = 2 * B*H*W * K*K * C_in * C_out; the pipe
// executes 3x that.  Algorithmic bytes = B*H*W*(C_in + C_out)*4 + K*K*C_in*C_out*4.
#include <cuda.h>

#include "epilogue16.cuh"

namespace d3b {

constexpr int kBvTileY = 16, kBvTileX = 16;     // output pixels per tile
constexpr int kBvHalfX = 8;                     // one half = 16 rows x 8 columns = two wgmma M = 64 blocks
constexpr int kBvKc = 64;                       // channels per stage (128 bytes of f16)
constexpr int kBvMathWarps = 8;                 // warps 0..7: consumer warpgroup `half`
constexpr int kBvTmaWarp = kBvMathWarps;        // first warp of the producer warpgroup (warps 8..11)
constexpr int kBvThreads = 32 * (kBvMathWarps + 4);   // 384 (registers are allocated per warpgroup: 168 each)
constexpr int kBvAStages = 2;

// PLANES = 2: FP16x3 (hi and lo planes); 1: single-pass FP16 (hi only).  Every expect-tx byte count below is the sum
// of the copies it covers: an A stage is 2 halves x PLANES boxes of kPatchBytes (the box make_map encodes: 64 channels x
// kBvHalfX pixels x kPatchRows rows of f16), a B stage the first PLANES parts of one slot of the packed weight image.
template <int KS, int STRIDE, int COUT, int PLANES = 2>
struct BvCfg {
  static constexpr int kPatchRows = STRIDE == 1 ? kBvTileY + KS - 1 : kBvTileY;      // rows in one staged patch
  static constexpr int kPatchBytes = kPatchRows * kBvHalfX * 128;
  static constexpr int kAStageBytes = 2 * PLANES * kPatchBytes;                       // {half 0, half 1} x {hi, lo}
  static constexpr int kSlotHalves = 2 * COUT * kBvKc;                                // packed slot: [W_hi | W_lo]
  static constexpr int kBBytes = PLANES * COUT * 128;                                 // [B_hi rows | B_lo rows]
  static constexpr int kBStages = COUT >= 128 ? 2 : 4;
  static constexpr int kSmemBytes = kBvAStages * kAStageBytes + kBStages * kBBytes + 1024 + 256;
  // with stride 1 one A stage serves the KS kernel rows of a (kx, kb); with stride > 1 every (ky, kx) has its own
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
};

// The kernel body for PLANES operand planes; bev_conv16_kernel (FP16x3) and bev_conv16_f16_kernel (single pass) below.
template <int KS, int STRIDE, int COUT, int PLANES>
__device__ __forceinline__ void bev_conv16_body(const CUtensorMap* tm_hi, const CUtensorMap* tm_lo, const BvGeom& g,
                                                const __half* __restrict__ packed, const Epi16& epi,
                                                __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                                                float* __restrict__ out_f32, int* __restrict__ overflow) {
  using Cfg = BvCfg<KS, STRIDE, COUT, PLANES>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + kBvAStages * Cfg::kAStageBytes;
  const uint32_t bar_base = b_base + Cfg::kBStages * Cfg::kBBytes;
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (kBvAStages + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (2 * kBvAStages + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (2 * kBvAStages + Cfg::kBStages + s); };

  D3B_CTA_MARK(0, epi.seq);
  pdl_launch_dependents();           // the next kernel of the stream may start its prologue behind this one's tail
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_group = g.batch * g.tiles_y * g.tiles_x;
  const int n_tiles = tiles_per_group * g.groups;
  const int k_vol = KS * KS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kBvAStages; ++s) { mbar_init(a_full(s), 1); mbar_init(a_empty(s), kBvMathWarps); }
    for (int s = 0; s < Cfg::kBStages; ++s) { mbar_init(b_full(s), 1); mbar_init(b_empty(s), kBvMathWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(tm_hi);
    if constexpr (PLANES == 2) tma_prefetch_desc(tm_lo);
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
        const __half* wgrp = packed + (size_t)grp * k_vol * g.n_kb * Cfg::kSlotHalves;
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
                tma_load_4d(dst + (PLANES * half) * Cfg::kPatchBytes, tm_hi, kb * kBvKc, cx, cy, b, a_full(sa));
                if constexpr (PLANES == 2)
                  tma_load_4d(dst + (2 * half + 1) * Cfg::kPatchBytes, tm_lo, kb * kBvKc, cx, cy, b, a_full(sa));
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
                             wgrp + ((size_t)(ky * KS + kx) * g.n_kb + kb) * Cfg::kSlotHalves, Cfg::kBBytes, b_full(sb));
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
              const uint32_t ah = a_base + sa * Cfg::kAStageBytes + (PLANES * half) * Cfg::kPatchBytes + row_adv;
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
                    if constexpr (PLANES == 2) {
                      // small terms first, the dominant hi.hi product last
                      wgmma_f16<Cfg::kPassN>(part, gmma_desc_sw128(a_lo + adv), gmma_desc_sw128(b_hi + nb + adv), ks > 0 ? 1u : 0u);
                      wgmma_f16<Cfg::kPassN>(part, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_lo + nb + adv), 1u);
                      wgmma_f16<Cfg::kPassN>(part, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_hi + nb + adv), 1u);
                    } else {
                      wgmma_f16<Cfg::kPassN>(part, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_hi + nb + adv), ks > 0 ? 1u : 0u);
                    }
                  }
                  gmma_commit();
                  gmma_wait();
                  gmma_fence_regs(part);
#pragma unroll
                  for (int q = 0; q < Cfg::kPassN / 2; ++q)
                    acc[m][np * Cfg::kPassN / 2 + q] += part[q];
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
            v0 = fmaf(v0, epi.corr, v0);
            v1 = fmaf(v1, epi.corr, v1);
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
            if (out_hi) ovf |= store_pair16<PLANES>(v0, v1, out_hi, out_lo, row_off + col);
            if (out_f32) *reinterpret_cast<float2*>(out_f32 + row_off + col) = make_float2(v0, v1);
          }
        }
      }
    }
    if (ovf && overflow) atomicOr(overflow, 1);
  }
  D3B_CTA_MARK(1, epi.seq);
}

template <int KS, int STRIDE, int COUT>
__global__ void __launch_bounds__(kBvThreads, 1)
bev_conv16_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, BvGeom g,
                  const __half* __restrict__ packed, Epi16 epi, __half* __restrict__ out_hi,
                  __half* __restrict__ out_lo, float* __restrict__ out_f32, int* __restrict__ overflow) {
  bev_conv16_body<KS, STRIDE, COUT, 2>(&tm_hi, &tm_lo, g, packed, epi, out_hi, out_lo, out_f32, overflow);
}

// Single-pass FP16: one A box per half and W_hi only per stage, one wgmma(A_hi, W_hi) per k-step (tm_lo, out_lo unused).
template <int KS, int STRIDE, int COUT>
__global__ void __launch_bounds__(kBvThreads, 1)
bev_conv16_f16_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, BvGeom g,
                      const __half* __restrict__ packed, Epi16 epi, __half* __restrict__ out_hi,
                      __half* __restrict__ out_lo, float* __restrict__ out_f32, int* __restrict__ overflow) {
  bev_conv16_body<KS, STRIDE, COUT, 1>(&tm_hi, &tm_lo, g, packed, epi, out_hi, out_lo, out_f32, overflow);
}

// ======================================================================================================================
// Variant "pipelined" (3x3, stride 1, output blocks of 128 channels, C_in % 64 == 0, up = 1; the automatic choice):
// tile = 16 rows x 8 columns x 128 channels (one half of the pixel-stationary tile).  Each consumer warpgroup owns one
// wgmma M = 64 block (8 x 8 pixels) x N = 128, i.e. 64 fp32 sums per thread, and computes a slot's 12-MMA partial as
// one m64n128k16 chain into one of two 64-register partials: slot s is issued into P[s & 1] while slot s - 1 is still
// running, then `wait_group 1` and s - 1 is folded.  Sums + two partials fit the 232 registers the consumer warpgroups
// take with setmaxnreg (the producer warpgroup keeps 40), so nothing spills and the tensor pipe always has the next slot
// queued.  Within one layer no tile size the register budget allows fills the grid (SECOND's 200 x 176 plane is 286
// tiles: 3 rounds of the 132 SMs, the last with 22 CTAs); chaining the layers of a block (below) does.  Same products, same order, same fold, same correction and epilogue as
// the pixel-stationary kernel: bit-identical to it.
//  * A stage = one box per plane, 64 channels x 8 pixels x 18 rows (18 KB); block m reads kernel row ky at
//    m * 8192 + ky * 1024.  B stage = [W_hi | W_lo] of one (kb, kx, ky).  Three stages of each.
//  * Single-pass FP16 (PLANES = 1): the hi box and W_hi alone per stage, one MMA per k-step (4 per slot).
constexpr int kPlCout = 128;
constexpr int kPlStages = 3;
constexpr int kPlPatchBytes = (kBvTileY + 2) * kBvHalfX * 128;    // 18432
constexpr int kPlSlotHalves = 2 * kPlCout * kBvKc;                // packed slot: [W_hi | W_lo]
template <int PLANES>
struct PlCfg {
  static constexpr int kAStageBytes = PLANES * kPlPatchBytes;     // hi, lo: PLANES boxes of kPlPatchBytes
  static constexpr int kBBytes = PLANES * kPlCout * 128;          // [W_hi rows | W_lo rows]
  static constexpr int kSmemBytes = kPlStages * (kAStageBytes + kBBytes) + 1024 + 256;
};
constexpr int kPlConsumerRegs = 232, kPlProducerRegs = 40;        // 2 * 232 + 40 <= 512 per thread triple
static_assert(2 * kPlConsumerRegs + kPlProducerRegs <= 512, "register budget of one SM");

// Chains of 3x3 stride-1 layers (d3b_bev_conv16_chain): one persistent launch runs up to kPlMaxLayers layers of one
// grid, handing out the tiles of every layer in order.  A tile of layer l + 1 reads only the 3 x 3 neighbourhood of
// tiles layer l wrote, so it can start while layer l is still finishing elsewhere: SECOND's six 286-tile layers run as
// 1716 tiles = 13 rounds of the 132 SMs instead of 6 x 3, and there are no launch boundaries in between.
//  * Work list: ticket t -> (layer, sample, tile, output group), layer-major, the output groups of a tile next to each
//    other.  One global counter hands the tickets out; the producer's elected lane fetches one per tile and passes it
//    to the consumer warpgroups through a two-entry shared ring.  Without a workspace (d3b_bev_conv16, one layer) the
//    producer walks t = blockIdx.x, += gridDim.x instead.
//  * Dependencies: done[l][sample][tile] counts the output groups of a layer-l tile whose planes are written (the 256
//    consumer threads fence their stores to the async proxy, meet at a named barrier, and one thread adds with release
//    semantics).  Before the first A load of a layer-l tile (l >= 1) the producer polls, with acquire semantics, the
//    <= 9 neighbouring tiles of layer l - 1 until each counts all of that layer's groups, then fences to the async
//    proxy: the planes were written through the generic proxy and TMA reads them through the async one.
//  * No deadlock: a ticket only waits on smaller tickets, and every smaller ticket was claimed by a CTA that is already
//    running and has issued (or is issuing) all of that ticket's loads before it fetches another -- so the smallest
//    unfinished ticket can always progress, whether or not all CTAs are co-resident.
//  * Buffer reuse: the stacks ping-pong two buffers, so layer l + 1 overwrites what layer l - 1 wrote and layer l read.
//    Layer-l tiles that read the region of tile i are exactly the neighbours of i that the layer-(l + 1) tile i waits
//    on, and a tile counts as done only after its consumers have used every staged patch: the read-after-write wait
//    also covers the write-after-read hazard (transitively for any older layer).  The host requires layer k's input to
//    be layer k - 1's output and no layer to write its own input.
//  * Replay: the last CTA to leave (a second counter) sets the ticket counter and the done counters back to zero, so
//    a replayed graph needs no host action and no extra node.
constexpr int kPlMaxLayers = 8;
struct PlLayer {
  CUtensorMap tm_hi, tm_lo;
  BvGeom g;                       // tiles_x counts 8-column tiles
  const __half* packed;
  Epi16 epi;
  __half* out_hi;
  __half* out_lo;
  float* out_f32;
};
struct PlChain {
  PlLayer layer[kPlMaxLayers];
  int n_layers;
  int first_ticket[kPlMaxLayers + 1];   // layer l's tickets are [first_ticket[l], first_ticket[l + 1])
  int spatial;                          // tiles of one layer and output group: batch * tiles_y * tiles_x
  int seq;                              // launch counter (development traces only)
  int* overflow;
  unsigned int* work;                   // null: static walk; else [0] tickets, [1] CTAs done, [2 + l * spatial + s] done
};
static_assert(sizeof(PlChain) <= 4096, "chain parameters must fit the classic 4 KB kernel-parameter space");

__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// Waits until done[i] == want (bounded: a protocol bug traps instead of hanging the GPU; the development library
// records code 6 in the fault word and returns).
__device__ __forceinline__ void wait_done(const unsigned int* done, unsigned int want) {
  for (uint32_t spin = 0; ld_acquire_gpu(done) != want; ++spin) {
#ifdef D3B_SOFT_TIMEOUT
    if (spin > (1u << 20)) {
      const unsigned int slot = atomicAdd(&g_d3b_fault[0], 1u);
      if (slot < 7u) g_d3b_fault[1 + slot] = (6u << 16) | (blockIdx.x & 0xffffu);
      return;
    }
#else
    if (spin > (1u << 26)) __trap();
#endif
  }
}

template <int PLANES>
__device__ __forceinline__ void bev_conv16_pl_body(const PlChain& P) {
  constexpr int kPlAStageBytes = PlCfg<PLANES>::kAStageBytes, kPlBBytes = PlCfg<PLANES>::kBBytes;
  extern __shared__ uint8_t smem_raw[];
  __shared__ int tk_ring[2];
  __shared__ int last_cta;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + kPlStages * kPlAStageBytes;
  const uint32_t bar_base = b_base + kPlStages * kPlBBytes;
  auto a_full = [&](uint32_t s) { return bar_base + 8u * s; };
  auto a_empty = [&](uint32_t s) { return bar_base + 8u * (kPlStages + s); };
  auto b_full = [&](uint32_t s) { return bar_base + 8u * (2 * kPlStages + s); };
  auto b_empty = [&](uint32_t s) { return bar_base + 8u * (3 * kPlStages + s); };
  auto tk_full = [&](uint32_t s) { return bar_base + 8u * (4 * kPlStages + s); };
  auto tk_empty = [&](uint32_t s) { return bar_base + 8u * (4 * kPlStages + 2 + s); };

  D3B_CTA_MARK(0, P.seq);
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tickets = P.first_ticket[P.n_layers];

  if (threadIdx.x == 0) {
    for (int s = 0; s < kPlStages; ++s) {
      mbar_init(a_full(s), 1); mbar_init(a_empty(s), kBvMathWarps);
      mbar_init(b_full(s), 1); mbar_init(b_empty(s), kBvMathWarps);
    }
    for (int s = 0; s < 2; ++s) { mbar_init(tk_full(s), 1); mbar_init(tk_empty(s), kBvMathWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (int l = 0; l < P.n_layers; ++l) {
      tma_prefetch_desc(&P.layer[l].tm_hi);
      if constexpr (PLANES == 2) tma_prefetch_desc(&P.layer[l].tm_lo);
    }
  }
  __syncthreads();
  pdl_wait_prior_grid();             // everything below reads the previous layer's planes or writes buffers it may still read

  // ticket -> (layer, output group, sample, y0, x0, tile index within the layer's grid)
  auto decode = [&](int t, int& l, int& grp, int& b, int& y0, int& x0, int& sp) {
    l = 0;
    while (l + 1 < P.n_layers && t >= P.first_ticket[l + 1]) ++l;
    const BvGeom& g = P.layer[l].g;
    const int u = t - P.first_ticket[l];
    grp = u % g.groups;
    sp = u / g.groups;
    const int per_sample = g.tiles_y * g.tiles_x;
    b = sp / per_sample;
    const int r = sp - b * per_sample;
    y0 = (r / g.tiles_x) * kBvTileY;
    x0 = (r % g.tiles_x) * kBvHalfX;
  };

  if (warp >= kBvTmaWarp) {
    // ===================== TMA producer (one elected lane) =====================
    regs_dealloc<kPlProducerRegs>();
    if (warp == kBvTmaWarp && lane == 0) {
      uint32_t a_it = 0, b_it = 0;
      int t = blockIdx.x;
      for (uint32_t it = 0;; ++it) {
        const uint32_t s = it & 1u;
        D3B_WAIT(tk_empty(s), ((it >> 1) & 1u) ^ 1u, 7);
        if (P.work) t = (int)atomicAdd(P.work, 1u);
        tk_ring[s] = t;
        mbar_arrive(tk_full(s));
        if (t >= n_tickets) break;
        int l, grp, b, y0, x0, sp;
        decode(t, l, grp, b, y0, x0, sp);
        const PlLayer& L = P.layer[l];
        if (P.work && l > 0) {
          const BvGeom& gp = P.layer[l - 1].g;
          const unsigned int* done = P.work + 2 + (size_t)(l - 1) * P.spatial + b * gp.tiles_y * gp.tiles_x;
          const int ty = y0 / kBvTileY, tx = x0 / kBvHalfX;
          for (int y = max(ty - 1, 0); y <= min(ty + 1, gp.tiles_y - 1); ++y)
            for (int x = max(tx - 1, 0); x <= min(tx + 1, gp.tiles_x - 1); ++x)
              wait_done(done + y * gp.tiles_x + x, (unsigned int)gp.groups);
          fence_proxy_async_global();
        }
        const __half* wgrp = L.packed + (size_t)grp * 9 * L.g.n_kb * kPlSlotHalves;
        for (int kb = 0; kb < L.g.n_kb; ++kb) {
          for (int kx = 0; kx < 3; ++kx, ++a_it) {
            const uint32_t sa = a_it % kPlStages;
            D3B_WAIT(a_empty(sa), ((a_it / kPlStages) & 1u) ^ 1u, 1);
            mbar_arrive_expect_tx(a_full(sa), kPlAStageBytes);
            const uint32_t dst = a_base + sa * kPlAStageBytes;
            tma_load_4d(dst, &L.tm_hi, kb * kBvKc, x0 + kx - L.g.pad, y0 - L.g.pad, b, a_full(sa));
            if constexpr (PLANES == 2)
              tma_load_4d(dst + kPlPatchBytes, &L.tm_lo, kb * kBvKc, x0 + kx - L.g.pad, y0 - L.g.pad, b, a_full(sa));
            for (int ky = 0; ky < 3; ++ky, ++b_it) {
              const uint32_t sb = b_it % kPlStages;
              D3B_WAIT(b_empty(sb), ((b_it / kPlStages) & 1u) ^ 1u, 2);
              mbar_arrive_expect_tx(b_full(sb), kPlBBytes);
              tma_bulk_g2s(b_base + sb * kPlBBytes, wgrp + ((size_t)(ky * 3 + kx) * L.g.n_kb + kb) * kPlSlotHalves,
                           kPlBBytes, b_full(sb));
            }
          }
        }
        if (!P.work) t += gridDim.x;
      }
    }
  } else {
    // ===================== consumer warpgroups: warpgroup m -> tile rows [8m, 8m + 8) =====================
    regs_alloc<kPlConsumerRegs>();
    const int m = warp >> 2, wq = warp & 3;
    bool ovf = false;
    uint32_t a_it = 0, b_it = 0;                 // ring positions of the tile's first A / B stage
    uint32_t it = 0;                             // tickets taken from the ring
    auto next_ticket = [&]() {
      const uint32_t ts = it & 1u;
      D3B_WAIT(tk_full(ts), (it >> 1) & 1u, 8);
      const int t = tk_ring[ts];
      __syncwarp();
      if (lane == 0) mbar_arrive(tk_empty(ts));
      ++it;
      return t;
    };
    for (int t = next_ticket(); t < n_tickets;) {
      int l, grp, b, y0, x0, sp;
      decode(t, l, grp, b, y0, x0, sp);
      const PlLayer& L = P.layer[l];
      const int n_slots = 9 * L.g.n_kb;                                // (kb, kx, ky), ky fastest
      float acc[kPlCout / 2], p0[kPlCout / 2], p1[kPlCout / 2];
#pragma unroll
      for (int q = 0; q < kPlCout / 2; ++q) acc[q] = 0.f;
      // slot s = (kb, kx, ky): its 12 MMAs into the partial P, committed as one group
      auto issue = [&](float (&Pp)[kPlCout / 2], int s) {
        const int ky = s % 3;
        const uint32_t ai = a_it + s / 3, bi = b_it + s;
        const uint32_t sa = ai % kPlStages, sb = bi % kPlStages;
        if (ky == 0) D3B_WAIT(a_full(sa), (ai / kPlStages) & 1u, 4);
        D3B_WAIT(b_full(sb), (bi / kPlStages) & 1u, 5);
        const uint32_t a_hi = a_base + sa * kPlAStageBytes + m * 8192u + (uint32_t)ky * 1024u, a_lo = a_hi + kPlPatchBytes;
        const uint32_t b_hi = b_base + sb * kPlBBytes, b_lo = b_hi + kPlCout * 128;
        gmma_fence();
#pragma unroll
        for (int ks = 0; ks < kBvKc / 16; ++ks) {
          const uint32_t adv = ks * 32;
          if constexpr (PLANES == 2) {
            // small terms first, the dominant hi.hi product last (the order of the pixel-stationary kernel)
            wgmma_f16<kPlCout>(Pp, gmma_desc_sw128(a_lo + adv), gmma_desc_sw128(b_hi + adv), ks > 0 ? 1u : 0u);
            wgmma_f16<kPlCout>(Pp, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_lo + adv), 1u);
            wgmma_f16<kPlCout>(Pp, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_hi + adv), 1u);
          } else {
            wgmma_f16<kPlCout>(Pp, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_hi + adv), ks > 0 ? 1u : 0u);
          }
        }
        gmma_commit();
      };
      // slot s has completed: fold its partial (round-to-nearest) and release its stages
      auto retire = [&](float (&Pp)[kPlCout / 2], int s) {
        gmma_fence_regs(Pp);
#pragma unroll
        for (int q = 0; q < kPlCout / 2; ++q) acc[q] += Pp[q];
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(b_empty((b_it + s) % kPlStages));
          if (s % 3 == 2) mbar_arrive(a_empty((a_it + s / 3) % kPlStages));
        }
      };
      for (int s = 0; s < n_slots; s += 2) {
        issue(p0, s);
        if (s > 0) {
          gmma_wait_pending<1>();
          retire(p1, s - 1);
        }
        if (s + 1 < n_slots) {
          issue(p1, s + 1);
          gmma_wait_pending<1>();
          retire(p0, s);
        }
      }
      gmma_wait();
      if (n_slots & 1) retire(p0, n_slots - 1);
      else retire(p1, n_slots - 1);
      a_it += n_slots / 3;
      b_it += n_slots;

      // epilogue, column block outer: each column pair's parameters are loaded once and used for both rows of the
      // thread (row outer keeps all 16 blocks' parameters live next to the sums and spills)
      const BvGeom& g = L.g;
      const Epi16& epi = L.epi;
      __half* out_hi = L.out_hi;
      __half* out_lo = L.out_lo;
      float* out_f32 = L.out_f32;
      const int cg = grp % g.cgroups;
      const int pcol = grp * kPlCout;           // per-group epilogue parameters are laid out group-major
      const int x = x0 + (lane >> 2);
      bool live[2];
      size_t row_off[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int y = y0 + 8 * m + 2 * wq + h;
        live[h] = y < g.h_out && x < g.w_out;
        row_off[h] = (((size_t)b * g.out_h + y) * g.out_w + x) * (size_t)g.out_channels + g.out_c0 + cg * kPlCout;
      }
#pragma unroll
      for (int jn = 0; jn < kPlCout / 8; ++jn) {
        const int col = jn * 8 + 2 * (lane & 3);
        float2 bb, sc, sh;
        if (epi.bias) bb = __ldg(reinterpret_cast<const float2*>(epi.bias + pcol + col));
        if (epi.scale) {
          sc = __ldg(reinterpret_cast<const float2*>(epi.scale + pcol + col));
          sh = __ldg(reinterpret_cast<const float2*>(epi.shift + pcol + col));
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!live[h]) continue;
          float v0 = acc[4 * jn + 2 * h] * epi.acc_scale, v1 = acc[4 * jn + 2 * h + 1] * epi.acc_scale;
          v0 = fmaf(v0, epi.corr, v0);
          v1 = fmaf(v1, epi.corr, v1);
          if (epi.bias) { v0 += bb.x; v1 += bb.y; }
          if (epi.scale) { v0 = fmaf(v0, sc.x, sh.x); v1 = fmaf(v1, sc.y, sh.y); }
          if (epi.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          if (out_hi && PLANES == 2) {
            uint32_t hi, lo;
            ovf |= split_pack2(v0, v1, hi, lo);
            *reinterpret_cast<uint32_t*>(out_hi + row_off[h] + col) = hi;
            *reinterpret_cast<uint32_t*>(out_lo + row_off[h] + col) = lo;
          }
          if (out_hi && PLANES == 1) ovf |= store_pair16<1>(v0, v1, out_hi, out_lo, row_off[h] + col);
          if (out_f32) *reinterpret_cast<float2*>(out_f32 + row_off[h] + col) = make_float2(v0, v1);
        }
      }
      // publish the tile to the next layer of the chain
      if (P.work && l + 1 < P.n_layers) {
        fence_proxy_async_global();
        asm volatile("bar.sync 1, %0;" ::"n"(32 * kBvMathWarps) : "memory");
        if (threadIdx.x == 0) {
          __threadfence();
          red_release_gpu_add(P.work + 2 + (size_t)l * P.spatial + sp, 1u);
        }
      }
      t = next_ticket();
      // one flag write per thread, once it knows it has no further tile (placed after the tile loop, it costs 40
      // registers: ptxas then spills the sums)
      if (t >= n_tickets && ovf && P.overflow) atomicOr(P.overflow, 1);
    }
  }
  if (P.work) {
    // the last CTA out resets the counters for the next launch (or graph replay)
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      unsigned int prev;
      asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(P.work + 1) : "memory");
      last_cta = prev == gridDim.x - 1;
    }
    __syncthreads();
    if (last_cta) {
      const int n_words = 2 + (P.n_layers - 1) * P.spatial;
      for (int i = threadIdx.x; i < n_words; i += blockDim.x) P.work[i] = 0u;
    }
  }
  D3B_CTA_MARK(1, P.seq);
}

__global__ void __launch_bounds__(kBvThreads, 1) bev_conv16_pl_kernel(const __grid_constant__ PlChain P) {
  bev_conv16_pl_body<2>(P);
}

// Single-pass FP16 (tm_lo, out_lo unused).
__global__ void __launch_bounds__(kBvThreads, 1) bev_conv16_pl_f16_kernel(const __grid_constant__ PlChain P) {
  bev_conv16_pl_body<1>(P);
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

// What both kernels are launched with: the tensor maps of the input planes (boxes of box_w pixels x box_h rows) and the
// epilogue parameters.  Single pass (planes = 1): no lo plane; tm_lo repeats tm_hi and is never read.
static int bev_args(const d3b_bev16_params* p, int planes, int box_w, int box_h, int stride, CUtensorMap* tm_hi,
                    CUtensorMap* tm_lo, Epi16* e) {
  int st = make_map(tm_hi, p->in_hi, p->batch, p->h_in, p->w_in, p->c_in, box_w, box_h, stride);
  if (st == D3B_OK) {
    if (planes == 2) st = make_map(tm_lo, p->in_lo, p->batch, p->h_in, p->w_in, p->c_in, box_w, box_h, stride);
    else *tm_lo = *tm_hi;
  }
  if (st != D3B_OK) return st;
  e->bias = p->bias; e->scale = p->scale; e->shift = p->shift;
  e->res_hi = nullptr; e->res_lo = nullptr;
  e->acc_scale = p->acc_scale; e->relu = p->relu;
  e->corr = trunc_correction(p->c_in, planes == 2 ? 3 : 1);
  static std::atomic<int> launch_seq{0};
  e->seq = launch_seq.fetch_add(1, std::memory_order_relaxed);
  return D3B_OK;
}

// persistent grid: one CTA per tile, at most one per SM
static int bev_grid(const BvGeom& g) {
  const int n_tiles = g.batch * g.tiles_y * g.tiles_x * g.groups;
  return n_tiles < kNumSMs ? n_tiles : kNumSMs;
}

template <int KS, int STRIDE, int COUT, int PLANES>
static int launch_bev(const d3b_bev16_params* p, const BvGeom& g, cudaStream_t stream) {
  using Cfg = BvCfg<KS, STRIDE, COUT, PLANES>;
  constexpr auto kernel = PLANES == 2 ? bev_conv16_kernel<KS, STRIDE, COUT> : bev_conv16_f16_kernel<KS, STRIDE, COUT>;
  static SmemOptIn optin;
  D3B_CUDA(ensure_dynamic_smem(kernel, Cfg::kSmemBytes, optin));
  CUtensorMap tm_hi, tm_lo;
  Epi16 e;
  const int st = bev_args(p, PLANES, kBvHalfX, Cfg::kPatchRows, STRIDE, &tm_hi, &tm_lo, &e);
  if (st != D3B_OK) return st;
  D3B_CUDA(launch_maybe_pdl(kernel, dim3(bev_grid(g)), dim3(kBvThreads), Cfg::kSmemBytes,
                            stream, tm_hi, tm_lo, g, (const __half*)p->weight_packed, e, (__half*)p->out_hi,
                            (__half*)p->out_lo, p->out_f32, (int*)p->overflow));
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

// pipelined kernel over layers[0, n) (3x3, stride 1, output blocks of 128 channels, C_in % 64 == 0, pad 1, no
// sub-pixel groups); work = null: one layer, static tile walk
template <int PLANES>
static int launch_bev_pl(const d3b_bev16_params* layers, const BvGeom* gs, int n, unsigned int* work,
                         cudaStream_t stream) {
  constexpr auto kernel = PLANES == 2 ? bev_conv16_pl_kernel : bev_conv16_pl_f16_kernel;
  static SmemOptIn optin;
  D3B_CUDA(ensure_dynamic_smem(kernel, PlCfg<PLANES>::kSmemBytes, optin));
  PlChain c = {};
  c.n_layers = n;
  for (int k = 0; k < n; ++k) {
    const d3b_bev16_params* p = layers + k;
    PlLayer& L = c.layer[k];
    const int st = bev_args(p, PLANES, kBvHalfX, kBvTileY + 2, 1, &L.tm_hi, &L.tm_lo, &L.epi);
    if (st != D3B_OK) return st;
    L.g = gs[k];
    L.g.tiles_x = div_up(L.g.w_out, kBvHalfX);     // tiles of 16 rows x 8 columns
    L.packed = (const __half*)p->weight_packed;
    L.out_hi = (__half*)p->out_hi;
    L.out_lo = (__half*)p->out_lo;
    L.out_f32 = p->out_f32;
    c.spatial = L.g.batch * L.g.tiles_y * L.g.tiles_x;
    c.first_ticket[k + 1] = c.first_ticket[k] + c.spatial * L.g.groups;
  }
  c.seq = c.layer[0].epi.seq;
  c.overflow = (int*)layers[0].overflow;
  c.work = work;
  const int n_tickets = c.first_ticket[n];
  D3B_CUDA(launch_maybe_pdl(kernel, dim3(n_tickets < kNumSMs ? n_tickets : kNumSMs), dim3(kBvThreads),
                            PlCfg<PLANES>::kSmemBytes, stream, c));
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

// The argument checks of d3b_bev_conv16 (before any CUDA call); fills the conv geometry and the plane count.
static int bev_check(const d3b_bev16_params* p, BvGeom* gp, bool* two_planes) {
  D3B_REQUIRE(p && p->in_hi && p->weight_packed, "d3b_bev_conv16: null argument");
  PlanePairs pp;
  pp.add(p->in_hi, p->in_lo);
  pp.add(p->out_hi, p->out_lo);
  D3B_REQUIRE(pp.consistent(),
              "d3b_bev_conv16: give in_lo and out_lo with their hi planes (FP16x3) or neither (single-pass FP16); got "
              "in_lo %s, out_lo %s", p->in_lo ? "set" : "NULL", p->out_lo ? "set" : "NULL");
  *two_planes = pp.planes() == 2;
  D3B_REQUIRE(p->batch >= 1 && p->h_in >= 1 && p->w_in >= 1 && p->c_in >= 16 && p->c_in % 16 == 0,
              "d3b_bev_conv16: bad input shape [%d,%d,%d,%d] (C_in must be a multiple of 16)", p->batch, p->h_in, p->w_in, p->c_in);
  // kernel = stride = s (2..4): the strided Conv2d deblock; it tiles the input exactly, so it takes no padding
  const bool k_is_s = p->ksize == p->stride && p->ksize >= 2 && p->ksize <= 4;
  D3B_REQUIRE(k_is_s || ((p->ksize == 1 || p->ksize == 3) && (p->stride == 1 || p->stride == 2) &&
                         !(p->ksize == 1 && p->stride != 1)),
              "d3b_bev_conv16: ksize %d stride %d not built (3x3 s1/s2, 1x1 s1, k = s in {2, 3, 4})", p->ksize, p->stride);
  D3B_REQUIRE(k_is_s ? p->pad == 0 : (p->pad >= 0 && p->pad <= p->ksize / 2 + 1),
              "d3b_bev_conv16: pad %d not built for ksize %d stride %d", p->pad, p->ksize, p->stride);
  D3B_REQUIRE(p->up >= 1 && p->up <= 4 && p->cgroups >= 1 && p->groups == p->cgroups * p->up * p->up,
              "d3b_bev_conv16: groups %d != cgroups %d * up^2 (up %d)", p->groups, p->cgroups, p->up);
  D3B_REQUIRE(p->out_hi || p->out_f32, "d3b_bev_conv16: give out_hi (+ out_lo) and/or out_f32");
  D3B_REQUIRE((p->scale == nullptr) == (p->shift == nullptr), "d3b_bev_conv16: scale and shift go together");
  D3B_REQUIRE(p->out_channels % 8 == 0 && p->out_c0 % 8 == 0 && p->out_c0 + p->cgroups * p->c_out <= p->out_channels,
              "d3b_bev_conv16: output channel slice [%d, %d) does not fit rows of %d", p->out_c0,
              p->out_c0 + p->cgroups * p->c_out, p->out_channels);
  // (an input smaller than the kernel has no output; C division would round -1/s up to 0 and make one)
  D3B_REQUIRE(p->h_in + 2 * p->pad >= p->ksize && p->w_in + 2 * p->pad >= p->ksize,
              "d3b_bev_conv16: input %dx%d (pad %d) is smaller than the kernel %d", p->h_in, p->w_in, p->pad, p->ksize);
  BvGeom& g = *gp;
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
  return D3B_OK;
}

// the layers the pipelined kernel takes: 3x3 stride 1, output blocks of 128 channels, C_in % 64 == 0, no sub-pixel groups
static bool pl_eligible(const d3b_bev16_params* p) {
  return p->ksize == 3 && p->stride == 1 && p->c_out == kPlCout && p->c_in % kBvKc == 0 && p->up == 1;
}

}  // namespace d3b

using namespace d3b;

extern "C" int d3b_bev_conv16(const d3b_bev16_params* p, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  BvGeom g;
  bool two;
  const int st = bev_check(p, &g, &two);
  if (st != D3B_OK) return st;
  // Automatic (variant 2) = the pipelined kernel for the 3x3 stride-1 layers with 128-channel output blocks, the
  // pixel-stationary kernel for every other shape.  Variant 0 (pixel-stationary everywhere) is the reference the
  // pipelined kernel reproduces bit for bit.
  if (bev_variant() == 2 && pl_eligible(p))
    return two ? launch_bev_pl<2>(p, &g, 1, nullptr, stream) : launch_bev_pl<1>(p, &g, 1, nullptr, stream);
#define D3B_BEV_CASE(KS, ST)                                                                                        \
  if (p->ksize == KS && p->stride == ST) {                                                                          \
    switch (p->c_out) {                                                                                             \
      case 32: return two ? launch_bev<KS, ST, 32, 2>(p, g, stream) : launch_bev<KS, ST, 32, 1>(p, g, stream);       \
      case 64: return two ? launch_bev<KS, ST, 64, 2>(p, g, stream) : launch_bev<KS, ST, 64, 1>(p, g, stream);       \
      case 128: return two ? launch_bev<KS, ST, 128, 2>(p, g, stream) : launch_bev<KS, ST, 128, 1>(p, g, stream);    \
      default: break;                                                                                               \
    }                                                                                                               \
  }
  D3B_BEV_CASE(3, 1)
  D3B_BEV_CASE(3, 2)
  D3B_BEV_CASE(1, 1)
  D3B_BEV_CASE(2, 2)
  D3B_BEV_CASE(3, 3)
  D3B_BEV_CASE(4, 4)
#undef D3B_BEV_CASE
  set_error("d3b_bev_conv16: C_out per group %d not in {32, 64, 128}", p->c_out);
  return D3B_ERR_UNSUPPORTED;
}

extern "C" int64_t d3b_bev_conv16_chain_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t n_layers) {
  if (batch < 1 || h < 1 || w < 1 || n_layers < 1 || n_layers > kPlMaxLayers) return 0;
  const int64_t tiles = (int64_t)batch * div_up(h, kBvTileY) * div_up(w, kBvHalfX);
  return 4 * (2 + (int64_t)(n_layers - 1) * tiles);     // ticket and exit counters, done counters of layers 0..n-2
}

extern "C" int d3b_bev_conv16_chain(const d3b_bev16_params* layers, int32_t n_layers, void* workspace,
                                    int64_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(layers && n_layers >= 1 && n_layers <= kPlMaxLayers, "d3b_bev_conv16_chain: n_layers %d outside 1..%d",
              n_layers, kPlMaxLayers);
  BvGeom gs[kPlMaxLayers];
  bool two = false;
  for (int k = 0; k < n_layers; ++k) {
    const d3b_bev16_params* p = layers + k;
    bool tk;
    if (bev_check(p, &gs[k], &tk) != D3B_OK) {
      char why[256];
      snprintf(why, sizeof(why), "%s", d3b_last_error());
      set_error("d3b_bev_conv16_chain: layer %d: %s", k, why);
      return D3B_ERR_INVALID_ARG;
    }
    D3B_REQUIRE(pl_eligible(p) && p->pad == 1 && p->out_hi && p->out_c0 == 0 && p->out_channels == p->cgroups * p->c_out,
                "d3b_bev_conv16_chain: layer %d is not a 3x3 stride-1 pad-1 layer of 128-channel output blocks with "
                "C_in %% 64 == 0 writing whole output planes", k);
    D3B_REQUIRE(p->in_hi != p->out_hi && (p->in_lo == nullptr || p->in_lo != p->out_lo),
                "d3b_bev_conv16_chain: layer %d's input aliases its own output", k);
    if (k == 0) {
      two = tk;
      continue;
    }
    const d3b_bev16_params* q = layers + k - 1;
    D3B_REQUIRE(tk == two && p->batch == q->batch && p->h_in == q->h_in && p->w_in == q->w_in &&
                    p->c_in == q->out_channels && p->in_hi == q->out_hi && p->in_lo == q->out_lo,
                "d3b_bev_conv16_chain: layer %d's input is not layer %d's output planes", k, k - 1);
    D3B_REQUIRE(p->overflow == layers[0].overflow, "d3b_bev_conv16_chain: layer %d has another overflow flag than layer 0",
                k);
  }
  const int64_t need = d3b_bev_conv16_chain_workspace_bytes(layers[0].batch, layers[0].h_in, layers[0].w_in, n_layers);
  D3B_REQUIRE(workspace && workspace_bytes >= need, "d3b_bev_conv16_chain: workspace of %lld bytes, %lld needed",
              (long long)workspace_bytes, (long long)need);
  if (bev_variant() != 2) {             // the reference schedule: layer by layer through d3b_bev_conv16
    for (int k = 0; k < n_layers; ++k) {
      const int st = d3b_bev_conv16(layers + k, stream_);
      if (st != D3B_OK) return st;
    }
    return D3B_OK;
  }
  unsigned int* work = (unsigned int*)workspace;
  return two ? launch_bev_pl<2>(layers, gs, n_layers, work, stream) : launch_bev_pl<1>(layers, gs, n_layers, work, stream);
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
