// Output-stationary sparse convolution on the Hopper tensor cores with split-f16 operands ("FP16x3"), sm_90a.
//
//   out[o,:] = act((sum_k in[nbr[k][o],:] . W[k] + bias) * scale + shift + residual[o,:])
//
// Reference: spconv v1.x indice_conv (per offset: gather -> fp32 torch.mm -> scatter-add) followed by
// BatchNorm1d(eval) / ReLU / residual, call sites det3d/models/backbones/scn.py:73-89,106-157,323-355.
//
// Why this form.  A pair-based kernel (spconv's gather -> GEMM -> scatter-add) sums the offsets' partial products
// with fp32 atomics: summation order -- hence the last bits -- changes run to run, and it needs buffer-clearing launches
// and a deferred epilogue.  Here one CTA owns 128 output rows and walks the kernel offsets present in the tile
// (tile_mask); an (offset, 64-channel slice) is one pipeline slot: gather warps copy the 128 input rows (or zeros where
// the offset has no neighbour) with 16-byte cp.async straight into a K-major, 128B-swizzled tile, two consumer
// warpgroups (64 rows each) issue wgmma.m64nNk16 into fp32 register accumulators, and the fused bias/BN/residual/ReLU
// epilogue writes each output row once.  No atomics, fixed summation order: bit-identical results run to run, and a
// row's bits depend on its own neighbourhood only (not on the rows sharing its tile).
//
// fp32-equivalent accuracy on the f16 pipe (twice the tf32 rate, half the operand bytes).  Activations live in HBM as
// two f16 planes, hi = f16(x) and lo = f16(x - hi) (22 significant bits, written once by the producing layer's
// epilogue); weights are split the same way at load time after an exact power-of-two scaling that keeps their lo
// parts out of the f16 subnormal range.  D += A_lo.B_hi + A_hi.B_lo + A_hi.B_hi with fp32 accumulation; the dropped
// lo.lo term is 2^-22 relative.  |x| >= 65504 cannot be represented: the epilogue raises a device flag instead of
// silently saturating (the host checks it with the detections).
//
// Accumulation.  The tensor core adds every MMA's partial sum into the fp32 accumulator with truncation (round toward
// zero), a systematic shrink that grows with the number of MMAs chained into one accumulator; chaining a whole 3x3x3
// layer (up to 648 MMAs) into one accumulator puts the encoder output beyond 1e-4.  So the chain is bounded: the
// products of one slot (<= 12 MMAs) go into a fresh register partial, which is added into the running fp32 sums with
// round-to-nearest; the epilogue scales the sums by 1 + n * 2^-26 (the mean truncation of n MMAs, gmma.cuh) -- the summation structure of
// the reference's per-offset GEMM + scatter-add, in a fixed order.  An absent neighbour contributes an exact zero
// partial, so a row's bits depend on its own neighbourhood only.
//
// Roles: 8 consumer warps (two warpgroups, first so that they are warpgroup-aligned), one gather group of 2 warps per
// pipeline stage (slot j -> group j % stages; 4 stages, 3 at C_out = 128; pure cp.async issue); persistent grid <= one
// CTA per SM.  C_in = 16 / 32 layers pack 4 / 2 kernel offsets into one slot (os16_pack).  The tile's rulebook rows
// arrive by cp.async.bulk; the kernel is launched with programmatic stream serialisation (prologue overlaps the
// previous layer's tail).
// Algorithmic bytes per layer (SURVEY 8d): N_in*C_in*4 + N_out*C_out*4 + P*8 + K*C_in*C_out*4.
#include "epilogue16.cuh"

namespace d3b {

constexpr int kOsTileM = 128;
constexpr int kOsKc = 64;                                  // channels per stage = one 128-byte swizzle row of f16
constexpr int kOsABytes = kOsTileM * 128;                  // one A plane tile (hi or lo)

// PLANES = 2: FP16x3 (hi and lo of activations and weights); 1: single-pass FP16 (hi only).  A B stage holds the first
// PLANES parts of one slot of the packed weight image, whose slot stride is kSlotHalves in both modes.
template <int COUT, int PLANES = 2>
struct OsCfg {
  static constexpr int kSlotHalves = 2 * COUT * kOsKc;     // packed[slot][kb] = [W_hi rows | W_lo rows]
  static constexpr int kBBytes = PLANES * COUT * 128;      // [B_hi rows | B_lo rows], or B_hi rows
  static constexpr int kStageBytes = PLANES * kOsABytes + kBBytes;
  static constexpr int kStages = COUT >= 128 ? 3 : 4;
  // One gather group per pipeline stage: group g only ever fills stage g.  (A group waits for "stage free" on the
  // PARITY of the stage's empty barrier; that is unambiguous only if the group itself has seen the previous use of
  // the stage go by -- with more groups than stages a group would meet a stage it last touched two uses ago, read a
  // stale parity as "free" and overwrite live operands.)
  static constexpr int kGroups = kStages;
  static constexpr int kMathWarps = 8;                     // two consumer warpgroups, rows [0, 64) and [64, 128)
  static constexpr int kGatherWarp0 = kMathWarps;          // warps [8, 8 + 2 kGroups): gather groups of 2 warps
  static constexpr int kGroupThreads = 64;                 // (few threads: the register file goes to the accumulators)
  static constexpr int kThreads = 32 * (kGatherWarp0 + 2 * kGroups);   // 512 (C_out 16..64), 448 (128)
  // A slot's products are chained into a fresh register partial, one column pass of kPassN outputs at a time, and
  // added into the running sums with round-to-nearest (see the kernel comment); C_out = 128 runs two passes so that
  // partial + sums fit the register budget.
  static constexpr int kPassN = COUT >= 128 ? 64 : COUT;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/ + 32 * kOsTileM * 4;
};

// Fused epilogue on 16 consecutive output channels of one row (the FFMA first layer: its sums are not truncated, so no
// correction); returns true if a value left the f16 range.
template <int PLANES>
__device__ __forceinline__ bool epilogue16(float (&v)[16], const Epi16& e, size_t row_off, int col, __half* out_hi,
                                           __half* out_lo, float* out_f32) {
#pragma unroll
  for (int q = 0; q < 16; ++q) v[q] *= e.acc_scale;
  if (e.bias) {
#pragma unroll
    for (int q = 0; q < 16; q += 4) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(e.bias + col + q));
      v[q] += b.x; v[q + 1] += b.y; v[q + 2] += b.z; v[q + 3] += b.w;
    }
  }
  if (e.scale) {
#pragma unroll
    for (int q = 0; q < 16; q += 4) {
      const float4 s = __ldg(reinterpret_cast<const float4*>(e.scale + col + q));
      const float4 t = __ldg(reinterpret_cast<const float4*>(e.shift + col + q));
      v[q] = fmaf(v[q], s.x, t.x); v[q + 1] = fmaf(v[q + 1], s.y, t.y);
      v[q + 2] = fmaf(v[q + 2], s.z, t.z); v[q + 3] = fmaf(v[q + 3], s.w, t.w);
    }
  }
  if (e.res_hi) {
#pragma unroll
    for (int q = 0; q < 16; q += 8) {
      if constexpr (PLANES == 2) {
        const uint4 h = __ldg(reinterpret_cast<const uint4*>(e.res_hi + row_off + col + q));
        const uint4 l = __ldg(reinterpret_cast<const uint4*>(e.res_lo + row_off + col + q));
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&hw[j]));
          const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&lw[j]));
          v[q + 2 * j] += fh.x + fl.x;          // hi + lo is exact in fp32 (22 bits)
          v[q + 2 * j + 1] += fh.y + fl.y;
        }
      } else {
        const uint4 h = __ldg(reinterpret_cast<const uint4*>(e.res_hi + row_off + col + q));
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&hw[j]));
          v[q + 2 * j] += fh.x;
          v[q + 2 * j + 1] += fh.y;
        }
      }
    }
  }
  bool ovf = false;
  if (e.relu) {
#pragma unroll
    for (int q = 0; q < 16; ++q) v[q] = fmaxf(v[q], 0.f);
  }
  if (out_hi && PLANES == 2) {
    uint32_t hi[8], lo[8];
#pragma unroll
    for (int q = 0; q < 16; q += 2) ovf |= split_pack2(v[q], v[q + 1], hi[q >> 1], lo[q >> 1]);
    uint4* ph = reinterpret_cast<uint4*>(out_hi + row_off + col);
    uint4* pl = reinterpret_cast<uint4*>(out_lo + row_off + col);
    ph[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    ph[1] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
    pl[0] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    pl[1] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
  }
  if (out_hi && PLANES == 1) {
    uint32_t hi[8];
#pragma unroll
    for (int q = 0; q < 16; q += 2) {
      hi[q >> 1] = pack_half2(__float2half_rn(v[q]), __float2half_rn(v[q + 1]));
      ovf |= f16_out_of_range(v[q]) | f16_out_of_range(v[q + 1]);
    }
    uint4* ph = reinterpret_cast<uint4*>(out_hi + row_off + col);
    ph[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    ph[1] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
  }
  if (out_f32) {
    float4* pf = reinterpret_cast<float4*>(out_f32 + row_off + col);
#pragma unroll
    for (int q = 0; q < 16; q += 4) pf[q >> 2] = make_float4(v[q], v[q + 1], v[q + 2], v[q + 3]);
  }
  return ovf;
}

// The same epilogue on the two consecutive output channels a wgmma accumulator fragment holds, with the correction.
template <int PLANES>
__device__ __forceinline__ bool epilogue2(float v0, float v1, const Epi16& e, size_t row_off, int col, __half* out_hi,
                                          __half* out_lo, float* out_f32) {
  v0 *= e.acc_scale;
  v1 *= e.acc_scale;
  v0 = fmaf(v0, e.corr, v0);
  v1 = fmaf(v1, e.corr, v1);
  if (e.bias) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(e.bias + col));
    v0 += b.x; v1 += b.y;
  }
  if (e.scale) {
    const float2 s = __ldg(reinterpret_cast<const float2*>(e.scale + col));
    const float2 t = __ldg(reinterpret_cast<const float2*>(e.shift + col));
    v0 = fmaf(v0, s.x, t.x); v1 = fmaf(v1, s.y, t.y);
  }
  if (e.res_hi) {
    const float2 r = load_pair16<PLANES>(e.res_hi, e.res_lo, row_off + col);
    v0 += r.x;
    v1 += r.y;
  }
  if (e.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
  bool ovf = false;
  if (out_hi) ovf = store_pair16<PLANES>(v0, v1, out_hi, out_lo, row_off + col);
  if (out_f32) *reinterpret_cast<float2*>(out_f32 + row_off + col) = make_float2(v0, v1);
  return ovf;
}

// Offset packing.  A pipeline slot always moves 128 rows x 128 bytes per plane and costs about the same whatever part
// of it is live, so layers with C_in = 16 / 32 put `pack` = 4 / 2 kernel offsets side by side along K: slot p holds the
// rows of offsets p*pack .. p*pack + pack - 1 (16-byte chunks [sub * 8/pack, (sub+1) * 8/pack) of every row come from
// offset p*pack + sub), the weight slice is the matching K-concatenation (zero for offsets >= k_vol), and a 3x3x3 layer
// runs 14 / 7 slots per tile instead of 27.  A slot is skipped when none of its offsets occurs in the tile.
__host__ __device__ inline int os16_pack(int c_in, int k_vol) {
  return k_vol > 1 && (c_in == 16 || c_in == 32) ? kOsKc / c_in : 1;
}
__device__ __forceinline__ unsigned int os16_slot_mask(unsigned int offset_mask, int pack) {
  if (pack == 1) return offset_mask;
  unsigned int r = 0u;
  const unsigned int grp = (1u << pack) - 1u;
  for (int p = 0; p * pack < 32; ++p) r |= ((offset_mask >> (p * pack)) & grp) ? (1u << p) : 0u;
  return r;
}

// The kernel body for PLANES operand planes; spconv_os16_kernel (FP16x3) and spconv_os16_f16_kernel (single pass) below.
template <int COUT, int PLANES>
__device__ __forceinline__ void spconv_os16_body(
    const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, const int* __restrict__ nbr,
    const unsigned int* __restrict__ tile_mask, const int* __restrict__ n_out_p, int out_cap, int c_in, int n_kb, int pack,
    int k_vol, const __half* __restrict__ packed, const Epi16& epi, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
    float* __restrict__ out_f32, int* __restrict__ overflow) {
  using Cfg = OsCfg<COUT, PLANES>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + Cfg::kStages * Cfg::kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };
  const uint32_t nbr_bar = bar_base + 8u * (2 * Cfg::kStages);                    // neighbour rows of the tile have landed
  int* koff_s = reinterpret_cast<int*>(smem_gen + Cfg::kStages * Cfg::kStageBytes + 128);   // [32] active offsets
  int* nbr_s = reinterpret_cast<int*>(smem_gen + Cfg::kStages * Cfg::kStageBytes + 256);    // [32][128] neighbour rows

  D3B_CTA_MARK(0, epi.seq);
  pdl_launch_dependents();           // the next kernel of the stream may start its prologue behind this one's tail
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_out = min(*n_out_p, out_cap);
  const int n_tiles = (n_out + kOsTileM - 1) / kOsTileM;
  const int c_eff = c_in * pack;                 // K extent of the slots (64 when offsets are packed)

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(full_bar(s), Cfg::kGroupThreads + 1);   // the gather threads of one group + the expect_tx arrive
      mbar_init(empty_bar(s), Cfg::kMathWarps);         // every consumer warp, once its wgmmas have read the stage
    }
    mbar_init(nbr_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < Cfg::kMathWarps) {
    // ===================== consumer warpgroups =====================
    pdl_wait_prior_grid();           // (residual planes / output buffers belong to earlier kernels)
    // Per slot: wgmma of the warpgroup's 64 rows into fp32 registers.  At the end of the tile: truncation correction,
    // fused bias / BN / residual / ReLU, split into f16 planes.
    const int wg = warp >> 2, wq = warp & 3;
    bool ovf = false;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const unsigned int smask = os16_slot_mask(tile_mask[tile], pack);
      const int n_slots = __popc(smask) * n_kb;
      float acc[COUT / 2];                       // running fp32 sums (round-to-nearest adds of the slot partials)
#pragma unroll
      for (int q = 0; q < COUT / 2; ++q) acc[q] = 0.f;
      for (int j = 0; j < n_slots; ++j, ++it) {
        const int kb = n_kb == 1 ? 0 : j % n_kb;
        const int s = it % Cfg::kStages;
        const uint32_t ph = (it / Cfg::kStages) & 1u;
        const int n_ks = min(kOsKc / 16, (c_eff - kb * kOsKc + 15) / 16);
        if (warp == 0 && lane == 0) D3B_STAMP(6, it);
        D3B_WAIT(full_bar(s), ph, 3);
        const uint32_t a_hi = smem_base + s * Cfg::kStageBytes + wg * 8192u;   // rows 64 wg .. 64 wg + 63
        const uint32_t a_lo = a_hi + kOsABytes;                                  // (PLANES = 2 only)
        const uint32_t b_hi = smem_base + s * Cfg::kStageBytes + PLANES * kOsABytes;
        const uint32_t b_lo = b_hi + COUT * 128;
#pragma unroll
        for (int np = 0; np < COUT / Cfg::kPassN; ++np) {
          float part[Cfg::kPassN / 2];
          const uint32_t nb = np * Cfg::kPassN * 128;             // first B row of this column pass
          gmma_fence();
          // always the full 64-channel slot: the K tail of a slot (channels >= C_in) is zero in both operands, so its
          // MMAs add exact zeros -- and a uniform batch keeps the wgmmas from being serialised
#pragma unroll
          for (int ks = 0; ks < kOsKc / 16; ++ks) {
            const uint32_t adv = ks * 32;               // 16 f16 = 32 bytes along K
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
          for (int q = 0; q < Cfg::kPassN / 2; ++q) acc[np * Cfg::kPassN / 2 + q] += part[q];
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(s));     // the gather group may refill this stage
        if (warp == 0 && lane == 0) D3B_STAMP(7, it);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = tile * kOsTileM + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (o >= n_out) continue;
#pragma unroll
        for (int jn = 0; jn < COUT / 8; ++jn)
          ovf |= epilogue2<PLANES>(acc[4 * jn + 2 * h], acc[4 * jn + 2 * h + 1], epi, (size_t)o * COUT, jn * 8 + 2 * (lane & 3),
                           out_hi, out_lo, out_f32);
      }
    }
    if (ovf && overflow) atomicOr(overflow, 1);
  } else {
    // ===================== gather producers =====================
    const int gw = warp - Cfg::kGatherWarp0;
    const int group = gw >> 1, wq = gw & 1;                     // two warps per group, 64 rows each
    const int g = lane >> 3, c = lane & 7;
    const bool issues_tma = (wq == 0 && lane == 0);
    const int ptid = threadIdx.x - 32 * Cfg::kGatherWarp0;      // 0 .. 64 * kGroups - 1
    const int cpo = 8 / pack;                                   // 16-byte chunks per packed offset
    const int sub = c / cpo;                                    // which of the slot's offsets feeds this thread's chunk
    const int c_src = c - sub * cpo;                            // ... and which chunk of that offset's source row
    uint32_t it0 = 0;       // pipeline slots consumed by earlier tiles (same sequence in every role)
    uint32_t tile_count = 0;                       // tiles with work so far (phase of nbr_bar)
    const bool bulk_nbr = (out_cap & 3) == 0;      // 16-byte aligned rows: cp.async.bulk can fetch them
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int row0 = tile * kOsTileM;
      const unsigned int mask = os16_slot_mask(tile_mask[tile], pack);
      const int n_off = __popc(mask);                 // slots' worth of offsets (groups of `pack`) present in the tile
      const int n_slots = n_off * n_kb;

      // stage nbr[k][row0 .. row0+127] for the active offsets (one global round trip per tile)
      asm volatile("bar.sync 1, %0;" ::"r"(Cfg::kGroupThreads * Cfg::kGroups) : "memory");   // previous tile's readers are done
      if (ptid < 32) {                                    // n-th active offset of the tile
        unsigned int m = mask;
        for (int t = ptid; t > 0; --t) m &= m - 1;
        const int k = __ffs(m) - 1;
        if (ptid < n_off) koff_s[ptid] = k;
        __syncwarp();
        // neighbour rows of the tile by bulk copy (one 512-byte copy per offset of an active slot, no thread touches
        // them): entry e = (slot e / pack, member e % pack) -> nbr_s[e][0..127]
        const int rows = min(kOsTileM, out_cap - row0);
        const int e_slot = ptid / pack;
        const int k_src = ptid < n_off * pack ? koff_s[e_slot] * pack + (ptid - e_slot * pack) : k_vol;
        const bool valid = k_src < k_vol;             // (the last group of a 27-offset kernel has phantom members)
        const unsigned int vm = __ballot_sync(0xffffffffu, valid);
        if (bulk_nbr && vm != 0u && ptid == 0) mbar_arrive_expect_tx(nbr_bar, (uint32_t)(__popc(vm) * rows * 4));
        __syncwarp();
        if (bulk_nbr && valid)
          tma_bulk_g2s(smem_u32(nbr_s + ptid * kOsTileM), nbr + (size_t)k_src * out_cap + row0, (uint32_t)(rows * 4), nbr_bar);
      }
      if (bulk_nbr) {
        if (n_off > 0) D3B_WAIT(nbr_bar, tile_count & 1u, 5);
      } else {
        asm volatile("bar.sync 1, %0;" ::"r"(Cfg::kGroupThreads * Cfg::kGroups) : "memory");
#pragma unroll 8
        for (int idx = ptid; idx < n_off * pack * kOsTileM; idx += Cfg::kGroupThreads * Cfg::kGroups) {   // independent loads
          const int r = idx & 127, e = idx >> 7;
          const int k_src = koff_s[e / pack] * pack + e % pack;
          nbr_s[idx] = k_src < k_vol ? __ldg(nbr + (size_t)k_src * out_cap + min(row0 + r, out_cap - 1)) : -1;
        }
      }
      asm volatile("bar.sync 1, %0;" ::"r"(Cfg::kGroupThreads * Cfg::kGroups) : "memory");
      if (n_off > 0) ++tile_count;
      if (tile == (int)blockIdx.x) pdl_wait_prior_grid();     // rulebook rows staged; the activations need the previous layer done

      for (int j = (int)((group + Cfg::kGroups - (it0 % Cfg::kGroups)) % Cfg::kGroups); j < n_slots; j += Cfg::kGroups) {
        const int n = j / n_kb, kb = j - n * n_kb;
        const int ch = pack > 1 ? c_src * 8 : kb * kOsKc + c * 8;     // this thread's 8 channels (16 bytes) of the source row
        const uint32_t it = it0 + (uint32_t)j;
        const int s = it % Cfg::kStages;
        const uint32_t ph = (it / Cfg::kStages) & 1u;
        if (issues_tma) D3B_STAMP(0, it);
        D3B_WAIT(empty_bar(s), ph ^ 1u, 1);
        if (issues_tma) D3B_STAMP(1, it);
        const uint32_t stage = smem_base + s * Cfg::kStageBytes;
        if (issues_tma) {
          mbar_arrive_expect_tx(full_bar(s), Cfg::kBBytes);
          tma_bulk_g2s(stage + PLANES * kOsABytes, packed + ((size_t)koff_s[n] * n_kb + kb) * Cfg::kSlotHalves, Cfg::kBBytes,
                       full_bar(s));
        }
        {   // chunks past C_in are zero-filled (the consumers always multiply the full 64-channel slot)
          // this thread: 16 consecutive rows (indices fetched as four 16-byte shared-memory loads), one 16-byte chunk
          const int row_base = wq * 64 + g * 16;
          const int4* idx4 = reinterpret_cast<const int4*>(nbr_s + (n * pack + sub) * kOsTileM + row_base);
          const bool col_live = pack > 1 ? koff_s[n] * pack + sub < k_vol : ch < c_in;
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const int4 iv = idx4[q4];
            const int srcs[4] = {iv.x, iv.y, iv.z, iv.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int row = row_base + q4 * 4 + u;
              const bool live = srcs[u] >= 0 && col_live && row0 + row < n_out;    // (rows past n_out hold stale indices)
              const size_t off = live ? (size_t)srcs[u] * c_in + ch : 0;
              const uint32_t dst = stage + sw128_offset(row, c);
              cp_async16(dst, in_hi + off, live ? 16u : 0u);
              if constexpr (PLANES == 2) cp_async16(dst + kOsABytes, in_lo + off, live ? 16u : 0u);
            }
          }
        }
        if (issues_tma) D3B_STAMP(2, it);
        cp_async_wait_all();
        if (issues_tma) D3B_STAMP(3, it);
        fence_proxy_async();      // generic-proxy writes -> visible to the tensor core (async proxy)
        mbar_arrive(full_bar(s));
      }
      it0 += (uint32_t)n_slots;
    }
  }
  D3B_CTA_MARK(1, epi.seq);
}

template <int COUT>
__global__ void __launch_bounds__(OsCfg<COUT>::kThreads, 1)
spconv_os16_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, const int* __restrict__ nbr,
                   const unsigned int* __restrict__ tile_mask, const int* __restrict__ n_out_p, int out_cap, int c_in,
                   int n_kb, int pack, int k_vol, const __half* __restrict__ packed, Epi16 epi, __half* __restrict__ out_hi,
                   __half* __restrict__ out_lo, float* __restrict__ out_f32, int* __restrict__ overflow) {
  spconv_os16_body<COUT, 2>(in_hi, in_lo, nbr, tile_mask, n_out_p, out_cap, c_in, n_kb, pack, k_vol, packed, epi, out_hi,
                            out_lo, out_f32, overflow);
}

// Single-pass FP16: the same kernel on the hi planes alone, one wgmma(A_hi, W_hi) per k-step (in_lo / out_lo unused).
template <int COUT>
__global__ void __launch_bounds__(OsCfg<COUT, 1>::kThreads, 1)
spconv_os16_f16_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, const int* __restrict__ nbr,
                       const unsigned int* __restrict__ tile_mask, const int* __restrict__ n_out_p, int out_cap, int c_in,
                       int n_kb, int pack, int k_vol, const __half* __restrict__ packed, Epi16 epi,
                       __half* __restrict__ out_hi, __half* __restrict__ out_lo, float* __restrict__ out_f32,
                       int* __restrict__ overflow) {
  spconv_os16_body<COUT, 1>(in_hi, in_lo, nbr, tile_mask, n_out_p, out_cap, c_in, n_kb, pack, k_vol, packed, epi, out_hi,
                            out_lo, out_f32, overflow);
}

// ---- first layer: fp32 rows with a handful of channels (C_in <= 16: the voxel mean, 4 or 5 features) -----------------
// 2*27*C_in*C_out flops per row -- nothing for the tensor cores.  fp32 FFMA, output-stationary, same epilogue and
// output format as the tensor-core kernel.  Four lanes share a (row, 16-column part), each taking every fourth offset (their
// neighbour-index loads are independent and in flight together: the kernel is pure latency), combined by a fixed shuffle tree.
template <int COUT, int PLANES>
__device__ __forceinline__ void spconv_first16_body(
    const float* __restrict__ feat_in, const int* __restrict__ nbr, const int* __restrict__ n_out_p, int out_cap, int c_in,
    int in_ld, int k_vol, const float* __restrict__ weight, Epi16 epi, __half* __restrict__ out_hi,
    __half* __restrict__ out_lo, float* __restrict__ out_f32, int* __restrict__ overflow) {
  extern __shared__ float w_s[];                 // [k_vol][c_in][COUT]
  for (int i = threadIdx.x; i < k_vol * c_in * COUT; i += blockDim.x) w_s[i] = weight[i];
  __syncthreads();
  constexpr int kParts = COUT / 16;              // 16-column parts of a row
  constexpr int kSub = 4;                        // lanes per (row, part): lane `sub` takes the offsets k = sub, sub + 4, ...
  constexpr int kMaxK = 8;                       // ceil(32 / 4) offsets per lane at most
  const int n_out = min(*n_out_p, out_cap);
  const long long items = (long long)n_out * kParts;
  const long long items_pad = (items + 7) / 8 * 8;          // whole warps (8 items each) run the shuffles together
  bool ovf = false;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < items_pad * kSub; e += (long long)gridDim.x * blockDim.x) {
    const long long item = e / kSub;
    const int sub = (int)(e % kSub);
    const bool on = item < items;
    const int o = on ? (int)(item / kParts) : 0, col = (int)(item % kParts) * 16;
    int src[kMaxK];
#pragma unroll
    for (int t = 0; t < kMaxK; ++t) {            // the neighbour indices first: independent loads, all in flight together
      const int k = sub + t * kSub;
      src[t] = (on && k < k_vol) ? __ldg(nbr + (size_t)k * out_cap + o) : -1;
    }
    float acc[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[q] = 0.f;
#pragma unroll
    for (int t = 0; t < kMaxK; ++t) {
      if (src[t] < 0) continue;
      const int k = sub + t * kSub;
      for (int ci = 0; ci < c_in; ++ci) {
        const float a = __ldg(feat_in + (size_t)src[t] * in_ld + ci);
        const float* w = w_s + ((size_t)k * c_in + ci) * COUT + col;
#pragma unroll
        for (int q = 0; q < 16; ++q) acc[q] = fmaf(a, w[q], acc[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) {               // fixed-order tree over the four offset classes
      acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], 1);
      acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], 2);
    }
    if (on && sub == 0) ovf |= epilogue16<PLANES>(acc, epi, (size_t)o * COUT, col, out_hi, out_lo, out_f32);
  }
  if (ovf && overflow) atomicOr(overflow, 1);
}

template <int COUT>
__global__ void __launch_bounds__(256)
spconv_first16_kernel(const float* __restrict__ feat_in, const int* __restrict__ nbr, const int* __restrict__ n_out_p,
                      int out_cap, int c_in, int in_ld, int k_vol, const float* __restrict__ weight, Epi16 epi,
                      __half* __restrict__ out_hi, __half* __restrict__ out_lo, float* __restrict__ out_f32,
                      int* __restrict__ overflow) {
  spconv_first16_body<COUT, 2>(feat_in, nbr, n_out_p, out_cap, c_in, in_ld, k_vol, weight, epi, out_hi, out_lo, out_f32,
                               overflow);
}

// Single-pass FP16: writes the hi plane only.
template <int COUT>
__global__ void __launch_bounds__(256)
spconv_first16_f16_kernel(const float* __restrict__ feat_in, const int* __restrict__ nbr, const int* __restrict__ n_out_p,
                          int out_cap, int c_in, int in_ld, int k_vol, const float* __restrict__ weight, Epi16 epi,
                          __half* __restrict__ out_hi, __half* __restrict__ out_lo, float* __restrict__ out_f32,
                          int* __restrict__ overflow) {
  spconv_first16_body<COUT, 1>(feat_in, nbr, n_out_p, out_cap, c_in, in_ld, k_vol, weight, epi, out_hi, out_lo, out_f32,
                               overflow);
}

// ---- f16 weight image ------------------------------------------------------------------------------------------------
// packed[slot][kb][part][n][swizzled 64 halves], part 0 = hi, 1 = lo of w * 2^w_exp; zero beyond c_in.  slot = kernel
// offset, or with offset packing (C_in 16 / 32, see os16_pack) a group of `pack` offsets side by side along K.
__global__ void __launch_bounds__(256)
pack_weight16_kernel(const float* __restrict__ w, int c_in, int c_out, int k_vol, int n_slots_k, int n_kb, int pack,
                     float w_mul, __half* __restrict__ packed) {
  const long long total = (long long)n_slots_k * n_kb * 2 * c_out * kOsKc;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    long long t = e;
    const int cc = (int)(t % kOsKc); t /= kOsKc;
    const int n = (int)(t % c_out); t /= c_out;
    const int part = (int)(t % 2); t /= 2;
    const int kb = (int)(t % n_kb); t /= n_kb;
    int k = (int)t;                                  // slot
    int ci = kb * kOsKc + cc;
    if (pack > 1) { k = k * pack + cc / c_in; ci = cc % c_in; }
    const float x = (ci < c_in && k < k_vol) ? w[((size_t)k * c_in + ci) * c_out + n] * w_mul : 0.0f;
    k = (int)t;
    __half hi, lo;
    split_f16(x, hi, lo);
    const size_t tile = (((size_t)k * n_kb + kb) * 2 + part) * (size_t)(c_out * kOsKc);
    const uint32_t off = sw128_offset(n, cc >> 3) + (cc & 7) * 2;     // bytes
    packed[tile + off / 2] = part == 0 ? hi : lo;
  }
}

// ---- plane <-> fp32 conversions (API boundary, tests); PLANES = 1 reads / writes the hi plane alone -------------------
template <int PLANES>
__global__ void __launch_bounds__(256)
split16_kernel(const float* __restrict__ x, long long n, __half* __restrict__ hi, __half* __restrict__ lo,
               int* __restrict__ overflow) {
  bool ovf = false;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    ovf |= store16p<PLANES>(x[e], hi + e, lo + e);
  }
  if (ovf && overflow) atomicOr(overflow, 1);
}

template <int PLANES>
__global__ void __launch_bounds__(256)
merge16_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, long long n, float* __restrict__ x) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    if constexpr (PLANES == 2) x[e] = __half2float(hi[e]) + __half2float(lo[e]);
    else x[e] = __half2float(hi[e]);
  }
}

// rows (f16 planes or fp32) -> channels-last BEV planes [B*H*W, C*D] (pre-zeroed), channel = c*D + z: the values of
// `dense.view(B, C*D, H, W)` (scn.py:192-195) in NHWC order.  fp32 rows are split here, so a written value outside the
// f16 range ORs 1 into `overflow`; plane rows were range-checked by the kernel that wrote them.  The OR is issued where
// the value is met, by the lowest lane of the lanes that meet one together: a per-thread flag carried to the end of the
// grid-stride loop (as in split16_kernel) takes this kernel from 32 to 40 registers, and the PointPillars reader +
// scatter stage (B = 8) from 0.191 to 0.201 ms in the replayed graph on an H100 80GB HBM3 at 700 W; this form keeps it
// at 26 registers and 0.192 ms.  PLANES = 1 copies / rounds into the hi plane only.
template <int PLANES>
__global__ void __launch_bounds__(256)
sparse_to_bev16_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, const float* __restrict__ in_f32,
                       const int* __restrict__ coors, const int* __restrict__ n_rows, int row_cap, int C, int D, int H,
                       int W, int B, __half* __restrict__ out_hi, __half* __restrict__ out_lo, int* __restrict__ overflow) {
  const int n = min(*n_rows, row_cap);
  const long long total = (long long)n * C;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / C), c = (int)(e - (long long)r * C);
    const int4 q = *reinterpret_cast<const int4*>(coors + (size_t)r * 4);
    if ((unsigned)q.x >= (unsigned)B || (unsigned)q.y >= (unsigned)D || (unsigned)q.z >= (unsigned)H ||
        (unsigned)q.w >= (unsigned)W)
      continue;
    const size_t dst = (((size_t)q.x * H + q.z) * W + q.w) * ((size_t)C * D) + (size_t)c * D + q.y;
    if (in_f32) {
      if (store16p<PLANES>(in_f32[e], out_hi + dst, out_lo + dst) && overflow) {
        if ((__activemask() & ((1u << (threadIdx.x & 31)) - 1u)) == 0u) atomicOr(overflow, 1);
      }
    } else {
      out_hi[dst] = in_hi[e];
      if constexpr (PLANES == 2) out_lo[dst] = in_lo[e];
    }
  }
}

static bool os16_shape_ok(int c_in, int c_out) {
  const bool cin_ok = c_in >= 8 && c_in <= 512 && c_in % 8 == 0;    // rows are gathered in 16-byte chunks
  const bool cout_ok = c_out == 16 || c_out == 32 || c_out == 64 || c_out == 128;
  return cin_ok && cout_ok;
}

static Epi16 epi_of(const d3b_conv16_params* p) {
  Epi16 e;
  e.bias = p->bias; e.scale = p->scale; e.shift = p->shift;
  e.res_hi = (const __half*)p->residual_hi; e.res_lo = (const __half*)p->residual_lo;
  e.acc_scale = p->acc_scale; e.relu = p->relu;
  e.corr = 0.f;                                   // (set by the tensor-core launch; the FFMA first layer is exact-sum)
  static std::atomic<int> launch_seq{0};
  e.seq = launch_seq.fetch_add(1, std::memory_order_relaxed);
  return e;
}

template <int COUT, int PLANES>
static int launch_os16(const d3b_conv16_params* p, const int32_t* nbr, const uint32_t* tile_mask, const int32_t* n_out,
                       int32_t out_cap, cudaStream_t stream) {
  using Cfg = OsCfg<COUT, PLANES>;
  constexpr auto kernel = PLANES == 2 ? spconv_os16_kernel<COUT> : spconv_os16_f16_kernel<COUT>;
  static SmemOptIn optin;
  D3B_CUDA(ensure_dynamic_smem(kernel, Cfg::kSmemBytes, optin));
  const int n_tiles = div_up(out_cap, kOsTileM);
  const int grid = n_tiles < kNumSMs ? (n_tiles > 0 ? n_tiles : 1) : kNumSMs;
  const int pack = os16_pack(p->c_in, p->k_vol);
  const int n_kb = pack > 1 ? 1 : (p->c_in + kOsKc - 1) / kOsKc;
  Epi16 epi = epi_of(p);
  epi.corr = trunc_correction(p->c_in * pack, PLANES == 2 ? 3 : 1);
  D3B_CUDA(launch_maybe_pdl(kernel, dim3(grid), dim3(Cfg::kThreads), Cfg::kSmemBytes, stream,
                            (const __half*)p->in_hi, (const __half*)p->in_lo, (const int*)nbr, (const unsigned int*)tile_mask,
                            (const int*)n_out, (int)out_cap, (int)p->c_in, n_kb, pack, (int)p->k_vol,
                            (const __half*)p->weight_packed, epi,
                            (__half*)p->out_hi, (__half*)p->out_lo, p->out_f32, (int*)p->overflow));
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

template <int COUT, int PLANES>
static int launch_first16(const d3b_conv16_params* p, const int32_t* nbr, const int32_t* n_out, int32_t out_cap,
                          cudaStream_t stream) {
  constexpr auto kernel = PLANES == 2 ? spconv_first16_kernel<COUT> : spconv_first16_f16_kernel<COUT>;
  const size_t smem = (size_t)p->k_vol * p->c_in * COUT * sizeof(float);
  static SmemOptIn optin;
  D3B_REQUIRE(smem <= 160 * 1024, "first-layer sparse conv: weights (%zu bytes) do not fit in shared memory", smem);
  D3B_CUDA(ensure_dynamic_smem(kernel, smem, optin));
  const int grid = grid_for((long long)out_cap * (COUT / 16) * 4, 256, 8);
  const int in_ld = p->in_f32_ld ? p->in_f32_ld : p->c_in;
  kernel<<<grid, 256, smem, stream>>>(p->in_f32, nbr, n_out, out_cap, p->c_in, in_ld, p->k_vol, p->weight,
                                                         epi_of(p), (__half*)p->out_hi, (__half*)p->out_lo, p->out_f32,
                                                         p->overflow);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

}  // namespace d3b

using namespace d3b;

extern "C" size_t d3b_conv16_packed_weight_halves(int32_t c_in, int32_t c_out, int32_t k_vol) {
  if (c_in < 1 || c_in > 512 || k_vol < 1 || k_vol > 32) return 0;
  if (!(c_out == 16 || c_out == 32 || c_out == 64 || c_out == 128)) return 0;
  const int pack = os16_pack(c_in, k_vol);
  const int n_kb = pack > 1 ? 1 : (c_in + kOsKc - 1) / kOsKc;
  return (size_t)div_up(k_vol, pack) * n_kb * 2 * c_out * kOsKc;
}

extern "C" int d3b_conv16_pack_weight(const float* weight_dev, int32_t c_in, int32_t c_out, int32_t k_vol,
                                      int32_t w_exp, void* packed_dev, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(weight_dev && packed_dev, "d3b_conv16_pack_weight: null argument");
  D3B_REQUIRE(w_exp >= -60 && w_exp <= 60, "d3b_conv16_pack_weight: w_exp %d outside [-60, 60]", w_exp);
  const size_t n = d3b_conv16_packed_weight_halves(c_in, c_out, k_vol);
  if (n == 0) {
    set_error("d3b_conv16_pack_weight: unsupported C_in=%d C_out=%d k_vol=%d", c_in, c_out, k_vol);
    return D3B_ERR_UNSUPPORTED;
  }
  const int pack = os16_pack(c_in, k_vol);
  const int n_kb = pack > 1 ? 1 : (c_in + kOsKc - 1) / kOsKc;
  pack_weight16_kernel<<<grid_for((long long)n, 256), 256, 0, stream>>>(weight_dev, c_in, c_out, k_vol, div_up(k_vol, pack),
                                                                        n_kb, pack, ldexpf(1.0f, w_exp), (__half*)packed_dev);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_sparse_conv16(const int32_t* nbr, const uint32_t* tile_mask, const int32_t* n_out, int32_t out_cap,
                                 const d3b_conv16_params* p, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(nbr && n_out && p, "d3b_sparse_conv16: null argument");
  D3B_REQUIRE(p->k_vol >= 1 && p->k_vol <= 32 && out_cap >= 0, "d3b_sparse_conv16: bad shape (k_vol %d)", p->k_vol);
  D3B_REQUIRE(p->out_hi || p->out_f32, "d3b_sparse_conv16: give out_hi (+ out_lo) and/or out_f32");
  D3B_REQUIRE((p->scale == nullptr) == (p->shift == nullptr), "d3b_sparse_conv16: scale and shift go together");
  PlanePairs pp;
  pp.add(p->in_f32 ? nullptr : p->in_hi, p->in_lo);
  pp.add(p->out_hi, p->out_lo);
  pp.add(p->residual_hi, p->residual_lo);
  D3B_REQUIRE(pp.consistent(),
              "d3b_sparse_conv16: give in_lo, out_lo and residual_lo with their hi planes (FP16x3) or none of them "
              "(single-pass FP16); got in_lo %s, out_lo %s, residual_lo %s",
              p->in_lo ? "set" : "NULL", p->out_lo ? "set" : "NULL", p->residual_lo ? "set" : "NULL");
  const bool two = pp.planes() == 2;
  if (out_cap == 0) return D3B_OK;
  if (p->in_f32) {      // first layer: fp32 rows, few channels
    D3B_REQUIRE(p->weight && p->c_in >= 1 && p->c_in <= 16, "d3b_sparse_conv16: fp32-input layers need weight and C_in <= 16");
    D3B_REQUIRE(p->in_f32_ld == 0 || p->in_f32_ld >= p->c_in, "d3b_sparse_conv16: in_f32_ld %d < C_in %d", p->in_f32_ld,
                p->c_in);
    switch (p->c_out) {
      case 16: return two ? launch_first16<16, 2>(p, nbr, n_out, out_cap, stream) : launch_first16<16, 1>(p, nbr, n_out, out_cap, stream);
      case 32: return two ? launch_first16<32, 2>(p, nbr, n_out, out_cap, stream) : launch_first16<32, 1>(p, nbr, n_out, out_cap, stream);
      case 64: return two ? launch_first16<64, 2>(p, nbr, n_out, out_cap, stream) : launch_first16<64, 1>(p, nbr, n_out, out_cap, stream);
      default:
        set_error("d3b_sparse_conv16: fp32-input layer with C_out=%d (16/32/64 built)", p->c_out);
        return D3B_ERR_UNSUPPORTED;
    }
  }
  D3B_REQUIRE(tile_mask && p->in_hi && p->weight_packed, "d3b_sparse_conv16: null planes / tile_mask / packed weights");
  if (!os16_shape_ok(p->c_in, p->c_out)) {
    set_error("d3b_sparse_conv16: unsupported C_in=%d C_out=%d", p->c_in, p->c_out);
    return D3B_ERR_UNSUPPORTED;
  }
  switch (p->c_out) {
    case 16: return two ? launch_os16<16, 2>(p, nbr, tile_mask, n_out, out_cap, stream) : launch_os16<16, 1>(p, nbr, tile_mask, n_out, out_cap, stream);
    case 32: return two ? launch_os16<32, 2>(p, nbr, tile_mask, n_out, out_cap, stream) : launch_os16<32, 1>(p, nbr, tile_mask, n_out, out_cap, stream);
    case 64: return two ? launch_os16<64, 2>(p, nbr, tile_mask, n_out, out_cap, stream) : launch_os16<64, 1>(p, nbr, tile_mask, n_out, out_cap, stream);
    default: return two ? launch_os16<128, 2>(p, nbr, tile_mask, n_out, out_cap, stream) : launch_os16<128, 1>(p, nbr, tile_mask, n_out, out_cap, stream);
  }
}

// lo == NULL: the single plane hi = f16(x) (split16), x = hi (merge16)
extern "C" int d3b_split16(const float* x, int64_t n, void* hi, void* lo, int32_t* overflow, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(n >= 0 && (n == 0 || (x && hi)), "d3b_split16: null argument");
  if (n == 0) return D3B_OK;
  if (lo) split16_kernel<2><<<grid_for(n, 256), 256, 0, stream>>>(x, n, (__half*)hi, (__half*)lo, overflow);
  else split16_kernel<1><<<grid_for(n, 256), 256, 0, stream>>>(x, n, (__half*)hi, nullptr, overflow);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_merge16(const void* hi, const void* lo, int64_t n, float* x, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(n >= 0 && (n == 0 || (x && hi)), "d3b_merge16: null argument");
  if (n == 0) return D3B_OK;
  if (lo) merge16_kernel<2><<<grid_for(n, 256), 256, 0, stream>>>((const __half*)hi, (const __half*)lo, n, x);
  else merge16_kernel<1><<<grid_for(n, 256), 256, 0, stream>>>((const __half*)hi, nullptr, n, x);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_sparse_to_bev16(const void* in_hi, const void* in_lo, const float* in_f32, const int32_t* coors,
                                   const int32_t* n_rows, int32_t row_cap, int32_t channels, const int32_t spatial[3],
                                   int32_t batch, void* out_hi, void* out_lo, int32_t* overflow, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(coors && n_rows && spatial && out_hi, "d3b_sparse_to_bev16: null argument");
  D3B_REQUIRE((in_f32 != nullptr) != (in_hi != nullptr), "d3b_sparse_to_bev16: give fp32 rows OR planes");
  PlanePairs pp;
  pp.add(in_hi, in_lo);
  pp.add(out_hi, out_lo);
  D3B_REQUIRE(pp.consistent(),
              "d3b_sparse_to_bev16: give in_lo (plane rows) and out_lo together (FP16x3) or neither (single-pass FP16); "
              "got in_lo %s, out_lo %s", in_lo ? "set" : "NULL", out_lo ? "set" : "NULL");
  D3B_REQUIRE(channels >= 1 && batch >= 1 && row_cap >= 0, "d3b_sparse_to_bev16: bad shape");
  if (row_cap == 0) return D3B_OK;
  const int grid = grid_for((long long)row_cap * channels, 256);
  if (pp.planes() == 2)
    sparse_to_bev16_kernel<2><<<grid, 256, 0, stream>>>((const __half*)in_hi, (const __half*)in_lo, in_f32, coors, n_rows,
                                                        row_cap, channels, spatial[0], spatial[1], spatial[2], batch,
                                                        (__half*)out_hi, (__half*)out_lo, overflow);
  else
    sparse_to_bev16_kernel<1><<<grid, 256, 0, stream>>>((const __half*)in_hi, nullptr, in_f32, coors, n_rows, row_cap,
                                                        channels, spatial[0], spatial[1], spatial[2], batch,
                                                        (__half*)out_hi, nullptr, overflow);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

#ifdef D3B_SOFT_TIMEOUT
extern "C" int d3b_debug_fault_spconv16(unsigned int* host8) {
  cudaError_t e = cudaMemcpyFromSymbol(host8, d3b::g_d3b_fault, 32);
  unsigned int zeros[8] = {0};
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(d3b::g_d3b_fault, zeros, 32);
  return (int)e;
}
extern "C" int d3b_debug_cta_ns_spconv16(unsigned long long* host4096) {
  return (int)cudaMemcpyFromSymbol(host4096, d3b::g_d3b_cta_ns, sizeof(unsigned long long) * 4096);
}
extern "C" int d3b_debug_cta_clk_spconv16(long long* host4096) {
  return (int)cudaMemcpyFromSymbol(host4096, d3b::g_d3b_cta_clk, sizeof(long long) * 4096);
}
extern "C" int d3b_debug_trace_spconv16(long long* host, int clear) {
  cudaError_t e = cudaMemcpyFromSymbol(host, d3b::g_d3b_trace, sizeof(long long) * 16 * 512);
  if (e == cudaSuccess && clear) {
    static long long zeros[16 * 512];
    e = cudaMemcpyToSymbol(d3b::g_d3b_trace, zeros, sizeof(zeros));
  }
  return (int)e;
}
#endif
