// Output-stationary sparse convolution on the Hopper tensor cores (sm_90a, wgmma).
//
//   out[o,:] = act((sum_k in[nbr[k][o],:] . W[k] + bias) * scale + shift + residual[o,:])
//
// The reference computes this contraction as fp32 SGEMMs (spconv v1.x indice_conv:
// per offset gather -> torch.mm -> scatter-add; call sites
// det3d/models/backbones/scn.py:106-157).  Here one CTA owns 128 output rows; for
// every kernel offset that has a neighbour in the tile (tile_mask) and every 32-channel
// slice of C_in ("slot"), a group of four producer warps gathers the 128 input rows
// straight from global/L2 into a K-major, 128B-swizzled shared-memory tile, and two
// consumer warpgroups (64 rows each) issue wgmma.m64nNk8.tf32 accumulating in registers.
// No scatter, no atomics; BN/bias/residual/ReLU are applied on the way out of the registers.
//
// fp32-equivalent accuracy ("3xTF32"): every fp32 operand x is split exactly into
//   hi = x with the low 13 mantissa bits cleared (a TF32 number), lo = x - hi (13 bits),
// and D += A_lo.B_hi + A_hi.B_lo + A_hi.B_hi with fp32 accumulation; the dropped
// lo.lo term is O(2^-22) relative.  Activations are split in registers while being
// gathered; weights are split once at load time by d3b_conv_pack_weight, which also
// lays them out as the exact shared-memory image (K-major, 128B swizzle) so that one
// cp.async.bulk (TMA) per slot brings the B operand in.
//
// Pipeline: NSTAGE-deep ring of {A_hi, A_lo, B_hi, B_lo} tiles guarded by full/empty
// mbarriers; producers -> (generic-proxy stores + fence.proxy.async + arrive),
// TMA -> complete_tx, consumer warps -> arrive on the empty barrier once their wgmmas have
// read the stage.  Two producer groups take alternate slots so two global round trips are in
// flight per SM (a thread cannot keep loads in flight across fence.proxy.async: the fence waits
// for them); the tile's neighbour indices are staged in shared memory once per tile.  Persistent
// grid (<= one CTA per SM), 16 warps: 8 gather, 8 MMA + epilogue.
//
// Algorithmic bytes per layer: N_in*C_in*4 + N_out*C_out*4 + P*8 + K*C_in*C_out*4
// (SURVEY 8d); tensor work issued: 3 * 2 * 128 * C_out * 32 flop per slot.
#include "gmma.cuh"

namespace d3b {

constexpr int kTcTileM = 128;
constexpr int kTcKc = 32;               // channels per stage = one 128-byte swizzle row
constexpr int kTcGroups = 2;            // gather groups of 4 warps, each producing every 2nd pipeline slot
constexpr int kTcMathWarp0 = 4 * kTcGroups;               // two consumer warpgroups (warpgroup-aligned)
constexpr int kTcMathWarps = 8;
constexpr int kTcThreads = 32 * (kTcMathWarp0 + kTcMathWarps);   // 512
constexpr int kABytes = kTcTileM * 128; // one A tile (hi or lo)
constexpr uint32_t kHalfTileBytes = 64 * 128;             // rows 64..127 of a K-major SW128 tile start here

template <int COUT>
struct TcCfg {
  static constexpr int kBBytes = COUT * 128;                       // one B tile (hi or lo)
  static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
  static constexpr int kStages = (COUT >= 128) ? 3 : 4;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers, offsets*/ +
                                    32 * kTcTileM * 4 /*neighbour rows of the tile*/;
};

// the three split products of one 32-channel slot (4 k-steps), small terms first
template <int COUT>
__device__ __forceinline__ void tf32x3_slot(float (&acc)[COUT / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                            uint32_t b_lo) {
  gmma_fence();
#pragma unroll
  for (int kk = 0; kk < kTcKc / 8; ++kk) {
    const uint32_t adv = kk * 32;  // 8 tf32 = 32 bytes along K inside the swizzle row
    wgmma_tf32<COUT>(acc, gmma_desc_sw128(a_lo + adv), gmma_desc_sw128(b_hi + adv), 1u);
    wgmma_tf32<COUT>(acc, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_lo + adv), 1u);
    wgmma_tf32<COUT>(acc, gmma_desc_sw128(a_hi + adv), gmma_desc_sw128(b_hi + adv), 1u);
  }
  gmma_commit();
  gmma_wait();
  gmma_fence_regs(acc);
}

template <int COUT>
__global__ void __launch_bounds__(kTcThreads, 1)
spconv_tc_kernel(const float* __restrict__ feat_in, const int* __restrict__ nbr,
                 const unsigned int* __restrict__ tile_mask, const int* __restrict__ n_out_p, int out_cap,
                 int c_in, int n_kb, const float* __restrict__ packed, const float* __restrict__ bias,
                 const float* __restrict__ scale, const float* __restrict__ shift,
                 const float* __restrict__ residual, int relu, float* __restrict__ feat_out) {
  using Cfg = TcCfg<COUT>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + Cfg::kStages * Cfg::kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };
  int* koff_s = reinterpret_cast<int*>(smem_gen + Cfg::kStages * Cfg::kStageBytes + 128);          // [32] active offsets
  int* nbr_s = reinterpret_cast<int*>(smem_gen + Cfg::kStages * Cfg::kStageBytes + 256);           // [32][128] neighbour rows

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_out = min(*n_out_p, out_cap);
  const int n_tiles = (n_out + kTcTileM - 1) / kTcTileM;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(full_bar(s), 128 + 1);        // the 128 gather threads of one group + the expect_tx arrive
      mbar_init(empty_bar(s), kTcMathWarps);  // every consumer warp, after its wgmmas have read the stage
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < kTcMathWarp0) {
    // ============ gather producers (kTcGroups groups of 4 warps) ============
    // Group g produces the pipeline slots it with it % kTcGroups == g, so kTcGroups dependent
    // "feature rows -> shared memory" chains are in flight per SM.  A thread must not hold
    // outstanding global loads across fence.proxy.async (the fence waits for them), hence no
    // register prefetch: latency is hidden across groups, and the tile's neighbour indices are
    // staged in shared memory once per tile so a slot costs one global round trip, not two.
    const int group = warp >> 2, wq = warp & 3;
    const int g = lane >> 3, c = lane & 7;
    const bool issues_tma = (wq == 0 && lane == 0);
    const int ptid = threadIdx.x;  // 0 .. 128*kTcGroups-1 (producer threads come first)
    uint32_t it0 = 0;       // pipeline slots consumed by earlier tiles (same sequence in every role)
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int row0 = tile * kTcTileM;
      const unsigned int mask = tile_mask[tile];
      const int n_off = __popc(mask);
      const int n_slots = n_off * n_kb;

      // ---- stage nbr[k][row0 .. row0+127] for the active offsets (one global round trip) ----
      asm volatile("bar.sync 1, %0;" ::"r"(128 * kTcGroups) : "memory");   // previous tile's readers are done
      for (int idx = ptid; idx < n_off * kTcTileM; idx += 128 * kTcGroups) {
        const int n = idx >> 7, r = idx & 127;
        unsigned int m = mask;
        for (int t = n; t > 0; --t) m &= m - 1;
        const int k = __ffs(m) - 1;
        if (r == 0) koff_s[n] = k;
        nbr_s[idx] = (row0 + r < n_out) ? __ldg(nbr + (size_t)k * out_cap + row0 + r) : -1;
      }
      asm volatile("bar.sync 1, %0;" ::"r"(128 * kTcGroups) : "memory");

      for (int j = (int)((group + kTcGroups - (it0 % kTcGroups)) % kTcGroups); j < n_slots; j += kTcGroups) {
        const int n = j / n_kb, kb = j - n * n_kb;
        const int ch = kb * kTcKc + c * 4;
        float4 v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int src = nbr_s[n * kTcTileM + wq * 32 + 4 * q + g];
          v[q] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (src >= 0 && ch < c_in) v[q] = __ldg(reinterpret_cast<const float4*>(feat_in + (size_t)src * c_in + ch));
        }
        const uint32_t it = it0 + (uint32_t)j;
        const int s = it % Cfg::kStages;
        const uint32_t ph = (it / Cfg::kStages) & 1u;
        mbar_wait(empty_bar(s), ph ^ 1u);
        uint8_t* stage = smem_gen + (size_t)s * Cfg::kStageBytes;
        if (issues_tma) {
          mbar_arrive_expect_tx(full_bar(s), 2 * Cfg::kBBytes);
          tma_bulk_g2s(smem_base + s * Cfg::kStageBytes + 2 * kABytes,
                       packed + ((size_t)koff_s[n] * n_kb + kb) * (2 * Cfg::kBBytes / 4), 2 * Cfg::kBBytes,
                       full_bar(s));
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int row = wq * 32 + 4 * q + g;
          float4 hi, lo;
          split_tf32(v[q].x, hi.x, lo.x);
          split_tf32(v[q].y, hi.y, lo.y);
          split_tf32(v[q].z, hi.z, lo.z);
          split_tf32(v[q].w, hi.w, lo.w);
          const uint32_t off = sw128_offset(row, c);
          *reinterpret_cast<float4*>(stage + off) = hi;
          *reinterpret_cast<float4*>(stage + kABytes + off) = lo;
        }
        fence_proxy_async();      // generic-proxy stores -> visible to the tensor core (async proxy)
        mbar_arrive(full_bar(s));
      }
      it0 += (uint32_t)n_slots;
    }
  } else {
    // ===================== consumer warpgroups: wgmma into registers, fused bias/BN/residual/ReLU -> global =====================
    const int wg = (warp - kTcMathWarp0) >> 2;      // rows [64 wg, 64 wg + 64) of the tile
    const int wq = warp & 3;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const unsigned int mask = tile_mask[tile];
      const int n_slots = __popc(mask) * n_kb;
      float acc[COUT / 2];
#pragma unroll
      for (int q = 0; q < COUT / 2; ++q) acc[q] = 0.f;
      for (int j = 0; j < n_slots; ++j, ++it) {
        const int s = it % Cfg::kStages;
        const uint32_t ph = (it / Cfg::kStages) & 1u;
        mbar_wait(full_bar(s), ph);
        const uint32_t a_hi = smem_base + s * Cfg::kStageBytes + wg * kHalfTileBytes;
        const uint32_t b_hi = smem_base + s * Cfg::kStageBytes + 2 * kABytes;
        tf32x3_slot<COUT>(acc, a_hi, a_hi + kABytes, b_hi, b_hi + Cfg::kBBytes);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(s));   // this warp's share of the stage has been read
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = tile * kTcTileM + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (o >= n_out) continue;
#pragma unroll
        for (int jn = 0; jn < COUT / 8; ++jn) {
          const int col = jn * 8 + 2 * (lane & 3);
          float2 val = make_float2(acc[4 * jn + 2 * h], acc[4 * jn + 2 * h + 1]);
          if (bias) {
            const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + col));
            val.x += b2.x; val.y += b2.y;
          }
          if (scale) {
            const float2 s2 = __ldg(reinterpret_cast<const float2*>(scale + col));
            const float2 t2 = __ldg(reinterpret_cast<const float2*>(shift + col));
            val.x = fmaf(val.x, s2.x, t2.x); val.y = fmaf(val.y, s2.y, t2.y);
          }
          if (residual) {
            const float2 q2 = __ldg(reinterpret_cast<const float2*>(residual + (size_t)o * COUT + col));
            val.x += q2.x; val.y += q2.y;
          }
          if (relu) { val.x = fmaxf(val.x, 0.f); val.y = fmaxf(val.y, 0.f); }
          *reinterpret_cast<float2*>(feat_out + (size_t)o * COUT + col) = val;
        }
      }
    }
  }
}

// =============================================================================================
// Pair-based variant (D3B_ALGO_TC_PAIRS): spconv's classic "gather -> GEMM -> scatter-add" on the
// tensor cores.  The output-stationary kernel above pads every (tile, offset) slot to 128 rows; at
// lidar densities only ~1/3 of those rows have a neighbour, so 2/3 of the gather, shared-memory and
// MMA work is padding.  Here the rulebook is first compacted per offset (d3b_rulebook_pairs) and a
// work item is 128 VALID pairs of one offset: every A row is live.  The price: partial sums go to
// the output rows with fp32 atomics (red.global.add.v2.f32), so the summation order -- not the
// value within fp32 rounding -- varies run to run, and the layer's own bias/BN/ReLU cannot be fused
// here; it is applied by the consumer while it gathers (in_bias/in_scale/in_shift/in_relu) or by
// d3b_feature_epilogue.
//
// Roles: 2 gather groups x 4 warps (slots alternate), 2 consumer warpgroups (wgmma + red, 64 rows each).
// =============================================================================================
constexpr int kPairGroups = 2;
constexpr int kPairMathWarp0 = 4 * kPairGroups;                   // warps 8..15
constexpr int kPairThreads = 32 * (kPairMathWarp0 + kTcMathWarps);  // 512

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// stages + barriers/offsets (256) + work-item tables (512) + producer-epilogue parameters (3 x 128 floats)
template <int COUT>
constexpr int kPairSmem = TcCfg<COUT>::kStages * TcCfg<COUT>::kStageBytes + 1024 + 256 + 512 + 3 * 128 * 4;

template <int COUT>
__global__ void __launch_bounds__(kPairThreads, 1)
spconv_pairs_kernel(const float* __restrict__ feat_in, const int* __restrict__ pair_in,
                    const int* __restrict__ pair_out, const int* __restrict__ pair_count, int out_cap, int k_vol,
                    int c_in, int n_kb, const float* __restrict__ packed, const float* __restrict__ in_bias,
                    const float* __restrict__ in_scale, const float* __restrict__ in_shift, int in_relu,
                    float* __restrict__ feat_out) {
  using Cfg = TcCfg<COUT>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + Cfg::kStages * Cfg::kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };
  int* chunk_prefix = reinterpret_cast<int*>(smem_gen + Cfg::kStages * Cfg::kStageBytes + 256);   // [k_vol + 1]
  int* count_s = chunk_prefix + 40;                                                                // [k_vol]
  float* act_s = reinterpret_cast<float*>(smem_gen + Cfg::kStages * Cfg::kStageBytes + 256 + 512);        // [3][128] bias, scale, shift

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(full_bar(s), 128 + 1);
      mbar_init(empty_bar(s), kTcMathWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // the producing layer's deferred epilogue, staged once (identity where a pointer is NULL)
  for (int ch = threadIdx.x; ch < 128; ch += blockDim.x) {
    const bool in = ch < c_in;
    act_s[ch] = (in && in_bias) ? in_bias[ch] : 0.f;
    act_s[128 + ch] = (in && in_scale) ? in_scale[ch] : 1.f;
    act_s[256 + ch] = (in && in_scale) ? in_shift[ch] : 0.f;
  }
  if (warp == 0) {
    // work-item table: one lane per offset (k_vol <= 32), a warp scan instead of k_vol dependent global loads
    const int cnt = lane < k_vol ? min(pair_count[lane], out_cap) : 0;
    const int chunks = (cnt + kTcTileM - 1) / kTcTileM;
    int incl = chunks;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    if (lane < k_vol) {
      count_s[lane] = cnt;
      chunk_prefix[lane] = incl - chunks;
    }
    if (lane == k_vol - 1) chunk_prefix[k_vol] = incl;
  }
  __syncthreads();
  const int n_items = chunk_prefix[k_vol];

  // offset of a work item = number of offsets whose first item precedes it; one LDS + a ballot instead of a
  // k_vol-long dependent walk (every caller is warp-uniform)
  auto item_k = [&](int item) {
    const bool before = lane + 1 < k_vol && chunk_prefix[lane + 1] <= item;
    return __popc(__ballot_sync(0xffffffffu, before));
  };

  if (warp < kPairMathWarp0) {
    // ===================== gather producers =====================
    // A group owns whole work items (alternating with the other group): one round trip for the
    // 128 input-row indices, then the feature rows of TWO 32-channel slices are fetched together,
    // so an item of a 64-channel layer costs two global round trips, not four.
    const int group = warp >> 2, wq = warp & 3;
    const int g = lane >> 3, c = lane & 7;
    const bool issues_tma = (wq == 0 && lane == 0);
    const bool has_act = in_scale != nullptr || in_bias != nullptr || in_relu;
    // Which items this group works on, and which 32-channel slices of them.  A group waits for a stage on the
    // parity of its empty barrier, which is only unambiguous if the previous use of that stage is known to have
    // been consumed; a group's own earlier slots provide that guarantee when they are at most kStages - 1 slots
    // behind, so the split keeps every group's consecutive slots close: items alternate between the groups for
    // n_kb <= 2, both groups take half of every item for n_kb == 4, and the (unused by the named configs)
    // n_kb == 3 case runs on one group.
    auto mine = [&](uint32_t sq) {
      return n_kb == 4 ? true : (n_kb == 3 ? group == 0 : (int)(sq % kPairGroups) == group);
    };
    auto load_src = [&](int item, int (&dst)[8]) {   // the 8 input-row indices this thread gathers for `item`
      const int k = item_k(item);
      const int first = (item - chunk_prefix[k]) * kTcTileM;
      const int cnt = count_s[k];
      const int* pin = pair_in + (size_t)k * out_cap + first;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int row = wq * 32 + 4 * q + g;
        dst[q] = first + row < cnt ? __ldg(pin + row) : -1;
      }
    };
    int item = blockIdx.x;
    uint32_t seq = 0;                     // CTA-local item ordinal
    while (item < n_items && !mine(seq)) { item += gridDim.x; ++seq; }
    int src_next[8];
    if (item < n_items) load_src(item, src_next);
    while (item < n_items) {
      int src[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) src[q] = src_next[q];
      int next_item = item + gridDim.x;
      uint32_t next_seq = seq + 1;
      while (next_item < n_items && !mine(next_seq)) { next_item += gridDim.x; ++next_seq; }
      bool prefetched = false;
      int kb_begin = 0, kb_end = n_kb;
      if (n_kb == 4) {
        kb_begin = 2 * group;
        kb_end = kb_begin + 2;
      }
      const int k = item_k(item);
      for (int kb0 = kb_begin; kb0 < kb_end; kb0 += 2) {
        // the indices of this group's NEXT item travel together with this round's feature rows: one global round
        // trip per item instead of two (they complete before the fence.proxy.async below would wait for them anyway)
        if (!prefetched && next_item < n_items) { load_src(next_item, src_next); prefetched = true; }
        float4 v[2][8];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ch = (kb0 + h) * kTcKc + c * 4;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            v[h][q] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (src[q] >= 0 && ch < c_in && kb0 + h < kb_end)
              v[h][q] = __ldg(reinterpret_cast<const float4*>(feat_in + (size_t)src[q] * c_in + ch));
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int kb = kb0 + h;
          if (kb >= kb_end) break;
          const int ch = kb * kTcKc + c * 4;
          if (has_act && ch < c_in) {
            // deferred epilogue of the producing layer: relu((x + bias) * scale + shift)
            const float4 b4 = *reinterpret_cast<const float4*>(act_s + ch);
            const float4 s4 = *reinterpret_cast<const float4*>(act_s + 128 + ch);
            const float4 t4 = *reinterpret_cast<const float4*>(act_s + 256 + ch);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              if (src[q] >= 0) {
                float4 x = v[h][q];
                x.x += b4.x; x.y += b4.y; x.z += b4.z; x.w += b4.w;
                if (in_scale) {
                  x.x = fmaf(x.x, s4.x, t4.x); x.y = fmaf(x.y, s4.y, t4.y); x.z = fmaf(x.z, s4.z, t4.z); x.w = fmaf(x.w, s4.w, t4.w);
                }
                if (in_relu) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
                v[h][q] = x;
              }
            }
          }
          const uint32_t it = seq * (uint32_t)n_kb + (uint32_t)kb;
          const int s = it % Cfg::kStages;
          const uint32_t ph = (it / Cfg::kStages) & 1u;
          mbar_wait(empty_bar(s), ph ^ 1u);
          uint8_t* stage = smem_gen + (size_t)s * Cfg::kStageBytes;
          if (issues_tma) {
            mbar_arrive_expect_tx(full_bar(s), 2 * Cfg::kBBytes);
            tma_bulk_g2s(smem_base + s * Cfg::kStageBytes + 2 * kABytes,
                         packed + ((size_t)k * n_kb + kb) * (2 * Cfg::kBBytes / 4), 2 * Cfg::kBBytes, full_bar(s));
          }
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int row = wq * 32 + 4 * q + g;
            float4 hi, lo;
            split_tf32(v[h][q].x, hi.x, lo.x);
            split_tf32(v[h][q].y, hi.y, lo.y);
            split_tf32(v[h][q].z, hi.z, lo.z);
            split_tf32(v[h][q].w, hi.w, lo.w);
            const uint32_t off = sw128_offset(row, c);
            *reinterpret_cast<float4*>(stage + off) = hi;
            *reinterpret_cast<float4*>(stage + kABytes + off) = lo;
          }
          fence_proxy_async();
          mbar_arrive(full_bar(s));
        }
      }
      item = next_item;
      seq = next_seq;
    }
  } else {
    // ===================== consumer warpgroups: wgmma into registers -> fp32 atomics on the output rows =====================
    const int wg = (warp - kPairMathWarp0) >> 2;     // rows [64 wg, 64 wg + 64) of the work item
    const int wq = warp & 3;
    uint32_t it = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int k = item_k(item);
      const int first = (item - chunk_prefix[k]) * kTcTileM;
      int o[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = first + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        o[h] = row < count_s[k] ? __ldg(pair_out + (size_t)k * out_cap + row) : -1;
      }
      float acc[COUT / 2];
#pragma unroll
      for (int q = 0; q < COUT / 2; ++q) acc[q] = 0.f;
      for (int kb = 0; kb < n_kb; ++kb, ++it) {
        const int s = it % Cfg::kStages;
        const uint32_t ph = (it / Cfg::kStages) & 1u;
        mbar_wait(full_bar(s), ph);
        const uint32_t a_hi = smem_base + s * Cfg::kStageBytes + wg * kHalfTileBytes;
        const uint32_t b_hi = smem_base + s * Cfg::kStageBytes + 2 * kABytes;
        tf32x3_slot<COUT>(acc, a_hi, a_hi + kABytes, b_hi, b_hi + Cfg::kBBytes);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(s));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (o[h] < 0) continue;
#pragma unroll
        for (int jn = 0; jn < COUT / 8; ++jn)
          red_add_v2(feat_out + (size_t)o[h] * COUT + jn * 8 + 2 * (lane & 3), acc[4 * jn + 2 * h], acc[4 * jn + 2 * h + 1]);
      }
    }
  }
}

__global__ void __launch_bounds__(256)
zero_rows_kernel(float* __restrict__ feat, const int* __restrict__ n_rows, int row_cap, int channels) {
  const long long total = (long long)min(*n_rows, row_cap) * channels / 4;
  float4* p = reinterpret_cast<float4*>(feat);
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
    p[e] = make_float4(0.f, 0.f, 0.f, 0.f);
}

constexpr int kZeroMaxBufs = 16;
struct ZeroList {
  float* buf[kZeroMaxBufs];
  int channels[kZeroMaxBufs];
  int count;
};

// blockIdx.y selects the buffer; every buffer clears its first *n_rows rows
__global__ void __launch_bounds__(256)
zero_rows_multi_kernel(ZeroList list, const int* __restrict__ n_rows, int row_cap) {
  const int c = list.channels[blockIdx.y];
  const long long total = (long long)min(*n_rows, row_cap) * c / 4;
  float4* p = reinterpret_cast<float4*>(list.buf[blockIdx.y]);
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
    p[e] = make_float4(0.f, 0.f, 0.f, 0.f);
}

__global__ void __launch_bounds__(256)
feature_epilogue_kernel(float* __restrict__ feat, const int* __restrict__ n_rows, int row_cap, int channels,
                        const float* __restrict__ bias, const float* __restrict__ scale,
                        const float* __restrict__ shift, const float* __restrict__ residual, int relu) {
  const long long total = (long long)min(*n_rows, row_cap) * channels / 4;
  float4* p = reinterpret_cast<float4*>(feat);
  const int c4 = channels / 4;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(e % c4) * 4;
    float4 x = p[e];
    if (bias) { const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col)); x.x += b.x; x.y += b.y; x.z += b.z; x.w += b.w; }
    if (scale) {
      const float4 s = __ldg(reinterpret_cast<const float4*>(scale + col));
      const float4 t = __ldg(reinterpret_cast<const float4*>(shift + col));
      x.x = fmaf(x.x, s.x, t.x); x.y = fmaf(x.y, s.y, t.y); x.z = fmaf(x.z, s.z, t.z); x.w = fmaf(x.w, s.w, t.w);
    }
    if (residual) { const float4 r = reinterpret_cast<const float4*>(residual)[e]; x.x += r.x; x.y += r.y; x.z += r.z; x.w += r.w; }
    if (relu) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
    p[e] = x;
  }
}

// ---- weight image ------------------------------------------------------------------------
// packed[k][kb][part][n][swizzled 32 floats], part 0 = hi, 1 = lo; zero beyond c_in.
__global__ void __launch_bounds__(256)
pack_weight_kernel(const float* __restrict__ w, int c_in, int c_out, int k_vol, int n_kb,
                   float* __restrict__ packed) {
  const long long total = (long long)k_vol * n_kb * 2 * c_out * kTcKc;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    long long t = e;
    const int cc = (int)(t % kTcKc); t /= kTcKc;   // channel within the slice
    const int n = (int)(t % c_out); t /= c_out;
    const int part = (int)(t % 2); t /= 2;
    const int kb = (int)(t % n_kb); t /= n_kb;
    const int k = (int)t;
    const int ci = kb * kTcKc + cc;
    float x = ci < c_in ? w[((size_t)k * c_in + ci) * c_out + n] : 0.0f;
    float hi, lo;
    split_tf32(x, hi, lo);
    const size_t tile = (((size_t)k * n_kb + kb) * 2 + part) * (size_t)(c_out * kTcKc);
    const uint32_t off = sw128_offset(n, cc >> 2) + (cc & 3) * 4;
    packed[tile + off / 4] = part == 0 ? hi : lo;
  }
}

static bool tc_shape_ok(int c_in, int c_out) {
  const bool cin_ok = c_in >= 4 && c_in <= 128 && c_in % 4 == 0;   // rows are gathered as float4
  const bool cout_ok = c_out == 16 || c_out == 32 || c_out == 64 || c_out == 128;
  return cin_ok && cout_ok;
}

template <int COUT>
static int launch_tc(const float* feat_in, const int32_t* nbr, const uint32_t* tile_mask, const int32_t* n_out,
                     int32_t out_cap, const d3b_conv_params* p, float* feat_out, cudaStream_t stream) {
  using Cfg = TcCfg<COUT>;
  static SmemOptIn optin;
  D3B_CUDA(ensure_dynamic_smem(spconv_tc_kernel<COUT>, Cfg::kSmemBytes, optin));
  const int n_tiles = div_up(out_cap, kTcTileM);
  const int grid = n_tiles < kNumSMs ? (n_tiles > 0 ? n_tiles : 1) : kNumSMs;
  const int n_kb = (p->c_in + kTcKc - 1) / kTcKc;
  spconv_tc_kernel<COUT><<<grid, kTcThreads, Cfg::kSmemBytes, stream>>>(
      feat_in, nbr, tile_mask, n_out, out_cap, p->c_in, n_kb, p->weight_packed, p->bias, p->scale, p->shift,
      p->residual, p->relu, feat_out);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

template <int COUT>
static int launch_pairs(const float* feat_in, const int32_t* n_out, int32_t out_cap, const d3b_conv_params* p,
                        float* feat_out, cudaStream_t stream) {
  using Cfg = TcCfg<COUT>;
  static SmemOptIn optin;
  D3B_CUDA(ensure_dynamic_smem(spconv_pairs_kernel<COUT>, kPairSmem<COUT>, optin));
  if (!p->out_zeroed) {
    zero_rows_kernel<<<grid_for((long long)out_cap * COUT / 4, 256), 256, 0, stream>>>(feat_out, n_out, out_cap, COUT);
    D3B_LAUNCH_CHECK();
  }
  const int n_kb = (p->c_in + kTcKc - 1) / kTcKc;
  spconv_pairs_kernel<COUT><<<kNumSMs, kPairThreads, kPairSmem<COUT>, stream>>>(
      feat_in, p->pair_in, p->pair_out, p->pair_count, out_cap, p->k_vol, p->c_in, n_kb, p->weight_packed, p->in_bias,
      p->in_scale, p->in_shift, p->in_relu, feat_out);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

int sparse_conv_tc_pairs(const float* feat_in, const int32_t* n_out, int32_t out_cap, const d3b_conv_params* p,
                         float* feat_out, cudaStream_t stream) {
  if (!tc_shape_ok(p->c_in, p->c_out)) {
    set_error("pair-based sparse conv: unsupported C_in=%d C_out=%d", p->c_in, p->c_out);
    return D3B_ERR_UNSUPPORTED;
  }
  D3B_REQUIRE(p->weight_packed && p->pair_in && p->pair_out && p->pair_count,
              "pair-based sparse conv: weight_packed / pair lists missing");
  D3B_REQUIRE((p->in_scale == nullptr) == (p->in_shift == nullptr), "in_scale and in_shift must be given together");
  switch (p->c_out) {
    case 16: return launch_pairs<16>(feat_in, n_out, out_cap, p, feat_out, stream);
    case 32: return launch_pairs<32>(feat_in, n_out, out_cap, p, feat_out, stream);
    case 64: return launch_pairs<64>(feat_in, n_out, out_cap, p, feat_out, stream);
    default: return launch_pairs<128>(feat_in, n_out, out_cap, p, feat_out, stream);
  }
}

int sparse_conv_tc(const float* feat_in, const int32_t* nbr, const uint32_t* tile_mask, const int32_t* n_out,
                   int32_t out_cap, const d3b_conv_params* p, float* feat_out, cudaStream_t stream) {
  if (!tc_shape_ok(p->c_in, p->c_out)) {
    set_error("tensor-core sparse conv: unsupported C_in=%d C_out=%d", p->c_in, p->c_out);
    return D3B_ERR_UNSUPPORTED;
  }
  D3B_REQUIRE(p->weight_packed, "tensor-core sparse conv: weight_packed is null (call d3b_conv_pack_weight)");
  D3B_REQUIRE((p->scale == nullptr) == (p->shift == nullptr), "scale and shift must be given together");
  switch (p->c_out) {
    case 16: return launch_tc<16>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
    case 32: return launch_tc<32>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
    case 64: return launch_tc<64>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
    default: return launch_tc<128>(feat_in, nbr, tile_mask, n_out, out_cap, p, feat_out, stream);
  }
}

}  // namespace d3b

using namespace d3b;

extern "C" int d3b_zero_rows(float* const* bufs, const int32_t* channels, int32_t count, const int32_t* n_rows,
                             int32_t row_cap, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(count >= 0 && count <= kZeroMaxBufs && row_cap >= 0, "d3b_zero_rows: count %d outside [0, %d]", count, kZeroMaxBufs);
  if (count == 0 || row_cap == 0) return D3B_OK;
  D3B_REQUIRE(bufs && channels && n_rows, "d3b_zero_rows: null argument");
  ZeroList list;
  int c_max = 0;
  for (int i = 0; i < count; ++i) {
    D3B_REQUIRE(bufs[i] && channels[i] > 0 && channels[i] % 4 == 0, "d3b_zero_rows: buffer %d: null or channels %% 4 != 0", i);
    list.buf[i] = bufs[i];
    list.channels[i] = channels[i];
    c_max = channels[i] > c_max ? channels[i] : c_max;
  }
  list.count = count;
  const dim3 grid((unsigned)grid_for((long long)row_cap * c_max / 4, 256, 2), (unsigned)count);
  zero_rows_multi_kernel<<<grid, 256, 0, stream>>>(list, n_rows, row_cap);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_feature_epilogue(float* feat, const int32_t* n_rows, int32_t row_cap, int32_t channels,
                                    const float* bias, const float* scale, const float* shift,
                                    const float* residual, int32_t relu, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(feat && n_rows && channels >= 4 && channels % 4 == 0 && row_cap >= 0, "d3b_feature_epilogue: bad argument");
  D3B_REQUIRE((scale == nullptr) == (shift == nullptr), "d3b_feature_epilogue: scale and shift go together");
  if (row_cap == 0) return D3B_OK;
  feature_epilogue_kernel<<<grid_for((long long)row_cap * channels / 4, 256), 256, 0, stream>>>(
      feat, n_rows, row_cap, channels, bias, scale, shift, residual, relu);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" size_t d3b_conv_packed_weight_floats(int32_t c_in, int32_t c_out, int32_t k_vol) {
  if (!tc_shape_ok(c_in, c_out) || k_vol < 1 || k_vol > 32) return 0;
  const int n_kb = (c_in + kTcKc - 1) / kTcKc;
  return (size_t)k_vol * n_kb * 2 * c_out * kTcKc;
}

extern "C" int d3b_conv_pack_weight(const float* weight_dev, int32_t c_in, int32_t c_out, int32_t k_vol,
                                    float* packed_dev, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(weight_dev && packed_dev, "d3b_conv_pack_weight: null argument");
  const size_t n = d3b_conv_packed_weight_floats(c_in, c_out, k_vol);
  if (n == 0) {
    set_error("d3b_conv_pack_weight: unsupported C_in=%d C_out=%d k_vol=%d", c_in, c_out, k_vol);
    return D3B_ERR_UNSUPPORTED;
  }
  const int n_kb = (c_in + kTcKc - 1) / kTcKc;
  pack_weight_kernel<<<grid_for((long long)n, 256), 256, 0, stream>>>(weight_dev, c_in, c_out, k_vol, n_kb, packed_dev);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}
