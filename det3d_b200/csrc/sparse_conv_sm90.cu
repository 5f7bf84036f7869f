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
