// What every kernel that writes FP16x3 planes shares (spconv16_sm90.cu, bevconv16_sm90.cu): the epilogue parameters
// of a convolution launch, the split of fp32 values into the planes hi = f16(v), lo = f16(v - hi), and the f16-range
// guard.  A value the planes cannot hold (|v| >= 65504, inf or NaN) is not saturated silently: the writer ORs 1 into the
// launch's overflow flag, and the host re-runs that forward on the tf32x3 kernels (DESIGN 3.0).
#pragma once
#include "gmma.cuh"

namespace d3b {

// Epilogue parameters of one launch; null pointers switch their step off (scale and shift go together, so do the
// residual planes).
struct Epi16 {
  const float* bias;
  const float* scale;             // folded BatchNorm: v * scale + shift
  const float* shift;
  const __half* res_hi;           // residual planes, rows laid out like the output (sparse layers)
  const __half* res_lo;
  float acc_scale;
  float corr;                     // mean truncation of the layer's partials (gmma.cuh), applied to the sums
  int relu;
  int seq;                        // launch counter of the translation unit (development traces only)
};

// The range guard: true when v cannot be written to the planes.  (NaN fails `<` as well.)
__device__ __forceinline__ bool f16_out_of_range(float v) { return !(fabsf(v) < 65504.f); }

__device__ __forceinline__ uint32_t pack_half2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// hi / lo of two consecutive values as half2 words; returns the range bit of either value
__device__ __forceinline__ bool split_pack2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  __half h0, l0, h1, l1;
  split_f16(v0, h0, l0);
  split_f16(v1, h1, l1);
  hi = pack_half2(h0, h1);
  lo = pack_half2(l0, l1);
  return f16_out_of_range(v0) | f16_out_of_range(v1);
}

// One value into the planes; returns its range bit.
__device__ __forceinline__ bool store16(float v, __half* hi, __half* lo) {
  __half h, l;
  split_f16(v, h, l);
  *hi = h;
  *lo = l;
  return f16_out_of_range(v);
}

// Host side: the plane count of a launch from its (hi, lo) pointer pairs.  A null lo plane selects single-pass FP16,
// so either every pair that has a hi plane also has its lo plane (FP16x3) or none has (single pass); a lo plane without
// its hi plane, or a mix of the two, is an argument error the entry point reports before any CUDA call.
struct PlanePairs {
  int hi = 0, lo = 0, orphan = 0;
  void add(const void* h, const void* l) {
    hi += h != nullptr;
    lo += h != nullptr && l != nullptr;
    orphan += h == nullptr && l != nullptr;
  }
  bool consistent() const { return orphan == 0 && (lo == 0 || lo == hi); }
  int planes() const { return hi > 0 && lo == 0 ? 1 : 2; }
};

// Single-pass FP16 (PLANES = 1): an activation is the hi plane alone, hi = f16(v), and there is no lo plane to read or
// write.  The range guard is the same.  PLANES = 2 is the FP16x3 code above, unchanged.
template <int PLANES>
__device__ __forceinline__ bool store16p(float v, __half* hi, __half* lo) {
  if constexpr (PLANES == 2) {
    return store16(v, hi, lo);
  } else {
    *hi = __float2half_rn(v);
    return f16_out_of_range(v);
  }
}

// Two consecutive values of a row into the planes at `off`; returns the range bit of either value.
template <int PLANES>
__device__ __forceinline__ bool store_pair16(float v0, float v1, __half* out_hi, __half* out_lo, size_t off) {
  if constexpr (PLANES == 2) {
    uint32_t hi, lo;
    const bool ovf = split_pack2(v0, v1, hi, lo);
    *reinterpret_cast<uint32_t*>(out_hi + off) = hi;
    *reinterpret_cast<uint32_t*>(out_lo + off) = lo;
    return ovf;
  } else {
    *reinterpret_cast<uint32_t*>(out_hi + off) = pack_half2(__float2half_rn(v0), __float2half_rn(v1));
    return f16_out_of_range(v0) | f16_out_of_range(v1);
  }
}

// The residual read of the epilogue: hi + lo (exact in fp32, 22 bits), or the hi plane alone.
template <int PLANES>
__device__ __forceinline__ float2 load_pair16(const __half* res_hi, const __half* res_lo, size_t off) {
  const float2 fh = __half22float2(__ldg(reinterpret_cast<const __half2*>(res_hi + off)));
  if constexpr (PLANES == 2) {
    const float2 fl = __half22float2(__ldg(reinterpret_cast<const __half2*>(res_lo + off)));
    return make_float2(fh.x + fl.x, fh.y + fl.y);
  } else {
    return fh;
  }
}

}  // namespace d3b
