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

}  // namespace d3b
