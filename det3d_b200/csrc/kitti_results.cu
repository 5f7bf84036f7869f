// KITTI result rows on the device: predict's packed LiDAR-frame detections -> the reference's per-frame KITTI annos
// (clipped image box, alpha, camera-frame dimensions / location / rotation_y, score, label), with the reference's
// in-image filter applied and its order kept.
//
// Reference semantics, det3d/datasets/kitti/kitti.py:78-158 (KittiDataset.convert_detection_to_kitti_annos) with
// det3d/core/bbox/box_np_ops.py:267-297 (corners_nd), 358-391 (rotation_3d_in_axis), 453-474 (center_to_corner_box3d),
// 572-573 (limit_period), 900-906 (project_to_image), 917-922 (lidar_to_camera), 933-938 (box_lidar_to_camera).  Per
// valid detection, in predict's order (box = x, y, z, w, l, h, [..,] r as predict packs it):
//   float32   box[nd-1] = v - floor(v / fl(2pi) + 0.5) * fl(2pi); box[2] -= box[5] / 2     (each op rounded in f32)
//   float64   X, Y, Z = box[0..2];  loc_i = ((X*M[i][0] + Y*M[i][1]) + Z*M[i][2]) + M[i][3],  M = rect @ Trv2c
//             dims = (l, h, w) = (box[4], box[5], box[3]);  ry = box[6];  s, c = sin(ry), cos(ry)
//             corner k (k = 0..7, corners_nd's order, origin (0.5, 1, 0.5)): p = (l*ax_k, h*ay_k, w*az_k),
//               X_k = (p0*c + p2*s) + loc_x,  Y_k = p1 + loc_y,  Z_k = (p0*(-s) + p2*c) + loc_z
//             n_j = ((X_k*P[j][0] + Y_k*P[j][1]) + Z_k*P[j][2]) + 0*P[j][3]   (project_to_image appends ZEROS, so
//             P2's translation column never enters), u = n_0 / n_2, v = n_1 / n_2 (a negative depth is divided as is)
//             bbox = (min u, min v, max u, max v) over the 8 corners, NaN propagating as numpy's min / max
//   filter    dropped when bbox[0] > W or bbox[1] > H or bbox[2] < 0 or bbox[3] < 0 (a NaN fails every test: kept)
//   clip      bbox[2:] = minimum(bbox[2:], (W, H)), bbox[:2] = maximum(bbox[:2], 0), NaN propagating
//   alpha     -atan2f(-y, x) (float32 x, y), promoted, + ry
// Every float64 product, sum and quotient written here is __dmul_rn / __dadd_rn / __ddiv_rn and every float32 step
// __f*_rn, so nothing is contracted into an FMA; sin / cos / atan2 are the CUDA math library's.  The SASS's DFMA / FFMA
// come only from those and from the correctly rounded division sequences.
//
// One CTA per sample walks its D rows in chunks of kKrThreads and compacts the kept rows in order (compact_rows.cuh);
// rows past the sample's count are written as zeros.  No workspace.
#include "common.cuh"
#include "compact_rows.cuh"

namespace d3b {
namespace {

constexpr int kKrThreads = 256;
constexpr int kKrMaxBatch = 64;
constexpr int kKrCalibDoubles = 32;               // M [4][4], P2 rows 0..2 [3][4], H, W, 2 unused
constexpr int kKrCols = 14;

__device__ __forceinline__ bool is_nan(double a) { return a != a; }

// numpy's minimum / maximum: a NaN operand is the result (fmin / fmax would drop it)
__device__ __forceinline__ double np_min(double a, double b) { return is_nan(a) ? a : is_nan(b) ? b : (b < a ? b : a); }
__device__ __forceinline__ double np_max(double a, double b) { return is_nan(a) ? a : is_nan(b) ? b : (b > a ? b : a); }

__device__ __forceinline__ double dot3_zero(const double* Pj, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, Pj[0]), __dmul_rn(y, Pj[1])), __dmul_rn(z, Pj[2])),
                   __dmul_rn(0.0, Pj[3]));
}

// The conversion of one valid detection `d` (nd + 3 floats) under calibration `cal`; row = bbox 4, alpha, dims 3,
// location 3, rotation_y, score, label.  Returns whether the reference keeps it.
__device__ __forceinline__ bool kitti_row(const float* __restrict__ d, int nd, const double* cal, double* row) {
  const float two_pi = 6.28318530717958647692f;   // fl32(np.pi * 2)
  float box[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) box[j] = j < nd ? d[j] : 0.f;
  // limit_period on the last box column (kitti.py:117 indexes it as [:, -1]); for nd = 7 that is the yaw
  const float r = nd == 7 ? box[6] : box[8];
  const float r_wrapped = __fsub_rn(r, __fmul_rn(floorf(__fadd_rn(__fdiv_rn(r, two_pi), 0.5f)), two_pi));
  if (nd == 7) box[6] = r_wrapped; else box[8] = r_wrapped;
  box[2] = __fsub_rn(box[2], __fdiv_rn(box[5], 2.0f));

  const double X = box[0], Y = box[1], Z = box[2];
  double loc[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double* Mi = cal + 4 * i;
    loc[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, Mi[0]), __dmul_rn(Y, Mi[1])), __dmul_rn(Z, Mi[2])), Mi[3]);
  }
  const double l = box[4], h = box[5], w = box[3], ry = box[6];
  double s, c;
  sincos(ry, &s, &c);
  const double* P = cal + 16;
  double u0 = 0.0, v0 = 0.0, u1 = 0.0, v1 = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    // corners_nd's order x0y0z0, x0y0z1, x0y1z1, x0y1z0, x1y0z0, x1y0z1, x1y1z1, x1y1z0 minus (0.5, 1, 0.5)
    const double ax = k < 4 ? -0.5 : 0.5;
    const double ay = (k & 3) < 2 ? -1.0 : 0.0;
    const double az = ((k + 1) & 2) ? 0.5 : -0.5;
    const double p0 = __dmul_rn(l, ax), p1 = __dmul_rn(h, ay), p2 = __dmul_rn(w, az);
    const double cx = __dadd_rn(__dadd_rn(__dmul_rn(p0, c), __dmul_rn(p2, s)), loc[0]);
    const double cy = __dadd_rn(p1, loc[1]);
    const double cz = __dadd_rn(__dadd_rn(__dmul_rn(p0, -s), __dmul_rn(p2, c)), loc[2]);
    const double n2 = dot3_zero(P + 8, cx, cy, cz);
    const double u = __ddiv_rn(dot3_zero(P, cx, cy, cz), n2), v = __ddiv_rn(dot3_zero(P + 4, cx, cy, cz), n2);
    if (k == 0) {
      u0 = u1 = u; v0 = v1 = v;
    } else {
      u0 = np_min(u0, u); v0 = np_min(v0, v); u1 = np_max(u1, u); v1 = np_max(v1, v);
    }
  }
  const double H = cal[28], W = cal[29];
  const bool keep = !(u0 > W || v0 > H) && !(u1 < 0.0 || v1 < 0.0);
  row[0] = np_max(u0, 0.0); row[1] = np_max(v0, 0.0); row[2] = np_min(u1, W); row[3] = np_min(v1, H);
  // atan2 in f64 rounded once to f32: the f32 atan2 within half an f32 ulp (bar double rounding)
  const float a32 = (float)atan2(-(double)box[1], (double)box[0]);
  row[4] = __dadd_rn(-(double)a32, ry);
  row[5] = l; row[6] = h; row[7] = w;
  row[8] = loc[0]; row[9] = loc[1]; row[10] = loc[2];
  row[11] = ry;
  row[12] = d[nd];
  row[13] = d[nd + 1];
  return keep;
}

__global__ void __launch_bounds__(kKrThreads)
kitti_results_kernel(const float* __restrict__ det, const double* __restrict__ calib, int D, int nd,
                     double* __restrict__ results, int* __restrict__ counts) {
  __shared__ double cal[kKrCalibDoubles];
  __shared__ int warp_cnt[kKrThreads / 32];
  const int b = blockIdx.x;
  if (threadIdx.x < kKrCalibDoubles) cal[threadIdx.x] = calib[(size_t)b * kKrCalibDoubles + threadIdx.x];
  __syncthreads();
  const int stride = nd + 3;
  const float* __restrict__ det_b = det + (size_t)b * D * stride;
  const int count = compact_rows<kKrThreads, kKrCols>(D, results + (size_t)b * D * kKrCols, warp_cnt,
                                                      [&](int i, double* row) {
    const float* d = det_b + (size_t)i * stride;
    return d[nd + 2] > 0.5f && kitti_row(d, nd, cal, row);
  });
  if (threadIdx.x == 0) counts[b] = count;
}

}  // namespace
}  // namespace d3b

using namespace d3b;

extern "C" int d3b_kitti_results_dev(const float* detections, const double* calib, int32_t batch, int32_t max_det,
                                     int32_t nd, double* results, int32_t* counts, void* stream_) {
  static const char* name = "d3b_kitti_results_dev";
  D3B_REQUIRE(calib && counts, "%s: null argument", name);
  D3B_REQUIRE(batch >= 1 && batch <= kKrMaxBatch, "%s: batch %d outside [1, %d]", name, batch, kKrMaxBatch);
  D3B_REQUIRE(max_det >= 0 && max_det <= (1 << 20), "%s: max_det %d outside [0, 2^20]", name, max_det);
  if (nd != 7 && nd != 9) {
    set_error("%s: nd %d not built (7 or 9)", name, nd);
    return D3B_ERR_UNSUPPORTED;
  }
  D3B_REQUIRE(max_det == 0 || (detections && results), "%s: null buffer", name);
  kitti_results_kernel<<<batch, kKrThreads, 0, (cudaStream_t)stream_>>>(detections, calib, max_det, nd, results,
                                                                         counts);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}
