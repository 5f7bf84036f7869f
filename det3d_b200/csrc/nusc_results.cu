// nuScenes result rows on the device: predict's packed LiDAR-frame detections -> the reference's submission boxes in the
// global frame (translation, size, orientation quaternion, velocity, score, label and the speed test that picks the
// attribute), with predict's order kept.
//
// Reference semantics, det3d/datasets/nuscenes/nusc_common.py:222-240 (_second_det_to_nusc_box), 243-265
// (_lidar_nusc_box_to_global) and det3d/datasets/nuscenes/nuscenes.py:219-259 (NuScenesDataset.evaluation's per-box
// loop), with pyquaternion's Quaternion(axis, radians), rotation_matrix and Hamilton product and the nuScenes devkit's
// Box.rotate / Box.translate.  Per valid detection (nd = 9: x, y, z, w, l, h, vx, vy, r), in predict's order:
//   float32   yaw' = fl32(-r) - fl32(pi/2)   (box3d[:, -1] = -box3d[:, -1] - np.pi / 2 on a float32 array)
//   float64   th = yaw' / 2;  qy = (cos th, 0 * sin th, 0 * sin th, sin th)          (_from_axis_angle, axis (0, 0, 1))
//             c1_i = ((Rc_i0*x + Rc_i1*y) + Rc_i2*z) + tc_i;  t_i = ((Rp_i0*c1_0 + Rp_i1*c1_1) + Rp_i2*c1_2) + tp_i
//             v1_i = (Rc_i0*vx + Rc_i1*vy) + Rc_i2*0;       vg_i = (Rp_i0*v1_0 + Rp_i1*v1_1) + Rp_i2*v1_2
//             q1 = qc (x) qy, rot = qp (x) q1, each component sum_k Q(a)_ik b_k in k order (a (x) b = Q(a) b, as
//             pyquaternion's __mul__ forms it); the reference's association is kept: Rp*Rc and qp (x) qc never form
//             moving = sqrt(vg_0^2 + vg_1^2) > 0.2, in float64 (fl32(0.2) is above 0.2 and counts as moving)
// Every float64 product and sum written here is __dmul_rn / __dadd_rn, so nothing is contracted into an FMA; sin / cos
// are the CUDA math library's and sqrt is correctly rounded.  Rc, Rp, qc and qp come from the host (pose_table), already
// normalised as pyquaternion normalises them.
//
// One CTA per sample compacts the valid rows in order (compact_rows.cuh); rows past the sample's count are written as
// zeros.  No workspace.
#include "common.cuh"
#include "compact_rows.cuh"

namespace d3b {
namespace {

constexpr int kNrThreads = 256;
constexpr int kNrMaxBatch = 64;
constexpr int kNrPoseDoubles = 32;                 // Rc [9], tc [3], Rp [9], tp [3], qc [4], qp [4]
constexpr int kNrCols = 15;
constexpr int kNrNd = 9;

__device__ __forceinline__ double dot3(const double* Ri, double a, double b, double c) {
  return __dadd_rn(__dadd_rn(__dmul_rn(Ri[0], a), __dmul_rn(Ri[1], b)), __dmul_rn(Ri[2], c));
}

// a (x) b, pyquaternion's _q_matrix(a) applied to b, each component summed in k order
__device__ __forceinline__ void hamilton(const double* a, const double* b, double* out) {
  const double Q[4][4] = {{a[0], -a[1], -a[2], -a[3]},
                          {a[1], a[0], -a[3], a[2]},
                          {a[2], a[3], a[0], -a[1]},
                          {a[3], -a[2], a[1], a[0]}};
#pragma unroll
  for (int i = 0; i < 4; ++i)
    out[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Q[i][0], b[0]), __dmul_rn(Q[i][1], b[1])),
                                 __dmul_rn(Q[i][2], b[2])), __dmul_rn(Q[i][3], b[3]));
}

// The conversion of one valid detection `d` (12 floats) under pose row `p`; row = translation 3, size 3 (w, l, h),
// rotation 4 (w, x, y, z), velocity 2, score, label, moving.
__device__ __forceinline__ void nusc_row(const float* __restrict__ d, const double* p, double* row) {
  const double *Rc = p, *tc = p + 9, *Rp = p + 12, *tp = p + 21, *qc = p + 24, *qp = p + 28;
  const float yaw = __fsub_rn(-d[8], 1.57079632679489661923f);      // fl32(pi / 2)
  double s, c;
  sincos(__dmul_rn((double)yaw, 0.5), &s, &c);
  const double qy[4] = {c, __dmul_rn(0.0, s), __dmul_rn(0.0, s), s};
  const double x = d[0], y = d[1], z = d[2], vx = d[6], vy = d[7];
  double c1[3], v1[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    c1[i] = __dadd_rn(dot3(Rc + 3 * i, x, y, z), tc[i]);
    v1[i] = dot3(Rc + 3 * i, vx, vy, 0.0);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) row[i] = __dadd_rn(dot3(Rp + 3 * i, c1[0], c1[1], c1[2]), tp[i]);
  row[3] = d[3]; row[4] = d[4]; row[5] = d[5];
  double q1[4];
  hamilton(qc, qy, q1);
  hamilton(qp, q1, row + 6);
  const double vg0 = dot3(Rp, v1[0], v1[1], v1[2]), vg1 = dot3(Rp + 3, v1[0], v1[1], v1[2]);
  row[10] = vg0; row[11] = vg1;
  row[12] = d[kNrNd];
  row[13] = d[kNrNd + 1];
  row[14] = __dsqrt_rn(__dadd_rn(__dmul_rn(vg0, vg0), __dmul_rn(vg1, vg1))) > 0.2 ? 1.0 : 0.0;
}

__global__ void __launch_bounds__(kNrThreads)
nusc_results_kernel(const float* __restrict__ det, const double* __restrict__ poses, int D,
                    double* __restrict__ results, int* __restrict__ counts) {
  __shared__ double pose[kNrPoseDoubles];
  __shared__ int warp_cnt[kNrThreads / 32];
  const int b = blockIdx.x;
  if (threadIdx.x < kNrPoseDoubles) pose[threadIdx.x] = poses[(size_t)b * kNrPoseDoubles + threadIdx.x];
  __syncthreads();
  constexpr int stride = kNrNd + 3;
  const float* __restrict__ det_b = det + (size_t)b * D * stride;
  const int count = compact_rows<kNrThreads, kNrCols>(D, results + (size_t)b * D * kNrCols, warp_cnt,
                                                      [&](int i, double* row) {
    const float* d = det_b + (size_t)i * stride;
    if (!(d[kNrNd + 2] > 0.5f)) return false;
    nusc_row(d, pose, row);
    return true;
  });
  if (threadIdx.x == 0) counts[b] = count;
}

}  // namespace
}  // namespace d3b

using namespace d3b;

extern "C" int d3b_nusc_results_dev(const float* detections, const double* poses, int32_t batch, int32_t max_det,
                                    int32_t nd, double* results, int32_t* counts, void* stream_) {
  static const char* name = "d3b_nusc_results_dev";
  D3B_REQUIRE(poses && counts, "%s: null argument", name);
  D3B_REQUIRE(batch >= 1 && batch <= kNrMaxBatch, "%s: batch %d outside [1, %d]", name, batch, kNrMaxBatch);
  D3B_REQUIRE(max_det >= 0 && max_det <= (1 << 20), "%s: max_det %d outside [0, 2^20]", name, max_det);
  if (nd != kNrNd) {
    set_error("%s: nd %d not built (9: x, y, z, w, l, h, vx, vy, r)", name, nd);
    return D3B_ERR_UNSUPPORTED;
  }
  D3B_REQUIRE(max_det == 0 || (detections && results), "%s: null buffer", name);
  nusc_results_kernel<<<batch, kNrThreads, 0, (cudaStream_t)stream_>>>(detections, poses, max_det, results, counts);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}
