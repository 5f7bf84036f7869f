// Rotated-box BEV IoU and greedy NMS, fully device-side.
//
// Two semantics are served (SURVEY App. A.5):
//   D3B_BOX_XYXYR  boxes [x1,y1,x2,y2,ry]; suppress when IoU >  thr.
//       Follows det3d/ops/iou3d/src/iou3d_kernel.cu:108-221 (box_overlap /
//       iou_bev) and the host sweep of det3d/ops/iou3d/src/iou3d.cpp:103-116.
//       The pair arithmetic below keeps the reference's fp32 expression tree
//       (same association, same libdevice calls, same EPS/MARGIN constants)
//       so nvcc makes the same FMA-contraction decisions and the keep mask is
//       bit-identical to the reference kernel's.
//   D3B_BOX_XYWLR  boxes [cx,cy,w,l,r]; suppress when IoU >= thr and the
//       axis-aligned hulls overlap.  Follows det3d/ops/nms/nms_cpu.py:34-45 and
//       det3d/ops/nms/nms_cpu.h:73-169 (boost polygon intersection / union):
//       corners in fp32 exactly as box_np_ops.py:419-497 builds them, polygon
//       clipping in fp64.
//
// Design: (1) the N x N/64 suppression bitmask is produced for the upper
// triangle only (the sweep never reads the rest) by one thread per row box,
// with an exact-safe disjoint-circle test in front of the ~2k-instruction
// polygon routine; (2) the greedy sweep runs on the device (one CTA, `remv`
// in shared memory, early exit at max_keep) -- the reference copies the whole
// mask to the host (1.25 GB at N=100k) and sweeps there.
#include "common.cuh"

namespace d3b {

constexpr int kNmsBlock = 64;  // boxes per mask word

// ============================================================================
// XYXYR pair arithmetic (iou3d semantic)
// ============================================================================
struct P2 {
  float x, y;
};

constexpr float kEps = 1e-8f;

__device__ __forceinline__ float cross2(const P2& a, const P2& b) { return a.x * b.y - a.y * b.x; }

__device__ __forceinline__ float cross3(const P2& u, const P2& v, const P2& o) {
  return (u.x - o.x) * (v.y - o.y) - (v.x - o.x) * (u.y - o.y);
}

__device__ __forceinline__ int seg_hulls_touch(const P2& p1, const P2& p2, const P2& q1, const P2& q2) {
  return fminf(p1.x, p2.x) <= fmaxf(q1.x, q2.x) && fminf(q1.x, q2.x) <= fmaxf(p1.x, p2.x) &&
         fminf(p1.y, p2.y) <= fmaxf(q1.y, q2.y) && fminf(q1.y, q2.y) <= fmaxf(p1.y, p2.y);
}

// iou3d_kernel.cu:50-65
__device__ __forceinline__ int point_in_box(const float* box, const P2& p) {
  const float margin = 1e-5f;
  const float cx = (box[0] + box[2]) / 2;
  const float cy = (box[1] + box[3]) / 2;
  const float c = cosf(-box[4]), s = sinf(-box[4]);
  const float rx = (p.x - cx) * c + (p.y - cy) * s + cx;
  const float ry = -(p.x - cx) * s + (p.y - cy) * c + cy;
  return (rx > box[0] - margin && rx < box[2] + margin && ry > box[1] - margin && ry < box[3] + margin);
}

// iou3d_kernel.cu:67-96
__device__ __forceinline__ int seg_intersection(const P2& p1, const P2& p0, const P2& q1, const P2& q0,
                                                P2& out) {
  if (seg_hulls_touch(p0, p1, q0, q1) == 0) return 0;
  const float s1 = cross3(q0, p1, p0);
  const float s2 = cross3(p1, q1, p0);
  const float s3 = cross3(p0, q1, q0);
  const float s4 = cross3(q1, p1, q0);
  if (!(s1 * s2 > 0 && s3 * s4 > 0)) return 0;
  const float s5 = cross3(q1, p1, p0);
  if (fabsf(s5 - s1) > kEps) {
    out.x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
    out.y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
  } else {
    const float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
    const float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
    const float D = a0 * b1 - a1 * b0;
    out.x = (b0 * c1 - b1 * c0) / D;
    out.y = (a1 * c0 - a0 * c1) / D;
  }
  return 1;
}

__device__ __forceinline__ void spin_about(const P2& ctr, const float c, const float s, P2& p) {
  const float nx = (p.x - ctr.x) * c + (p.y - ctr.y) * s + ctr.x;
  const float ny = -(p.x - ctr.x) * s + (p.y - ctr.y) * c + ctr.y;
  p.x = nx;
  p.y = ny;
}

__device__ __forceinline__ int angle_after(const P2& a, const P2& b, const P2& ctr) {
  return atan2f(a.y - ctr.y, a.x - ctr.x) > atan2f(b.y - ctr.y, b.x - ctr.x);
}

// iou3d_kernel.cu:108-212
__device__ __forceinline__ float overlap_xyxyr(const float* box_a, const float* box_b) {
  const float ax1 = box_a[0], ay1 = box_a[1], ax2 = box_a[2], ay2 = box_a[3], aang = box_a[4];
  const float bx1 = box_b[0], by1 = box_b[1], bx2 = box_b[2], by2 = box_b[3], bang = box_b[4];
  P2 ctr_a, ctr_b;
  ctr_a.x = (ax1 + ax2) / 2; ctr_a.y = (ay1 + ay2) / 2;
  ctr_b.x = (bx1 + bx2) / 2; ctr_b.y = (by1 + by2) / 2;

  P2 ca[5], cb[5];
  ca[0].x = ax1; ca[0].y = ay1; ca[1].x = ax2; ca[1].y = ay1;
  ca[2].x = ax2; ca[2].y = ay2; ca[3].x = ax1; ca[3].y = ay2;
  cb[0].x = bx1; cb[0].y = by1; cb[1].x = bx2; cb[1].y = by1;
  cb[2].x = bx2; cb[2].y = by2; cb[3].x = bx1; cb[3].y = by2;

  const float a_cos = cosf(aang), a_sin = sinf(aang);
  const float b_cos = cosf(bang), b_sin = sinf(bang);
  for (int k = 0; k < 4; k++) {
    spin_about(ctr_a, a_cos, a_sin, ca[k]);
    spin_about(ctr_b, b_cos, b_sin, cb[k]);
  }
  ca[4] = ca[0];
  cb[4] = cb[0];

  P2 pts[16];
  P2 centre;
  int cnt = 0, hit = 0;
  centre.x = 0; centre.y = 0;
  for (int i = 0; i < 4; i++) {
    for (int j = 0; j < 4; j++) {
      hit = seg_intersection(ca[i + 1], ca[i], cb[j + 1], cb[j], pts[cnt]);
      if (hit) {
        centre.x = centre.x + pts[cnt].x;
        centre.y = centre.y + pts[cnt].y;
        cnt++;
      }
    }
  }
  for (int k = 0; k < 4; k++) {
    if (point_in_box(box_a, cb[k])) {
      centre.x = centre.x + cb[k].x;
      centre.y = centre.y + cb[k].y;
      pts[cnt] = cb[k];
      cnt++;
    }
    if (point_in_box(box_b, ca[k])) {
      centre.x = centre.x + ca[k].x;
      centre.y = centre.y + ca[k].y;
      pts[cnt] = ca[k];
      cnt++;
    }
  }
  centre.x /= cnt;
  centre.y /= cnt;

  P2 tmp;
  for (int j = 0; j < cnt - 1; j++) {
    for (int i = 0; i < cnt - j - 1; i++) {
      if (angle_after(pts[i], pts[i + 1], centre)) {
        tmp = pts[i];
        pts[i] = pts[i + 1];
        pts[i + 1] = tmp;
      }
    }
  }
  float area = 0;
  for (int k = 0; k < cnt - 1; k++) {
    P2 u, v;
    u.x = pts[k].x - pts[0].x; u.y = pts[k].y - pts[0].y;
    v.x = pts[k + 1].x - pts[0].x; v.y = pts[k + 1].y - pts[0].y;
    area += cross2(u, v);
  }
  return fabsf(area) / 2.0;
}

// iou3d_kernel.cu:214-221
__device__ __forceinline__ float iou_xyxyr(const float* box_a, const float* box_b) {
  const float sa = (box_a[2] - box_a[0]) * (box_a[3] - box_a[1]);
  const float sb = (box_b[2] - box_b[0]) * (box_b[3] - box_b[1]);
  const float so = overlap_xyxyr(box_a, box_b);
  return so / fmaxf(sa + sb - so, kEps);
}

// iou3d_kernel.cu:295-303
__device__ __forceinline__ float iou_axis_aligned(const float* a, const float* b) {
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const float width = fmaxf(right - left, 0.f), height = fmaxf(bottom - top, 0.f);
  const float inter = width * height;
  const float sa = (a[2] - a[0]) * (a[3] - a[1]);
  const float sb = (b[2] - b[0]) * (b[3] - b[1]);
  return inter / fmaxf(sa + sb - inter, kEps);
}

// numba nms_gpu.py:22-33 (`iou_device`, the IoU behind box_torch_ops.nms): +1 "pixel" extents.  Under numba's
// typing the float32 differences are promoted to float64 by the integer literal, so everything after the
// fp32 subtraction is double arithmetic; the result is compared against the float32 threshold in double.
__device__ __forceinline__ double iou_pixel(const float* a, const float* b) {
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const double width = fmax((double)__fsub_rn(right, left) + 1.0, 0.0);
  const double height = fmax((double)__fsub_rn(bottom, top) + 1.0, 0.0);
  const double inter = width * height;
  const double sa = ((double)__fsub_rn(a[2], a[0]) + 1.0) * ((double)__fsub_rn(a[3], a[1]) + 1.0);
  const double sb = ((double)__fsub_rn(b[2], b[0]) + 1.0) * ((double)__fsub_rn(b[3], b[1]) + 1.0);
  return inter / (sa + sb - inter);
}

// Exact-safe rejection: when the circumscribed circles (about the rectangle
// centres, the rotation pivots) are separated by more than a 1e-3 cushion the
// reference routine finds no intersection point and no contained corner
// (MARGIN 1e-5), cnt = 0, area = 0, IoU = +0.  Any NaN/inf makes the test
// false and the pair takes the full path.
struct Disc {
  float cx, cy, r;
};
__device__ __forceinline__ Disc disc_of_xyxyr(const float* b) {
  Disc d;
  d.cx = 0.5f * (b[0] + b[2]);
  d.cy = 0.5f * (b[1] + b[3]);
  const float w = b[2] - b[0], h = b[3] - b[1];
  d.r = 0.5f * sqrtf(w * w + h * h) * 1.0001f + 1e-3f;
  return d;
}
__device__ __forceinline__ bool surely_disjoint(const Disc& a, const Disc& b) {
  const float dx = a.cx - b.cx, dy = a.cy - b.cy, rr = a.r + b.r;
  return dx * dx + dy * dy > rr * rr * 1.0001f;
}

// ============================================================================
// XYWLR pair arithmetic (rotate_nms_cc semantic), fp64 polygon clipping
// ============================================================================
struct Quad {
  float x[4], y[4];           // corners, fp32 as numpy builds them
  float minx, miny, maxx, maxy;
};

// box_np_ops.py:267-297 (corners_nd, clockwise from the minimum corner),
// :419-432 (rotation_2d: x' = x cos + y sin, y' = -x sin + y cos), :477-497.
__device__ __forceinline__ Quad quad_of_xywlr(const float* b) {
  Quad q;
  const float cx = b[0], cy = b[1], w = b[2], l = b[3], r = b[4];
  const float s = sinf(r), c = cosf(r);
  const float ox[4] = {-0.5f, -0.5f, 0.5f, 0.5f};
  const float oy[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float px = __fmul_rn(w, ox[k]), py = __fmul_rn(l, oy[k]);
    q.x[k] = __fadd_rn(__fadd_rn(__fmul_rn(px, c), __fmul_rn(py, s)), cx);
    q.y[k] = __fadd_rn(__fadd_rn(__fmul_rn(-px, s), __fmul_rn(py, c)), cy);
  }
  q.minx = fminf(fminf(q.x[0], q.x[1]), fminf(q.x[2], q.x[3]));
  q.maxx = fmaxf(fmaxf(q.x[0], q.x[1]), fmaxf(q.x[2], q.x[3]));
  q.miny = fminf(fminf(q.y[0], q.y[1]), fminf(q.y[2], q.y[3]));
  q.maxy = fmaxf(fmaxf(q.y[0], q.y[1]), fmaxf(q.y[2], q.y[3]));
  return q;
}

// box_np_ops.py:955-994 with eps = 0 (nms_cpu.py:43), fp32.
__device__ __forceinline__ float standup_iou(const Quad& a, const Quad& b) {
  const float iw = __fsub_rn(fminf(a.maxx, b.maxx), fmaxf(a.minx, b.minx));
  if (!(iw > 0)) return 0.0f;
  const float ih = __fsub_rn(fminf(a.maxy, b.maxy), fmaxf(a.miny, b.miny));
  if (!(ih > 0)) return 0.0f;
  const float area_b = __fmul_rn(__fsub_rn(b.maxx, b.minx), __fsub_rn(b.maxy, b.miny));
  const float area_a = __fmul_rn(__fsub_rn(a.maxx, a.minx), __fsub_rn(a.maxy, a.miny));
  const float inter = __fmul_rn(iw, ih);
  const float ua = __fsub_rn(__fadd_rn(area_a, area_b), inter);
  return __fdiv_rn(inter, ua);
}

// Vertex capacity of the clipper.  In exact arithmetic clipping a convex polygon by a half-plane adds at most one vertex,
// so the four steps never exceed 8.  In floating point the near-duplicate pairs NMS sees all the time (the same box one
// ulp or 1e-9 rad apart) make the sign tests of a clip step disagree with the geometry: the rounded polygon is not convex
// any more, and a clip step can meet more than two sign changes (more than 8 vertices).  The bound that holds for
// any sign pattern: one step keeps the k vertices with d >= 0 and adds one per sign change of the cyclic sequence of n
// vertices, and there are at most 2 * min(k, n - k) of those, so m <= k + 2 min(k, n - k) <= floor(3n / 2).  From 4
// corners: 6, 9, 13, 19.
constexpr int kClipMaxVertices = 19;

// Convex quad ∩ convex quad by Sutherland-Hodgman in fp64; returns area.
__device__ double quad_intersection_area(const Quad& A, const Quad& B) {
  double px[kClipMaxVertices], py[kClipMaxVertices], qx[kClipMaxVertices], qy[kClipMaxVertices];
  int n = 4;
  for (int k = 0; k < 4; ++k) { px[k] = A.x[k]; py[k] = A.y[k]; }
  // orientation of the clip polygon
  double area2 = 0.0;
  for (int k = 0; k < 4; ++k) {
    const int k1 = (k + 1) & 3;
    area2 += (double)B.x[k] * B.y[k1] - (double)B.x[k1] * B.y[k];
  }
  const double sgn = area2 >= 0.0 ? 1.0 : -1.0;
  for (int e = 0; e < 4 && n > 0; ++e) {
    const int e1 = (e + 1) & 3;
    const double ex = (double)B.x[e1] - B.x[e], ey = (double)B.y[e1] - B.y[e];
    int m = 0;
    for (int k = 0; k < n; ++k) {
      const int k1 = (k + 1 == n) ? 0 : k + 1;
      const double d0 = sgn * (ex * (py[k] - B.y[e]) - ey * (px[k] - B.x[e]));
      const double d1 = sgn * (ex * (py[k1] - B.y[e]) - ey * (px[k1] - B.x[e]));
      if (d0 >= 0.0) { qx[m] = px[k]; qy[m] = py[k]; ++m; }
      if ((d0 >= 0.0) != (d1 >= 0.0)) {
        const double t = d0 / (d0 - d1);
        qx[m] = px[k] + t * (px[k1] - px[k]);
        qy[m] = py[k] + t * (py[k1] - py[k]);
        ++m;
      }
    }
    n = m;
    for (int k = 0; k < n; ++k) { px[k] = qx[k]; py[k] = qy[k]; }
  }
  if (n < 3) return 0.0;
  double a = 0.0;
  for (int k = 0; k < n; ++k) {
    const int k1 = (k + 1 == n) ? 0 : k + 1;
    a += px[k] * py[k1] - px[k1] * py[k];
  }
  return fabs(a) * 0.5;
}

__device__ __forceinline__ double quad_area(const Quad& q) {
  double a = 0.0;
  for (int k = 0; k < 4; ++k) {
    const int k1 = (k + 1) & 3;
    a += (double)q.x[k] * q.y[k1] - (double)q.x[k1] * q.y[k];
  }
  return fabs(a) * 0.5;
}

// nms_cpu.h:103-158: skip unless hulls overlap; overlap = inter / union; suppress when >= thresh.
// The rotate_nms_cc IoU of a pair whose hulls overlap (standup_iou > 0; the caller applies that gate).  NaN when the
// pair is skipped (empty intersection -- boost's empty output -- or empty union): no threshold suppresses it, where an
// IoU of 0 would be suppressed at threshold 0.  The NMS mask and the mode-2 IoU matrix both call this.
__device__ __forceinline__ float clip_iou_xywlr(const Quad& a, const Quad& b) {
  const double inter = quad_intersection_area(a, b);
  if (!(inter > 0.0)) return __int_as_float(0x7fffffff);
  const double uni = quad_area(a) + quad_area(b) - inter;
  if (!(uni > 0.0)) return __int_as_float(0x7fffffff);
  return (float)(inter / uni);
}


// ============================================================================
// RRPN rotated IoU (numba rotate_iou_gpu / rotate_nms_gpu, det3d/ops/nms/nms_gpu.py:180-470).
// Boxes are [cx, cy, w, l, r].  Types follow numba's typing of the reference source: float32
// arithmetic throughout, except where an integer / float literal promotes to float64
// (triangle areas "/ 2.0", the area accumulator, "center /= n", the final ratio).
// ============================================================================
__device__ __forceinline__ void rrpn_corners(const float* rb, float* c) {                  // :368-390
  const float a_cos = cosf(rb[4]), a_sin = sinf(rb[4]);
  const float hx = (float)((double)rb[2] / 2.0), hy = (float)((double)rb[3] / 2.0);
  const float cx[4] = {-hx, -hx, hx, hx}, cy[4] = {-hy, hy, hy, -hy};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    c[2 * i] = a_cos * cx[i] + a_sin * cy[i] + rb[0];
    c[2 * i + 1] = -a_sin * cx[i] + a_cos * cy[i] + rb[1];
  }
}

__device__ __forceinline__ bool rrpn_point_in_quad(float px, float py, const float* c) {    // :325-341
  const float ab0 = c[2] - c[0], ab1 = c[3] - c[1];
  const float ad0 = c[6] - c[0], ad1 = c[7] - c[1];
  const float ap0 = px - c[0], ap1 = py - c[1];
  const float abab = ab0 * ab0 + ab1 * ab1, abap = ab0 * ap0 + ab1 * ap1;
  const float adad = ad0 * ad0 + ad1 * ad1, adap = ad0 * ap0 + ad1 * ap1;
  return abab >= abap && abap >= 0.f && adad >= adap && adap >= 0.f;
}

__device__ __forceinline__ bool rrpn_segment_intersection(const float* p1, const float* p2, int i, int j,
                                                          float* out) {                    // :239-281
  const float A0 = p1[2 * i], A1 = p1[2 * i + 1];
  const float B0 = p1[2 * ((i + 1) & 3)], B1 = p1[2 * ((i + 1) & 3) + 1];
  const float C0 = p2[2 * j], C1 = p2[2 * j + 1];
  const float D0 = p2[2 * ((j + 1) & 3)], D1 = p2[2 * ((j + 1) & 3) + 1];
  const float BA0 = B0 - A0, BA1 = B1 - A1, DA0 = D0 - A0, CA0 = C0 - A0, DA1 = D1 - A1, CA1 = C1 - A1;
  const bool acd = DA1 * CA0 > CA1 * DA0;
  const bool bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0);
  if (acd != bcd) {
    const bool abc = CA1 * BA0 > BA1 * CA0;
    const bool abd = DA1 * BA0 > BA1 * DA0;
    if (abc != abd) {
      const float DC0 = D0 - C0, DC1 = D1 - C1;
      const float ABBA = A0 * B1 - B0 * A1, CDDC = C0 * D1 - D0 * C1;
      const float DH = BA1 * DC0 - BA0 * DC1;
      const float Dx = ABBA * DC0 - BA0 * CDDC, Dy = ABBA * DC1 - BA1 * CDDC;
      out[0] = Dx / DH;
      out[1] = Dy / DH;
      return true;
    }
  }
  return false;
}

// intersection area of two rotated rectangles (`inter`, :393-408)
__device__ double rrpn_inter(const float* rb1, const float* rb2) {
  float c1[8], c2[8], pts[16];
  rrpn_corners(rb1, c1);
  rrpn_corners(rb2, c2);
  int n = 0;                                                                                 // :344-365
  // the reference writes into a 16-float buffer unchecked; two rectangles yield at most 8 points, the
  // guard only matters for non-finite input
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (n < 8 && rrpn_point_in_quad(c1[2 * i], c1[2 * i + 1], c2)) { pts[2 * n] = c1[2 * i]; pts[2 * n + 1] = c1[2 * i + 1]; ++n; }
    if (n < 8 && rrpn_point_in_quad(c2[2 * i], c2[2 * i + 1], c1)) { pts[2 * n] = c2[2 * i]; pts[2 * n + 1] = c2[2 * i + 1]; ++n; }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float t[2];
      if (n < 8 && rrpn_segment_intersection(c1, c2, i, j, t)) { pts[2 * n] = t[0]; pts[2 * n + 1] = t[1]; ++n; }
    }
  if (n > 0) {                                                                               // :199-236
    float cen0 = 0.f, cen1 = 0.f;
    for (int i = 0; i < n; ++i) { cen0 += pts[2 * i]; cen1 += pts[2 * i + 1]; }
    cen0 = (float)((double)cen0 / (double)n);
    cen1 = (float)((double)cen1 / (double)n);
    float vs[8];
    for (int i = 0; i < n; ++i) {
      float v0 = pts[2 * i] - cen0, v1 = pts[2 * i + 1] - cen1;
      const float d = sqrtf(v0 * v0 + v1 * v1);
      v0 = v0 / d;
      v1 = v1 / d;
      if (v1 < 0.f) v0 = (float)(-2.0 - (double)v0);
      vs[i] = v0;
    }
    for (int i = 1; i < n; ++i) {
      if (vs[i - 1] > vs[i]) {
        const float temp = vs[i], tx = pts[2 * i], ty = pts[2 * i + 1];
        int j = i;
        while (j > 0 && vs[j - 1] > temp) {
          vs[j] = vs[j - 1];
          pts[2 * j] = pts[2 * j - 2];
          pts[2 * j + 1] = pts[2 * j - 1];
          --j;
        }
        vs[j] = temp;
        pts[2 * j] = tx;
        pts[2 * j + 1] = ty;
      }
    }
  }
  double area = 0.0;                                                                         // :185-196
  for (int i = 0; i < n - 2; ++i) {
    const float a0 = pts[0], a1 = pts[1], b0 = pts[2 * i + 2], b1 = pts[2 * i + 3], q0 = pts[2 * i + 4], q1 = pts[2 * i + 5];
    area += fabs((double)((a0 - q0) * (b1 - q1) - (a1 - q1) * (b0 - q0)) / 2.0);
  }
  return area;
}

// devRotateIoUEval (:585-597): criterion -1 IoU, 0 inter/area1, 1 inter/area2, else the intersection area
__device__ __forceinline__ double rrpn_iou(const float* rb1, const float* rb2, int criterion) {
  const float area1 = rb1[2] * rb1[3], area2 = rb2[2] * rb2[3];
  const double ai = rrpn_inter(rb1, rb2);
  if (criterion == -1) return ai / ((double)(area1 + area2) - ai);
  if (criterion == 0) return ai / (double)area1;
  if (criterion == 1) return ai / (double)area2;
  return ai;
}

// rotate_iou_kernel(_eval) (:499-538,600-640): out[n, k] = IoU(query[k], boxes[n])
__global__ void __launch_bounds__(256)
rrpn_matrix_kernel(int n, const float* __restrict__ boxes, int k, const float* __restrict__ query, int criterion,
                   float* __restrict__ out) {
  const int a = blockIdx.y * 16 + threadIdx.y;
  const int b = blockIdx.x * 16 + threadIdx.x;
  if (a >= n || b >= k) return;
  out[(size_t)a * k + b] = (float)rrpn_iou(query + (size_t)b * 5, boxes + (size_t)a * 5, criterion);
}

// ============================================================================
// kernels
// ============================================================================
// Pairwise matrix, launch shape of the reference (iou3d_kernel.cu:223-248,354-371).
template <int MODE>
__global__ void __launch_bounds__(256)
pair_matrix_kernel(int na, const float* __restrict__ boxes_a, int nb, const float* __restrict__ boxes_b,
                   float* __restrict__ out) {
  const int a = blockIdx.y * 16 + threadIdx.y;
  const int b = blockIdx.x * 16 + threadIdx.x;
  if (a >= na || b >= nb) return;
  const float* pa = boxes_a + (size_t)a * 5;
  const float* pb = boxes_b + (size_t)b * 5;
  if constexpr (MODE == 2) {
    // rotate_nms_cc overlap: 0 for a pair the hull gate or the polygon test skips
    const Quad qa = quad_of_xywlr(pa), qb = quad_of_xywlr(pb);
    float v = 0.0f;
    if (standup_iou(qa, qb) > 0.0f) {
      v = clip_iou_xywlr(qa, qb);
      if (v != v) v = 0.0f;
    }
    out[(size_t)a * nb + b] = v;
  } else {
    out[(size_t)a * nb + b] = MODE == 0 ? iou_xyxyr(pa, pb) : overlap_xyxyr(pa, pb);
  }
}

// Suppression bitmask, upper triangle only.  A work item is (64-box row block, 64-box column
// block, 16-row slice) with col >= row; the CTA is 64 (column) x 4 threads, every thread tests 4
// pairs and a warp ballot assembles 32 mask bits at a time -- 16x more threads in flight per mask
// word than one-thread-per-row, which is what the ~2k-instruction polygon routine needs at the
// real operating point (N = 1000: 2176 CTAs instead of 136).
constexpr int kNmsRowsPerCta = 16;
constexpr int kNmsSlices = kNmsBlock / kNmsRowsPerCta;
constexpr int kNmsPairQueue = 2048;     // queued (row, column) pairs of the iou3d routine; one item adds at most 1024

template <int FMT>  // 0 xyxyr rotated, 1 xywlr rotated, 2 axis-aligned (xyxyr boxes, angle ignored), 3 axis-aligned "+1"
__global__ void __launch_bounds__(256)
nms_mask_kernel(const float* __restrict__ boxes, int n_cap, const int* __restrict__ n_dev, float thresh,
                int col_blocks, unsigned long long* __restrict__ mask, long long box_stride, long long mask_stride) {
  // blockIdx.y = box set of the batch (the detector runs one NMS per sample: all of them in one launch)
  boxes += (size_t)blockIdx.y * box_stride;
  mask += (size_t)blockIdx.y * mask_stride;
  if (n_dev) n_dev += blockIdx.y;
  const int n = n_dev ? min(*n_dev, n_cap) : n_cap;
  const int nb = (n + kNmsBlock - 1) / kNmsBlock;
  const long long tri = (long long)nb * (nb + 1) / 2;
  const long long items = tri * kNmsSlices;
  __shared__ float scol[kNmsBlock * 5];
  __shared__ float srow[kNmsRowsPerCta * 5];
  __shared__ Disc dcol[FMT == 0 ? kNmsBlock : 1];
  __shared__ Quad qcol[FMT == 1 ? kNmsBlock : 1];
  __shared__ Quad qrow[FMT == 1 ? kNmsRowsPerCta : 1];
  __shared__ unsigned short s_list[FMT == 1 ? kNmsRowsPerCta * kNmsBlock : 1];
  __shared__ unsigned int s_bits[2 * kNmsRowsPerCta];
  __shared__ int s_count;
  __shared__ int2 s_pairs[FMT == 0 ? kNmsPairQueue : 1];     // (row box, column box) pairs waiting for the full IoU
  __shared__ int s_npairs;
  if (threadIdx.x == 0) s_npairs = 0;
  if (threadIdx.x < 2 * kNmsRowsPerCta) s_bits[threadIdx.x] = 0u;
  if (threadIdx.x == 0) s_count = 0;
  const int tx = threadIdx.x & 63;        // column inside the block
  const int ty = threadIdx.x >> 6;        // 0..3
  unsigned int* mask32 = reinterpret_cast<unsigned int*>(mask);
  auto flush_pairs = [&]() {              // CTA-uniform: evaluate the queued iou3d pairs, 256 at a time
    const int n_pairs = s_npairs;
    for (int e = threadIdx.x; e < n_pairs; e += blockDim.x) {
      const int2 pr = s_pairs[e];
      if (iou_xyxyr(boxes + (size_t)pr.x * 5, boxes + (size_t)pr.y * 5) > thresh)
        atomicOr(&mask32[((size_t)pr.x * col_blocks + (pr.y >> 6)) * 2 + ((pr.y >> 5) & 1)], 1u << (pr.y & 31));
    }
    __syncthreads();
    if (threadIdx.x == 0) s_npairs = 0;
    __syncthreads();
  };
  for (long long item = blockIdx.x; item < items; item += gridDim.x) {
    const long long bid = item / kNmsSlices;
    const int slice = (int)(item - bid * kNmsSlices);
    // linear id over the nb x nb upper triangle -> (row, col): row r owns (nb - r) blocks
    int row = (int)(((2.0 * nb + 1.0) - sqrt((2.0 * nb + 1.0) * (2.0 * nb + 1.0) - 8.0 * (double)bid)) * 0.5);
    if (row < 0) row = 0;
    while ((long long)row * nb - (long long)row * (row - 1) / 2 > bid) --row;
    while ((long long)(row + 1) * nb - (long long)(row + 1) * row / 2 <= bid) ++row;
    const int col = row + (int)(bid - ((long long)row * nb - (long long)row * (row - 1) / 2));
    const int row_first = row * kNmsBlock + slice * kNmsRowsPerCta;
    const int col_size = min(n - col * kNmsBlock, kNmsBlock);
    __syncthreads();
    if (row_first >= n) continue;          // uniform for the CTA
    if ((int)threadIdx.x < col_size) {
      const float* src = boxes + (size_t)(kNmsBlock * col + threadIdx.x) * 5;
#pragma unroll
      for (int k = 0; k < 5; ++k) scol[threadIdx.x * 5 + k] = src[k];
      if (FMT == 0) dcol[threadIdx.x] = disc_of_xyxyr(src);
      if (FMT == 1) qcol[threadIdx.x] = quad_of_xywlr(src);
    }
    if ((int)threadIdx.x >= 64 && (int)threadIdx.x < 64 + kNmsRowsPerCta && row_first + (int)threadIdx.x - 64 < n) {
      const int r = threadIdx.x - 64;
      const float* src = boxes + (size_t)(row_first + r) * 5;
#pragma unroll
      for (int k = 0; k < 5; ++k) srow[r * 5 + k] = src[k];
      if (FMT == 1) qrow[r] = quad_of_xywlr(src);
    }
    __syncthreads();
    if constexpr (FMT == 0) {
      // iou3d pairs: the exact-safe disjoint-circle test rejects > 99 % of the pairs of a large box set; the few
      // that need the ~2k-instruction polygon routine are queued ACROSS work items and evaluated 256 at a time, so
      // the expensive part runs with full warps (100k boxes: 205 ms with one or two live lanes per warp).  This CTA
      // owns the mask words of its items: it zeroes them here and ORs the hits in after the evaluation.
      if (threadIdx.x < 2 * kNmsRowsPerCta && row_first + (int)(threadIdx.x >> 1) < n)
        mask32[((size_t)(row_first + (threadIdx.x >> 1)) * col_blocks + col) * 2 + (threadIdx.x & 1)] = 0u;
      for (int rr = ty; rr < kNmsRowsPerCta; rr += 4) {
        const int cur = row_first + rr;
        const bool active = cur < n && tx < col_size && (row != col || tx > slice * kNmsRowsPerCta + rr);
        if (active && !(thresh >= 0.0f && surely_disjoint(disc_of_xyxyr(srow + rr * 5), dcol[tx])))
          s_pairs[atomicAdd(&s_npairs, 1)] = make_int2(cur, col * kNmsBlock + tx);
      }
      __syncthreads();
      if (s_npairs > kNmsPairQueue - kNmsRowsPerCta * kNmsBlock) flush_pairs();   // no room for another item
      continue;
    }
    if constexpr (FMT == 1) {
      // rotate_nms_cc pairs: the hull gate (fp32, a few instructions) passes only a few percent of the pairs, the
      // fp64 polygon clip behind it costs thousands of instructions.  Testing the gate for all 16 x 64 pairs first and
      // compacting the survivors keeps every lane busy in the expensive part instead of one or two lanes per warp.
      for (int rr = ty; rr < kNmsRowsPerCta; rr += 4) {
        const int cur = row_first + rr;
        const bool active = cur < n && tx < col_size && (row != col || tx > slice * kNmsRowsPerCta + rr);
        if (active && standup_iou(qrow[rr], qcol[tx]) > 0.0f) s_list[atomicAdd(&s_count, 1)] = (unsigned short)(rr * 64 + tx);
      }
      __syncthreads();
      const int n_pairs = s_count;
      for (int e = threadIdx.x; e < n_pairs; e += blockDim.x) {
        const int rr = s_list[e] >> 6, cc = s_list[e] & 63;
        if (clip_iou_xywlr(qrow[rr], qcol[cc]) >= thresh) atomicOr(&s_bits[rr * 2 + (cc >> 5)], 1u << (cc & 31));
      }
      __syncthreads();
      if (threadIdx.x < 2 * kNmsRowsPerCta) {
        const int rr = threadIdx.x >> 1;
        if (row_first + rr < n) mask32[((size_t)(row_first + rr) * col_blocks + col) * 2 + (threadIdx.x & 1)] = s_bits[threadIdx.x];
        s_bits[threadIdx.x] = 0u;
      }
      if (threadIdx.x == 0) s_count = 0;
      continue;                            // the loop-top __syncthreads orders the reset before the next item
    }
    if constexpr (FMT >= 2) {             // axis-aligned and RRPN routines: cheap enough for the ballot layout
#pragma unroll 1
    for (int rr = ty; rr < kNmsRowsPerCta; rr += 4) {
      const int cur = row_first + rr;      // warp-uniform
      if (cur >= n) break;
      bool bit = false;
      // diagonal block: only columns after the row itself (iou3d_kernel.cu:277-280)
      const bool active = tx < col_size && (row != col || tx > slice * kNmsRowsPerCta + rr);
      if (active) {
        const float* cur_box = srow + rr * 5;
        if (FMT == 4) {
          bit = rrpn_iou(cur_box, scol + tx * 5, -1) > (double)thresh;     // rotate_nms_kernel, nms_gpu.py:411-450
        } else if (FMT == 2) {
          bit = iou_axis_aligned(cur_box, scol + tx * 5) > thresh;
        } else {
          bit = iou_pixel(cur_box, scol + tx * 5) > (double)thresh;
        }
      }
      const unsigned int word = __ballot_sync(0xffffffffu, bit);
      if ((threadIdx.x & 31) == 0)
        mask32[((size_t)cur * col_blocks + col) * 2 + ((threadIdx.x >> 5) & 1)] = word;
    }
    }
  }
  if constexpr (FMT == 0) {
    __syncthreads();
    flush_pairs();
  }
}

// Greedy sweep on the device (iou3d.cpp:103-116 semantics), one CTA.
// `remv` lives in dynamic shared memory; stops as soon as max_keep boxes are kept.  When the upper
// triangle of the mask fits in shared memory (N <= ~1400, i.e. always at the detector's operating
// point of 1000 boxes) it is staged there with coalesced loads first, so the serial block-by-block
// resolve never waits on global memory.
__global__ void __launch_bounds__(1024)
nms_sweep_kernel(const unsigned long long* __restrict__ mask, int n_cap, const int* __restrict__ n_dev,
                 int col_blocks_alloc, int max_keep, long long* __restrict__ keep_idx,
                 int* __restrict__ keep_count, int stage_mask, long long mask_stride) {
  // blockIdx.x = box set of the batch
  mask += (size_t)blockIdx.x * mask_stride;
  keep_idx += (size_t)blockIdx.x * max_keep;
  keep_count += blockIdx.x;
  if (n_dev) n_dev += blockIdx.x;
  extern __shared__ unsigned long long remv[];
  __shared__ unsigned long long diag[kNmsBlock];
  __shared__ unsigned long long kept_word;
  __shared__ int kept_total, kept_base;
  const int n = n_dev ? min(*n_dev, n_cap) : n_cap;
  const int nb = (n + kNmsBlock - 1) / kNmsBlock;
  unsigned long long* smask = remv + col_blocks_alloc;      // [n][nb] when stage_mask
  for (int j = threadIdx.x; j < nb; j += blockDim.x) remv[j] = 0ULL;
  if (threadIdx.x == 0) kept_total = 0;
  if (stage_mask) {
#pragma unroll 4
    for (int e = threadIdx.x; e < n * nb; e += blockDim.x) {      // independent 8-byte loads, four in flight per thread
      const int i = e / nb, j = e - i * nb;
      smask[e] = j >= (i >> 6) ? __ldg(mask + (size_t)i * col_blocks_alloc + j) : 0ULL;
    }
  }
  __syncthreads();
  if (stage_mask) {
    // The detector's operating point (N <= ~1400, mask staged in shared memory): ONE warp walks the kept rows only.
    // Lane j holds remv[j]; per column block the not-yet-suppressed candidates are the zero bits of its word, the next
    // kept row is found with ffs, its mask row (nb <= 22 words, one per lane) is ORed in -- ~(kept + nb) short iterations
    // instead of four block-wide barriers and a 64-step serial scan per block.
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      unsigned long long rem = 0ULL;
      int total = 0;
      for (int b = 0; b < nb && total < max_keep; ++b) {
        const int in_block = min(n - b * kNmsBlock, kNmsBlock);
        const unsigned long long valid = in_block >= 64 ? ~0ULL : ((1ULL << in_block) - 1ULL);
        unsigned long long avail = ~__shfl_sync(0xffffffffu, rem, b) & valid;
        while (avail != 0ULL && total < max_keep) {
          const int i = __ffsll((long long)avail) - 1;
          const int row = b * kNmsBlock + i;
          if (lane == 0) keep_idx[total] = (long long)row;
          ++total;
          const unsigned long long r = lane < nb ? smask[(size_t)row * nb + lane] : 0ULL;
          rem |= r;
          avail &= ~__shfl_sync(0xffffffffu, r, b);          // suppressed inside this block
          avail &= ~((2ULL << i) - 1ULL);                     // row i itself and everything before it is decided
        }
      }
      if (lane == 0) *keep_count = total;
    }
    return;
  }
  for (int b = 0; b < nb; ++b) {
    const int in_block = min(n - b * kNmsBlock, kNmsBlock);
    if ((int)threadIdx.x < in_block) {
      const int i = b * kNmsBlock + threadIdx.x;
      diag[threadIdx.x] = stage_mask ? smask[(size_t)i * nb + b] : mask[(size_t)i * col_blocks_alloc + b];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      // serial resolve of the 64 rows of this block: ALU-only chain (the diag words are fetched eight at a time, the
      // keep list is written afterwards, in parallel, from the `kept` bits)
      unsigned long long cur = remv[b], kept = 0ULL;
      int total = kept_total;
      for (int i0 = 0; i0 < in_block && total < max_keep; i0 += 8) {
        unsigned long long d8[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) d8[u] = diag[(i0 + u) & (kNmsBlock - 1)];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int i = i0 + u;
          if (i < in_block && total < max_keep && !((cur >> i) & 1ULL)) {
            kept |= 1ULL << i;
            cur |= d8[u];
            ++total;
          }
        }
      }
      kept_word = kept;
      kept_base = kept_total;
      kept_total = total;
    }
    __syncthreads();
    const unsigned long long kept = kept_word;
    if (threadIdx.x < kNmsBlock && ((kept >> threadIdx.x) & 1ULL))       // keep list: rank among the kept rows of the block
      keep_idx[kept_base + __popcll(kept & ((1ULL << threadIdx.x) - 1ULL))] = (long long)b * kNmsBlock + threadIdx.x;
    if (kept_total >= max_keep) break;
    if (kept != 0ULL && stage_mask) {
      // staged mask (the detector's operating point, nb <= 22): one warp per later column block ORs the kept rows' words
      // (two rows per lane, warp reduction) -- no atomics, no dependent shared-memory chain
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
      for (int j = b + 1 + warp; j < nb; j += n_warps) {
        unsigned long long v = 0ULL;
        if ((kept >> lane) & 1ULL) v |= smask[(size_t)(b * kNmsBlock + lane) * nb + j];
        if ((kept >> (lane + 32)) & 1ULL) v |= smask[(size_t)(b * kNmsBlock + lane + 32) * nb + j];
        unsigned int lo = __reduce_or_sync(0xffffffffu, (unsigned int)v);
        unsigned int hi = __reduce_or_sync(0xffffffffu, (unsigned int)(v >> 32));
        if (lane == 0) remv[j] |= ((unsigned long long)hi << 32) | lo;
      }
    } else if (kept != 0ULL) {
      for (int j = b + 1 + threadIdx.x; j < nb; j += blockDim.x) {
        unsigned long long acc = remv[j];
        unsigned long long bits = kept;
        while (bits) {
          const int i = __ffsll((long long)bits) - 1;
          bits &= bits - 1;
          const int row = b * kNmsBlock + i;
          acc |= stage_mask ? smask[(size_t)row * nb + j] : mask[(size_t)row * col_blocks_alloc + j];
        }
        remv[j] = acc;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *keep_count = kept_total;
}

// `batch` independent box sets of the same capacity in two launches: set b has its boxes at boxes + b * n_cap * 5, its
// live count at n_dev[b], its keep list at keep_idx + b * max_keep and keep_count[b]; the workspace holds one mask per set.
int nms_batched(int fmt_kernel, const float* boxes, int n_cap, const int* n_dev, float thresh, int max_keep,
                long long* keep_idx, int* keep_count, void* workspace, size_t workspace_bytes, int batch,
                cudaStream_t stream) {
  const int col_blocks = div_up(n_cap, kNmsBlock);
  const size_t per_set = d3b_nms_workspace_bytes(n_cap);
  const size_t need = per_set * (size_t)batch;
  if (need > workspace_bytes) {
    set_error("nms: workspace %zu < %zu", workspace_bytes, need);
    return D3B_ERR_WORKSPACE;
  }
  unsigned long long* mask = (unsigned long long*)workspace;
  const long long mask_stride = (long long)(per_set / 8), box_stride = (long long)n_cap * 5;
  const long long items = (long long)col_blocks * (col_blocks + 1) / 2 * kNmsSlices;
  const int per_set_cap = kNumSMs * 16 / batch > 0 ? kNumSMs * 16 / batch : 1;
  const dim3 grid((unsigned)(items < (long long)per_set_cap ? (items > 0 ? items : 1) : per_set_cap), (unsigned)batch);
  if (fmt_kernel == 0)
    nms_mask_kernel<0><<<grid, 256, 0, stream>>>(boxes, n_cap, n_dev, thresh, col_blocks, mask, box_stride, mask_stride);
  else if (fmt_kernel == 1)
    nms_mask_kernel<1><<<grid, 256, 0, stream>>>(boxes, n_cap, n_dev, thresh, col_blocks, mask, box_stride, mask_stride);
  else if (fmt_kernel == 2)
    nms_mask_kernel<2><<<grid, 256, 0, stream>>>(boxes, n_cap, n_dev, thresh, col_blocks, mask, box_stride, mask_stride);
  else if (fmt_kernel == 4)
    nms_mask_kernel<4><<<grid, 256, 0, stream>>>(boxes, n_cap, n_dev, thresh, col_blocks, mask, box_stride, mask_stride);
  else
    nms_mask_kernel<3><<<grid, 256, 0, stream>>>(boxes, n_cap, n_dev, thresh, col_blocks, mask, box_stride, mask_stride);
  D3B_LAUNCH_CHECK();
  size_t smem = (size_t)col_blocks * 8;
  if (smem > 200 * 1024) {
    set_error("nms: %d boxes exceed the single-CTA sweep capacity", n_cap);
    return D3B_ERR_UNSUPPORTED;
  }
  const size_t staged = smem + (size_t)n_cap * col_blocks * 8;
  const int stage_mask = staged <= 200 * 1024 ? 1 : 0;
  if (stage_mask) smem = staged;
  static SmemOptIn sweep_optin;
  if (smem > 48 * 1024) D3B_CUDA(ensure_dynamic_smem(nms_sweep_kernel, 200 * 1024, sweep_optin));
  nms_sweep_kernel<<<batch, 1024, smem, stream>>>(mask, n_cap, n_dev, col_blocks, max_keep, keep_idx, keep_count,
                                                  stage_mask, mask_stride);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

static int nms_common(int fmt_kernel, const float* boxes, int n_cap, const int* n_dev, float thresh,
                      int max_keep, long long* keep_idx, int* keep_count, void* workspace,
                      size_t workspace_bytes, cudaStream_t stream) {
  return nms_batched(fmt_kernel, boxes, n_cap, n_dev, thresh, max_keep, keep_idx, keep_count, workspace, workspace_bytes, 1,
                     stream);
}

}  // namespace d3b

using namespace d3b;

extern "C" int d3b_boxes_iou_bev(const float* boxes_a, int32_t na, const float* boxes_b, int32_t nb,
                                 int32_t mode, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(na >= 0 && nb >= 0 && mode >= 0 && mode <= 2, "d3b_boxes_iou_bev: bad argument (mode %d)", mode);
  if (na == 0 || nb == 0) return D3B_OK;
  D3B_REQUIRE(boxes_a && boxes_b && out, "d3b_boxes_iou_bev: null argument");
  dim3 blocks(div_up(nb, 16), div_up(na, 16)), threads(16, 16);
  if (mode == 0)
    pair_matrix_kernel<0><<<blocks, threads, 0, stream>>>(na, boxes_a, nb, boxes_b, out);
  else if (mode == 1)
    pair_matrix_kernel<1><<<blocks, threads, 0, stream>>>(na, boxes_a, nb, boxes_b, out);
  else
    pair_matrix_kernel<2><<<blocks, threads, 0, stream>>>(na, boxes_a, nb, boxes_b, out);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" int d3b_rotate_iou_rrpn(const float* boxes, int32_t n, const float* query_boxes, int32_t k,
                                   int32_t criterion, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(n >= 0 && k >= 0, "d3b_rotate_iou_rrpn: bad argument");
  if (n == 0 || k == 0) return D3B_OK;
  D3B_REQUIRE(boxes && query_boxes && out, "d3b_rotate_iou_rrpn: null argument");
  dim3 blocks(div_up(k, 16), div_up(n, 16)), threads(16, 16);
  rrpn_matrix_kernel<<<blocks, threads, 0, stream>>>(n, boxes, k, query_boxes, criterion, out);
  D3B_LAUNCH_CHECK();
  return D3B_OK;
}

extern "C" size_t d3b_nms_workspace_bytes(int32_t n_cap) {
  if (n_cap <= 0) return 16;
  return align_up((size_t)n_cap * div_up(n_cap, kNmsBlock) * 8);
}

extern "C" int d3b_rotate_nms(const float* boxes, int32_t n_cap, const int32_t* n_boxes_dev, int32_t fmt,
                              float thresh, int32_t max_keep, int64_t* keep_idx, int32_t* keep_count,
                              void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(n_cap >= 0 && max_keep >= 0 && keep_count, "d3b_rotate_nms: bad argument");
  D3B_REQUIRE(fmt == D3B_BOX_XYXYR || fmt == D3B_BOX_XYWLR || fmt == D3B_BOX_XYWLR_RRPN,
              "d3b_rotate_nms: unknown box format %d", fmt);
  if (n_cap == 0 || max_keep == 0) {
    D3B_CUDA(cudaMemsetAsync(keep_count, 0, 4, stream));
    return D3B_OK;
  }
  D3B_REQUIRE(boxes && keep_idx && workspace, "d3b_rotate_nms: null argument");
  return nms_common(fmt == D3B_BOX_XYXYR ? 0 : (fmt == D3B_BOX_XYWLR ? 1 : 4), boxes, n_cap, n_boxes_dev, thresh, max_keep,
                    (long long*)keep_idx, keep_count, workspace, workspace_bytes, stream);
}

extern "C" int d3b_normal_nms(const float* boxes, int32_t n_cap, const int32_t* n_boxes_dev, int32_t mode,
                              float thresh, int32_t max_keep, int64_t* keep_idx, int32_t* keep_count, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3B_REQUIRE(n_cap >= 0 && max_keep >= 0 && keep_count, "d3b_normal_nms: bad argument");
  D3B_REQUIRE(mode == D3B_AA_IOU3D || mode == D3B_AA_PIXEL, "d3b_normal_nms: unknown mode %d", mode);
  if (n_cap == 0 || max_keep == 0) {
    D3B_CUDA(cudaMemsetAsync(keep_count, 0, 4, stream));
    return D3B_OK;
  }
  D3B_REQUIRE(boxes && keep_idx && workspace, "d3b_normal_nms: null argument");
  return nms_common(mode == D3B_AA_PIXEL ? 3 : 2, boxes, n_cap, n_boxes_dev, thresh, max_keep, (long long*)keep_idx,
                    keep_count, workspace, workspace_bytes, stream);
}
