/*
 * TEST INFRASTRUCTURE -- CPU oracle, not product code.
 *
 * (A) fp32 restatement of the reference CUDA rotated-BEV IoU / NMS
 *       det3d/ops/iou3d/src/iou3d_kernel.cu:36-221 (cross, check_rect_cross,
 *       check_in_box2d, intersection, rotate_around_center, point_cmp,
 *       box_overlap, iou_bev), :295-303 (iou_normal) and the greedy sweep of
 *       det3d/ops/iou3d/src/iou3d.cpp:103-116.
 *     Boxes [x1, y1, x2, y2, ry], suppress when iou > thresh.
 *     Host libm sinf/cosf/atan2f and unfused mul/add replace libdevice and
 *     nvcc's FMA contraction, so values agree with the GPU reference to a few
 *     ulp, not bit for bit: the bit-exact pin of the CUDA product is the
 *     reference kernel itself (oracle/_ref/libiou3d_ref.so, built from the
 *     reference source by oracle/Makefile and run on the GPU box) plus the
 *     fixtures it generated (tests/golden/iou3d_*.npz).
 *
 * (B) restatement of the CPU rotated NMS that Det3D inference actually calls
 *       det3d/ops/nms/nms_cpu.py:34-45 (rotate_nms_cc)
 *       det3d/core/bbox/box_np_ops.py:267-297,335-340,419-432,477-497,955-994
 *       det3d/ops/nms/nms_cpu.h:73-169 (rotate_non_max_suppression_cpu)
 *     Boxes [cx, cy, w, l, r, score]; suppress when inter/union >= thresh and
 *     the axis-aligned hulls overlap.  boost::geometry is absent from this
 *     image, so polygon intersection is Sutherland-Hodgman in fp64 and
 *     union = area_a + area_b - inter ("parity unpinned" at the boost boundary:
 *     IoU agrees to rounding, decisions can differ only for |IoU - thr| ~ 1e-6).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float x, y; } pt;

static const float EPS = 1e-8f;

static float cross2(pt a, pt b) { return a.x * b.y - a.y * b.x; }                 /* :36-38 */
static float cross3(pt p1, pt p2, pt p0) {                                        /* :40-42 */
  return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}
static int rect_cross(pt p1, pt p2, pt q1, pt q2) {                               /* :44-50 */
  return fminf(p1.x, p2.x) <= fmaxf(q1.x, q2.x) && fminf(q1.x, q2.x) <= fmaxf(p1.x, p2.x) &&
         fminf(p1.y, p2.y) <= fmaxf(q1.y, q2.y) && fminf(q1.y, q2.y) <= fmaxf(p1.y, p2.y);
}
static int in_box2d(const float* box, pt p) {                                     /* :52-65 */
  const float MARGIN = 1e-5f;
  float cx = (box[0] + box[2]) / 2, cy = (box[1] + box[3]) / 2;
  float c = cosf(-box[4]), s = sinf(-box[4]);
  float rx = (p.x - cx) * c + (p.y - cy) * s + cx;
  float ry = -(p.x - cx) * s + (p.y - cy) * c + cy;
  return rx > box[0] - MARGIN && rx < box[2] + MARGIN && ry > box[1] - MARGIN && ry < box[3] + MARGIN;
}
static int intersection(pt p1, pt p0, pt q1, pt q0, pt* ans) {                    /* :67-96 */
  if (!rect_cross(p0, p1, q0, q1)) return 0;
  float s1 = cross3(q0, p1, p0), s2 = cross3(p1, q1, p0);
  float s3 = cross3(p0, q1, q0), s4 = cross3(q1, p1, q0);
  if (!(s1 * s2 > 0 && s3 * s4 > 0)) return 0;
  float s5 = cross3(q1, p1, p0);
  if (fabsf(s5 - s1) > EPS) {
    ans->x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
    ans->y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
  } else {
    float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
    float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
    float D = a0 * b1 - a1 * b0;
    ans->x = (b0 * c1 - b1 * c0) / D;
    ans->y = (a1 * c0 - a0 * c1) / D;
  }
  return 1;
}
static pt rot(pt c, float ac, float as, pt p) {                                   /* :98-102 */
  pt r;
  r.x = (p.x - c.x) * ac + (p.y - c.y) * as + c.x;
  r.y = -(p.x - c.x) * as + (p.y - c.y) * ac + c.y;
  return r;
}
static int pcmp(pt a, pt b, pt c) {                                               /* :104-106 */
  return atan2f(a.y - c.y, a.x - c.x) > atan2f(b.y - c.y, b.x - c.x);
}

float oracle_box_overlap(const float* A, const float* B) {                        /* :108-212 */
  pt ca = {(A[0] + A[2]) / 2, (A[1] + A[3]) / 2}, cb = {(B[0] + B[2]) / 2, (B[1] + B[3]) / 2};
  pt a[5] = {{A[0], A[1]}, {A[2], A[1]}, {A[2], A[3]}, {A[0], A[3]}};
  pt b[5] = {{B[0], B[1]}, {B[2], B[1]}, {B[2], B[3]}, {B[0], B[3]}};
  float aco = cosf(A[4]), asi = sinf(A[4]), bco = cosf(B[4]), bsi = sinf(B[4]);
  for (int k = 0; k < 4; k++) { a[k] = rot(ca, aco, asi, a[k]); b[k] = rot(cb, bco, bsi, b[k]); }
  a[4] = a[0]; b[4] = b[0];
  pt cp[16], ctr = {0, 0};
  int cnt = 0;
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++)
      if (intersection(a[i + 1], a[i], b[j + 1], b[j], &cp[cnt])) {
        ctr.x += cp[cnt].x; ctr.y += cp[cnt].y; cnt++;
      }
  for (int k = 0; k < 4; k++) {
    if (in_box2d(A, b[k])) { ctr.x += b[k].x; ctr.y += b[k].y; cp[cnt++] = b[k]; }
    if (in_box2d(B, a[k])) { ctr.x += a[k].x; ctr.y += a[k].y; cp[cnt++] = a[k]; }
  }
  ctr.x /= cnt; ctr.y /= cnt;                              /* 0/0 = NaN when cnt == 0; unused then */
  for (int j = 0; j < cnt - 1; j++)
    for (int i = 0; i < cnt - j - 1; i++)
      if (pcmp(cp[i], cp[i + 1], ctr)) { pt t = cp[i]; cp[i] = cp[i + 1]; cp[i + 1] = t; }
  float area = 0;
  for (int k = 0; k < cnt - 1; k++) {
    pt u = {cp[k].x - cp[0].x, cp[k].y - cp[0].y}, v = {cp[k + 1].x - cp[0].x, cp[k + 1].y - cp[0].y};
    area += cross2(u, v);
  }
  return (float)(fabsf(area) / 2.0);
}

float oracle_iou_bev(const float* A, const float* B) {                            /* :214-221 */
  float sa = (A[2] - A[0]) * (A[3] - A[1]), sb = (B[2] - B[0]) * (B[3] - B[1]);
  float so = oracle_box_overlap(A, B);
  return so / fmaxf(sa + sb - so, EPS);
}

float oracle_iou_normal(const float* a, const float* b) {                         /* :295-303 */
  float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  float w = fmaxf(right - left, 0.f), h = fmaxf(bottom - top, 0.f);
  float inter = w * h;
  float sa = (a[2] - a[0]) * (a[3] - a[1]), sb = (b[2] - b[0]) * (b[3] - b[1]);
  return inter / fmaxf(sa + sb - inter, EPS);
}

void oracle_iou_matrix(const float* A, int na, const float* B, int nb, int mode, float* out) {
#pragma omp parallel for schedule(dynamic, 16)
  for (int i = 0; i < na; ++i)
    for (int j = 0; j < nb; ++j)
      out[(size_t)i * nb + j] = mode == 0 ? oracle_iou_bev(A + 5 * i, B + 5 * j) : oracle_box_overlap(A + 5 * i, B + 5 * j);
}

/* Greedy sweep equivalent to nms_kernel's bitmask (:250-292) + iou3d.cpp:103-116:
 * boxes sorted by score; box j>i is removed when a KEPT box i has iou(i,j) > thresh.
 * rotated = 1: iou_bev, 0: iou_normal.  Returns the number kept. */
int64_t oracle_nms_xyxyr(const float* boxes, int64_t n, float thresh, int rotated, int64_t* keep) {
  uint8_t* dead = (uint8_t*)calloc((size_t)(n > 0 ? n : 1), 1);
  int64_t nk = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (dead[i]) continue;
    keep[nk++] = i;
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t j = i + 1; j < n; ++j) {
      if (dead[j]) continue;
      float v = rotated ? oracle_iou_bev(boxes + 5 * i, boxes + 5 * j) : oracle_iou_normal(boxes + 5 * i, boxes + 5 * j);
      if (v > thresh) dead[j] = 1;
    }
  }
  free(dead);
  return nk;
}

/* ------------------------------------------------------------------------- (B) */
typedef struct { float x[4], y[4], minx, miny, maxx, maxy; } quad;

/* box_np_ops.py:267-297 corners_nd (clockwise from the min corner, origin 0.5),
 * :419-432 rotation_2d (x' = x cos + y sin, y' = -x sin + y cos), :477-497, :335-340. */
static quad make_quad(const float* d) {
  quad q;
  const float ox[4] = {-0.5f, -0.5f, 0.5f, 0.5f}, oy[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
  float s = sinf(d[4]), c = cosf(d[4]);
  for (int k = 0; k < 4; ++k) {
    float px = d[2] * ox[k], py = d[3] * oy[k];
    q.x[k] = (px * c + py * s) + d[0];
    q.y[k] = (-px * s + py * c) + d[1];
  }
  q.minx = fminf(fminf(q.x[0], q.x[1]), fminf(q.x[2], q.x[3]));
  q.maxx = fmaxf(fmaxf(q.x[0], q.x[1]), fmaxf(q.x[2], q.x[3]));
  q.miny = fminf(fminf(q.y[0], q.y[1]), fminf(q.y[2], q.y[3]));
  q.maxy = fmaxf(fmaxf(q.y[0], q.y[1]), fmaxf(q.y[2], q.y[3]));
  return q;
}
/* box_np_ops.py:955-994 with eps = 0 */
static float standup_iou(const quad* a, const quad* b) {
  float iw = fminf(a->maxx, b->maxx) - fmaxf(a->minx, b->minx);
  if (!(iw > 0)) return 0.f;
  float ih = fminf(a->maxy, b->maxy) - fmaxf(a->miny, b->miny);
  if (!(ih > 0)) return 0.f;
  float ab = (b->maxx - b->minx) * (b->maxy - b->miny), aa = (a->maxx - a->minx) * (a->maxy - a->miny);
  float ua = aa + ab - iw * ih;
  return iw * ih / ua;
}
static double quad_area(const quad* q) {
  double a = 0;
  for (int k = 0; k < 4; ++k) { int k1 = (k + 1) & 3; a += (double)q->x[k] * q->y[k1] - (double)q->x[k1] * q->y[k]; }
  return fabs(a) * 0.5;
}
/* Vertex capacity, as csrc/nms.cu kClipMaxVertices: a clip step keeps k of n vertices and adds one per sign change
 * (at most 2 min(k, n - k)), so m <= floor(3n / 2) for ANY sign pattern -- rounding can break convexity for
 * near-duplicate pairs, where exact arithmetic would give at most 8.  4 -> 6 -> 9 -> 13 -> 19. */
#define CLIP_MAX_VERTICES 19

/* *max_n (when not NULL) receives the largest vertex count of any intermediate polygon */
static double clip_area_n(const quad* A, const quad* B, int* max_n) {
  double px[CLIP_MAX_VERTICES], py[CLIP_MAX_VERTICES], qx[CLIP_MAX_VERTICES], qy[CLIP_MAX_VERTICES];
  int n = 4, top = 4;
  for (int k = 0; k < 4; ++k) { px[k] = A->x[k]; py[k] = A->y[k]; }
  double area2 = 0;
  for (int k = 0; k < 4; ++k) { int k1 = (k + 1) & 3; area2 += (double)B->x[k] * B->y[k1] - (double)B->x[k1] * B->y[k]; }
  double sgn = area2 >= 0 ? 1.0 : -1.0;
  for (int e = 0; e < 4 && n > 0; ++e) {
    int e1 = (e + 1) & 3, m = 0;
    double ex = (double)B->x[e1] - B->x[e], ey = (double)B->y[e1] - B->y[e];
    for (int k = 0; k < n; ++k) {
      int k1 = (k + 1 == n) ? 0 : k + 1;
      double d0 = sgn * (ex * (py[k] - B->y[e]) - ey * (px[k] - B->x[e]));
      double d1 = sgn * (ex * (py[k1] - B->y[e]) - ey * (px[k1] - B->x[e]));
      if (d0 >= 0) { qx[m] = px[k]; qy[m] = py[k]; ++m; }
      if ((d0 >= 0) != (d1 >= 0)) {
        double t = d0 / (d0 - d1);
        qx[m] = px[k] + t * (px[k1] - px[k]); qy[m] = py[k] + t * (py[k1] - py[k]); ++m;
      }
    }
    n = m;
    if (n > top) top = n;
    memcpy(px, qx, sizeof(double) * n); memcpy(py, qy, sizeof(double) * n);
  }
  if (max_n) *max_n = top;
  if (n < 3) return 0;
  double a = 0;
  for (int k = 0; k < n; ++k) { int k1 = (k + 1 == n) ? 0 : k + 1; a += px[k] * py[k1] - px[k1] * py[k]; }
  return fabs(a) * 0.5;
}
static double clip_area(const quad* A, const quad* B) { return clip_area_n(A, B, NULL); }

/* Test access to the clipper.  Corners of one [cx,cy,w,l,r] box as the (B) path builds them: out = x[4], y[4]. */
void oracle_xywlr_corners(const float* d, float* out) {
  quad q = make_quad(d);
  memcpy(out, q.x, sizeof(float) * 4);
  memcpy(out + 4, q.y, sizeof(float) * 4);
}

/* Largest intermediate vertex count of clip_area(a[i], b[i]) for n pairs of [cx,cy,w,l,r] boxes -> out[i]. */
void oracle_clip_max_vertices(const float* da, const float* db, int64_t n, int32_t* out) {
#pragma omp parallel for schedule(static, 4096)
  for (int64_t i = 0; i < n; ++i) {
    quad a = make_quad(da + 5 * i), b = make_quad(db + 5 * i);
    int top = 0;
    clip_area_n(&a, &b, &top);
    out[i] = top;
  }
}

/* IoU the (B) path thresholds: 0 when the hulls do not overlap (pair skipped, nms_cpu.h:105). */
float oracle_rotate_iou_xywlr(const float* da, const float* db) {
  quad a = make_quad(da), b = make_quad(db);
  if (standup_iou(&a, &b) <= 0.0f) return 0.f;
  double inter = clip_area(&a, &b);
  if (!(inter > 0)) return 0.f;
  double uni = quad_area(&a) + quad_area(&b) - inter;
  if (!(uni > 0)) return 0.f;
  return (float)(inter / uni);
}

/* nms_cpu.py:34-45 + nms_cpu.h:73-169. dets [n,6] = cx,cy,w,l,r,score in ANY order;
 * `order` = indices by descending score (computed by the caller like argsort()[::-1]).
 * Returns kept count; keep[] holds ORIGINAL indices in visiting order. */
int64_t oracle_rotate_nms_cc(const float* dets, const int32_t* order, int64_t n, float thresh, int64_t* keep) {
  uint8_t* sup = (uint8_t*)calloc((size_t)(n > 0 ? n : 1), 1);
  quad* q = (quad*)malloc(sizeof(quad) * (size_t)(n > 0 ? n : 1));
  for (int64_t i = 0; i < n; ++i) q[i] = make_quad(dets + 6 * i);
  int64_t nk = 0;
  for (int64_t _i = 0; _i < n; ++_i) {
    int64_t i = order[_i];
    if (sup[i]) continue;
    keep[nk++] = i;
    for (int64_t _j = _i + 1; _j < n; ++_j) {
      int64_t j = order[_j];
      if (sup[j]) continue;
      if (standup_iou(&q[i], &q[j]) <= 0.0f) continue;                 /* nms_cpu.h:105 */
      double inter = clip_area(&q[i], &q[j]);
      if (!(inter > 0)) continue;                                      /* poly_inter.empty() */
      double uni = quad_area(&q[i]) + quad_area(&q[j]) - inter;
      if (!(uni > 0)) continue;
      if ((float)(inter / uni) >= thresh) sup[j] = 1;                  /* :157 */
    }
  }
  free(sup); free(q);
  return nk;
}

/* ==========================================================================
 * (C) RRPN rotated IoU -- restatement of the numba.cuda device functions
 *     det3d/ops/nms/nms_gpu.py:180-470 (rotate_iou_gpu / rotate_nms_gpu).
 *     Boxes [cx,cy,w,l,r].  float where numba types float32, double where a
 *     literal promotes (":185-196" areas, "center /= n", the final ratio).
 *     Pinned by tests/golden/rrpn_600.npz (reference source compiled for CPU).
 * ========================================================================== */
static void rrpn_corners(const float* rb, float* c) {                                  /* :368-390 */
  float a_cos = cosf(rb[4]), a_sin = sinf(rb[4]);
  float hx = (float)((double)rb[2] / 2.0), hy = (float)((double)rb[3] / 2.0);
  float cx[4] = {-hx, -hx, hx, hx}, cy[4] = {-hy, hy, hy, -hy};
  for (int i = 0; i < 4; ++i) {
    c[2 * i] = a_cos * cx[i] + a_sin * cy[i] + rb[0];
    c[2 * i + 1] = -a_sin * cx[i] + a_cos * cy[i] + rb[1];
  }
}
static int rrpn_point_in_quad(float px, float py, const float* c) {                    /* :325-341 */
  float ab0 = c[2] - c[0], ab1 = c[3] - c[1], ad0 = c[6] - c[0], ad1 = c[7] - c[1];
  float ap0 = px - c[0], ap1 = py - c[1];
  float abab = ab0 * ab0 + ab1 * ab1, abap = ab0 * ap0 + ab1 * ap1;
  float adad = ad0 * ad0 + ad1 * ad1, adap = ad0 * ap0 + ad1 * ap1;
  return abab >= abap && abap >= 0 && adad >= adap && adap >= 0;
}
static int rrpn_seg(const float* p1, const float* p2, int i, int j, float* out) {      /* :239-281 */
  float A0 = p1[2 * i], A1 = p1[2 * i + 1], B0 = p1[2 * ((i + 1) % 4)], B1 = p1[2 * ((i + 1) % 4) + 1];
  float C0 = p2[2 * j], C1 = p2[2 * j + 1], D0 = p2[2 * ((j + 1) % 4)], D1 = p2[2 * ((j + 1) % 4) + 1];
  float BA0 = B0 - A0, BA1 = B1 - A1, DA0 = D0 - A0, CA0 = C0 - A0, DA1 = D1 - A1, CA1 = C1 - A1;
  int acd = DA1 * CA0 > CA1 * DA0;
  int bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0);
  if (acd != bcd) {
    int abc = CA1 * BA0 > BA1 * CA0, abd = DA1 * BA0 > BA1 * DA0;
    if (abc != abd) {
      float DC0 = D0 - C0, DC1 = D1 - C1, ABBA = A0 * B1 - B0 * A1, CDDC = C0 * D1 - D0 * C1;
      float DH = BA1 * DC0 - BA0 * DC1, Dx = ABBA * DC0 - BA0 * CDDC, Dy = ABBA * DC1 - BA1 * CDDC;
      out[0] = Dx / DH;
      out[1] = Dy / DH;
      return 1;
    }
  }
  return 0;
}
static double rrpn_inter(const float* rb1, const float* rb2) {                         /* :393-408 */
  float c1[8], c2[8], pts[16], t[2];
  rrpn_corners(rb1, c1);
  rrpn_corners(rb2, c2);
  int n = 0;
  for (int i = 0; i < 4; ++i) {                                                         /* :344-365 */
    if (n < 8 && rrpn_point_in_quad(c1[2 * i], c1[2 * i + 1], c2)) { pts[2 * n] = c1[2 * i]; pts[2 * n + 1] = c1[2 * i + 1]; ++n; }
    if (n < 8 && rrpn_point_in_quad(c2[2 * i], c2[2 * i + 1], c1)) { pts[2 * n] = c2[2 * i]; pts[2 * n + 1] = c2[2 * i + 1]; ++n; }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j)
      if (n < 8 && rrpn_seg(c1, c2, i, j, t)) { pts[2 * n] = t[0]; pts[2 * n + 1] = t[1]; ++n; }
  if (n > 0) {                                                                          /* :199-236 */
    float cen0 = 0.f, cen1 = 0.f, vs[8];
    for (int i = 0; i < n; ++i) { cen0 += pts[2 * i]; cen1 += pts[2 * i + 1]; }
    cen0 = (float)((double)cen0 / (double)n);
    cen1 = (float)((double)cen1 / (double)n);
    for (int i = 0; i < n; ++i) {
      float v0 = pts[2 * i] - cen0, v1 = pts[2 * i + 1] - cen1;
      float d = sqrtf(v0 * v0 + v1 * v1);
      v0 = v0 / d;
      v1 = v1 / d;
      if (v1 < 0) v0 = (float)(-2.0 - (double)v0);
      vs[i] = v0;
    }
    for (int i = 1; i < n; ++i) {
      if (vs[i - 1] > vs[i]) {
        float temp = vs[i], tx = pts[2 * i], ty = pts[2 * i + 1];
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
  double area = 0.0;                                                                    /* :185-196 */
  for (int i = 0; i < n - 2; ++i)
    area += fabs((double)((pts[0] - pts[2 * i + 4]) * (pts[2 * i + 3] - pts[2 * i + 5]) -
                          (pts[1] - pts[2 * i + 5]) * (pts[2 * i + 2] - pts[2 * i + 4])) / 2.0);
  return area;
}

/* devRotateIoUEval :585-597 */
double oracle_rrpn_iou(const float* rb1, const float* rb2, int criterion) {
  float area1 = rb1[2] * rb1[3], area2 = rb2[2] * rb2[3];
  double ai = rrpn_inter(rb1, rb2);
  if (criterion == -1) return ai / ((double)(area1 + area2) - ai);
  if (criterion == 0) return ai / (double)area1;
  if (criterion == 1) return ai / (double)area2;
  return ai;
}

/* rotate_iou_kernel_eval :600-640: out[n,k] = f(query[k], boxes[n]) */
void oracle_rrpn_iou_matrix(const float* boxes, int n, const float* query, int k, int criterion, float* out) {
#pragma omp parallel for
  for (int a = 0; a < n; ++a)
    for (int b = 0; b < k; ++b) out[(size_t)a * k + b] = (float)oracle_rrpn_iou(query + 5 * b, boxes + 5 * a, criterion);
}

/* rotate_nms_gpu :453-496 (mask kernel :411-450 + nms_postprocess :110-127).  dets [n,6] = cx,cy,w,l,r,score,
 * `order` = argsort(score)[::-1]; keep[] receives ORIGINAL indices.  near[0] counts tested pairs whose IoU lies
 * within 1e-4 of the threshold (their outcome may differ between sin/cos / FMA implementations). */
int64_t oracle_rrpn_nms(const float* dets, const int32_t* order, int64_t n, float thresh, int64_t* keep, int64_t* near) {
  uint8_t* sup = (uint8_t*)calloc((size_t)(n > 0 ? n : 1), 1);
  int64_t nk = 0, nn = 0;
  for (int64_t _i = 0; _i < n; ++_i) {
    if (sup[_i]) continue;
    int64_t i = order[_i];
    keep[nk++] = i;
    for (int64_t _j = _i + 1; _j < n; ++_j) {
      double iou = oracle_rrpn_iou(dets + 6 * i, dets + 6 * order[_j], -1);
      if (fabs(iou - (double)thresh) < 1e-4) ++nn;
      if (iou > (double)thresh) sup[_j] = 1;
    }
  }
  if (near) near[0] = nn;
  free(sup);
  return nk;
}

/* Host greedy sweep of the reference's iou3d NMS, det3d/ops/iou3d/src/iou3d.cpp:103-116: mask [n][col_blocks] u64 as
 * copied back from nms_kernel, remv accumulates the suppressed columns; keep[] receives the kept (sorted) indices. */
int64_t oracle_iou3d_host_sweep(const uint64_t* mask, int64_t n, int64_t col_blocks, int64_t* keep) {
  uint64_t* remv = (uint64_t*)calloc((size_t)(col_blocks > 0 ? col_blocks : 1), sizeof(uint64_t));
  int64_t nk = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t nblock = i / 64, inblock = i % 64;
    if (!(remv[nblock] & (1ULL << inblock))) {
      keep[nk++] = i;
      const uint64_t* p = mask + i * col_blocks;
      for (int64_t j = nblock; j < col_blocks; ++j) remv[j] |= p[j];
    }
  }
  free(remv);
  return nk;
}
