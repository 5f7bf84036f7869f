"""TEST INFRASTRUCTURE: exact BEV overlap of two convex quadrilaterals, in rational arithmetic.

Every fp32 value is a dyadic rational, so `fractions.Fraction(float(v))` holds it exactly, and sums, products and
quotients of Fractions are exact.  Areas and IoUs computed here carry no rounding at all: they are the geometry of the
fp32 corners the kernels see, the yardstick for the fp64 Sutherland-Hodgman clipper of the rotate_nms_cc path
(csrc/nms.cu, oracle/iou3d_oracle.c (B)).

The method is deliberately not clipping.  The intersection of two convex polygons is the convex hull of (a) the
vertices of each polygon that lie inside or on the other and (b) the points where an edge of one crosses an edge of
the other: every vertex of the intersection is one of those points, and all of them lie in the intersection.  The hull
is taken with Andrew's monotone chain on exact coordinates, its area with the shoelace formula.

The gates of the rotate_nms_cc path are reproduced as the device has them: the IoU of the axis-aligned hulls in fp32
with eps 0 (box_np_ops.py:955-994, each operation rounded to fp32 as numpy float32 scalars do), then inter > 0 and
union > 0.
"""
import math
from fractions import Fraction

import numpy as np

_OX = (-0.5, -0.5, 0.5, 0.5)          # corners_nd order, origin 0.5 (box_np_ops.py:267-297)
_OY = (-0.5, 0.5, 0.5, -0.5)


def _cross(ox, oy, ax, ay, bx, by):
    return (ax - ox) * (by - oy) - (ay - oy) * (bx - ox)


def _exact(v):
    if float(np.float32(v)) != float(v):
        raise ValueError("corner %r is not an fp32 value" % (v,))
    return Fraction(float(v))


def _as_exact(quad):
    return [_exact(v) for v in quad[0]], [_exact(v) for v in quad[1]]


def _orientation(xs, ys):
    """+1 counter-clockwise, -1 clockwise; ValueError unless the quad is strictly convex."""
    signs = set()
    for k in range(4):
        k1, k2 = (k + 1) % 4, (k + 2) % 4
        c = _cross(xs[k], ys[k], xs[k1], ys[k1], xs[k2], ys[k2])
        signs.add((c > 0) - (c < 0))
    if signs == {1}:
        return 1
    if signs == {-1}:
        return -1
    raise ValueError("quad is not strictly convex: turn signs %s" % sorted(signs))


def polygon_area(xs, ys):
    """Exact area (non-negative Fraction) of a simple polygon given in order."""
    n = len(xs)
    s = sum(xs[k] * ys[(k + 1) % n] - xs[(k + 1) % n] * ys[k] for k in range(n))
    return abs(s) / 2


def _inside(px, py, xs, ys, orient):
    """p inside or on the boundary of the convex quad (xs, ys) of orientation `orient`."""
    for k in range(4):
        k1 = (k + 1) % 4
        if orient * _cross(xs[k], ys[k], xs[k1], ys[k1], px, py) < 0:
            return False
    return True


def _hull(points):
    """Andrew's monotone chain on exact points: hull vertices counter-clockwise, collinear points dropped."""
    pts = sorted(set(points))
    if len(pts) < 3:
        return pts
    lower, upper = [], []
    for p in pts:
        while len(lower) >= 2 and _cross(*lower[-2], *lower[-1], *p) <= 0:
            lower.pop()
        lower.append(p)
    for p in reversed(pts):
        while len(upper) >= 2 and _cross(*upper[-2], *upper[-1], *p) <= 0:
            upper.pop()
        upper.append(p)
    return lower[:-1] + upper[:-1]


def intersection_polygon(qa, qb):
    """Vertices (exact, counter-clockwise) of quad A ∩ quad B.  qa, qb = (x[4], y[4]) of fp32 corners, either
    orientation; each quad must be strictly convex."""
    ax, ay = _as_exact(qa)
    bx, by = _as_exact(qb)
    oa, ob = _orientation(ax, ay), _orientation(bx, by)
    pts = [(ax[k], ay[k]) for k in range(4) if _inside(ax[k], ay[k], bx, by, ob)]
    pts += [(bx[k], by[k]) for k in range(4) if _inside(bx[k], by[k], ax, ay, oa)]
    for i in range(4):
        i1 = (i + 1) % 4
        dx, dy = ax[i1] - ax[i], ay[i1] - ay[i]
        for j in range(4):
            j1 = (j + 1) % 4
            ex, ey = bx[j1] - bx[j], by[j1] - by[j]
            den = dx * ey - dy * ex
            if den == 0:            # parallel: a collinear overlap ends at vertices already collected above
                continue
            wx, wy = bx[j] - ax[i], by[j] - ay[i]
            t = (wx * ey - wy * ex) / den
            u = (wx * dy - wy * dx) / den
            if 0 <= t <= 1 and 0 <= u <= 1:
                pts.append((ax[i] + t * dx, ay[i] + t * dy))
    return _hull(pts)


def intersection_area(qa, qb):
    h = intersection_polygon(qa, qb)
    if len(h) < 3:
        return Fraction(0)
    return polygon_area([p[0] for p in h], [p[1] for p in h])


def quad_area(q):
    xs, ys = _as_exact(q)
    return polygon_area(xs, ys)


def standup_iou_f32(qa, qb):
    """The hull gate as the device computes it (csrc/nms.cu standup_iou): fp32, eps 0."""
    f = np.float32
    ax, ay = [f(v) for v in qa[0]], [f(v) for v in qa[1]]
    bx, by = [f(v) for v in qb[0]], [f(v) for v in qb[1]]
    iw = f(min(max(ax), max(bx)) - max(min(ax), min(bx)))
    if not iw > 0:
        return f(0)
    ih = f(min(max(ay), max(by)) - max(min(ay), min(by)))
    if not ih > 0:
        return f(0)
    area_b = f(f(max(bx) - min(bx)) * f(max(by) - min(by)))
    area_a = f(f(max(ax) - min(ax)) * f(max(ay) - min(ay)))
    inter = f(iw * ih)
    return f(inter / f(f(area_a + area_b) - inter))


def rotate_iou(qa, qb):
    """rotate_nms_cc overlap of two fp32 quads, exactly: (iou, union) as Fractions, or (None, None) when the hull gate,
    an empty intersection or an empty union skips the pair.  A skipped pair is never suppressed, not even at threshold
    0; the device's mode-2 matrix reports 0 for it."""
    if not standup_iou_f32(qa, qb) > 0:
        return None, None
    inter = intersection_area(qa, qb)
    if not inter > 0:
        return None, None
    union = quad_area(qa) + quad_area(qb) - inter
    if not union > 0:
        return None, None
    return inter / union, union


def suppresses(qa, qb, thresh):
    """The exact NMS decision: the pair is not skipped and IoU >= thresh (thresh a fp32 value)."""
    iou, _ = rotate_iou(qa, qb)
    return iou is not None and iou >= Fraction(float(np.float32(thresh)))


def to_f32(x):
    """Round a Fraction to the nearest fp32 (ties to even), exactly."""
    x = Fraction(x)
    if x == 0:
        return np.float32(0.0)
    lo = np.float32(float(x))                  # float() of a Fraction is correctly rounded to fp64
    # fp64 -> fp32 may double-round; settle on the fp32 neighbour nearest to x exactly
    cands = {lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))}
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.frombuffer(c.tobytes(), np.uint32)[0]) & 1))
    return np.float32(best)


def xywlr_corners_f32(box):
    """Corners of a [cx,cy,w,l,r] box in the device's fp32 operation order (csrc/nms.cu quad_of_xywlr), with the
    correctly rounded sin / cos of the fp32 angle.  Returns (x[4], y[4]) as np.float32."""
    f = np.float32
    cx, cy, w, l, r = (f(v) for v in box)
    s, c = f(math.sin(float(r))), f(math.cos(float(r)))
    xs, ys = [], []
    for k in range(4):
        px, py = f(w * f(_OX[k])), f(l * f(_OY[k]))
        xs.append(f(f(f(px * c) + f(py * s)) + cx))
        ys.append(f(f(f(-px * s) + f(py * c)) + cy))
    return np.array(xs, np.float32), np.array(ys, np.float32)
