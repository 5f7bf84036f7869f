"""Seeded families of [cx, cy, w, l, r] box pairs for the rotate_nms_cc IoU (tests/test_rotate_iou_exact.py on the
CPU oracle, tests/test_rotate_nms_exact_gpu.py on the device).  Each family aims at a regime where a polygon clipper
goes wrong: coincident edges and corners (sign tests at exactly 0), near-duplicates (t ~ 0 or 1, rounding that breaks
convexity), exact r = 0 answers, hulls that overlap while the polygons do not, maximal vertex counts, far range and
small or thin boxes."""
import math

import numpy as np

F = np.float32
HALF_PI, PI = F(math.pi / 2), F(math.pi)


def _box(cx, cy, w, l, r):
    return np.array([cx, cy, w, l, r], np.float32)


def _ulps(v, k):
    v = F(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, F(np.inf) if k > 0 else F(-np.inf))
    return v


def _car(rng):
    return F(rng.uniform(1.4, 2.2)), F(rng.uniform(3.4, 5.2))


def identical(rng, n):
    """The same rectangle twice: at r = 0, pi/2, pi and random r; written as (w, l, r) and (l, w, r + pi/2); r and
    r + pi."""
    out = []
    for i in range(n):
        cx, cy = F(rng.uniform(-40, 40)), F(rng.uniform(-40, 40))
        w, l = _car(rng)
        kind = i % 6
        r = [F(0), HALF_PI, PI, F(rng.uniform(-PI, PI))][min(kind, 3)]
        a = _box(cx, cy, w, l, r)
        if kind < 4:
            out.append((a, a.copy()))
        elif kind == 4:
            out.append((a, _box(cx, cy, l, w, F(r + HALF_PI))))
        else:
            out.append((a, _box(cx, cy, w, l, F(r + PI))))
    return out


def near_duplicates(rng, n, far=False):
    """The same box with the centre moved by 1-4 ulps, the angle perturbed by 1e-9 to 1e-3 rad and w or l scaled by
    1 +- 1e-7 to 1e-3; each perturbation alone or all together.  Most pairs are at r ~ 0 or pi/2, where the detector's
    anchors put them."""
    out = []
    for i in range(n):
        span = 100.0 if far else 40.0
        cx, cy = F(rng.uniform(-span, span)), F(rng.uniform(-span, span))
        w, l = _car(rng) if i % 3 else (F(rng.uniform(0.4, 0.8)), F(rng.uniform(0.4, 0.8)))
        r = [F(0), HALF_PI, F(rng.normal(0, 0.05)), F(rng.uniform(-PI, PI))][i % 4]
        a = _box(cx, cy, w, l, r)
        b = a.copy()
        what = rng.integers(0, 4)          # 0 centre, 1 angle, 2 size, 3 all three
        if what in (0, 3):
            b[0] = _ulps(b[0], int(rng.integers(1, 5)) * int(rng.choice([-1, 1])))
            b[1] = _ulps(b[1], int(rng.integers(1, 5)) * int(rng.choice([-1, 1])))
        if what in (1, 3):
            b[4] = F(float(b[4]) + rng.choice([-1, 1]) * 10.0 ** rng.uniform(-9, -3))
        if what in (2, 3):
            k = 2 + int(rng.integers(0, 2))
            b[k] = F(float(b[k]) * (1 + rng.choice([-1, 1]) * 10.0 ** rng.uniform(-7, -3)))
        out.append((a, b))
    return out


def near_duplicate_batch(rng, n, angle_exp=(-9, -3), scale_exp=(-7, -3)):
    """[n, 5] x 2 arrays of near-duplicate pairs for a bulk search: car- or pedestrian-sized boxes at r ~ 0 or pi/2 (or
    random r), the partner with its centre moved by 1-4 ulps in x and y, the angle perturbed by 1e-9 to 1e-3 rad and w
    or l scaled by 1 +- 1e-7 to 1e-3, all at once."""
    a = np.empty((n, 5), np.float32)
    a[:, 0:2] = rng.uniform(-40, 40, (n, 2))
    car = rng.random(n) < 0.5
    a[:, 2] = np.where(car, rng.uniform(1.4, 2.2, n), rng.uniform(0.4, 0.8, n))
    a[:, 3] = np.where(car, rng.uniform(3.4, 5.2, n), rng.uniform(0.4, 0.8, n))
    base = rng.integers(0, 3, n)
    a[:, 4] = np.where(base == 0, 0.0, np.where(base == 1, HALF_PI, rng.uniform(-math.pi, math.pi, n)))
    b = a.copy()
    for c in (0, 1):
        steps = rng.integers(1, 5, n) * rng.choice([-1, 1], n)
        for k in range(1, 5):
            m = np.abs(steps) >= k
            b[m, c] = np.nextafter(b[m, c], np.where(steps[m] > 0, np.inf, -np.inf).astype(np.float32))
    b[:, 4] = (b[:, 4].astype(np.float64) + rng.choice([-1, 1], n) * 10.0 ** rng.uniform(*angle_exp, n)).astype(np.float32)
    col = 2 + rng.integers(0, 2, n)
    scale = 1 + rng.choice([-1, 1], n) * 10.0 ** rng.uniform(*scale_exp, n)
    b[np.arange(n), col] = (b[np.arange(n), col].astype(np.float64) * scale).astype(np.float32)
    return a, b


def exact_r0():
    """Axis-aligned cases whose corners are exact on every host and device (sin 0 = 0, cos 0 = 1), with known answers:
    (box a, box b, exact IoU or None when a gate skips the pair)."""
    from fractions import Fraction as Q
    b = _box
    return [
        (b(0, 0, 2, 2, 0), b(2, 0, 2, 2, 0), None),                 # shared edge: hull width 0
        (b(0, 0, 2, 2, 0), b(2, 2, 2, 2, 0), None),                 # shared corner
        (b(0, 0, 4, 4, 0), b(0.5, -0.5, 2, 1, 0), Q(2, 16)),         # containment
        (b(0, 0, 4, 2, 0), b(1, 0, 4, 2, 0), Q(6, 10)),              # collinear edges, partial overlap (y edges shared)
        (b(0, 0, 4, 2, 0), b(1, 0.5, 2, 1, 0), Q(1, 4)),             # b's edge x = 2 lies on a's edge x = 2
        (b(0, 0, 3, 1, 0), b(1, 0, 3, 1, 0), Q(1, 2)),               # inter 2, union 4: IoU exactly 0.5
        (b(10.5, -3.25, 3, 1, 0), b(11.5, -3.25, 3, 1, 0), Q(1, 2)),
        (b(0, 0, 2, 4, 0), b(0, 0, 2, 4, 0), Q(1)),
        (b(-7.75, 3.5, 1.5, 0.5, 0), b(-7.75, 3.75, 1.5, 0.5, 0), Q(1, 3)),
    ]


def diamonds(rng, n):
    """Two squares at 45 deg near their tips: the axis-aligned hulls overlap, the polygons are apart by a gap of
    5 mm or more."""
    out = []
    q = F(math.pi / 4)
    for _ in range(n):
        s = rng.uniform(0.5, 4.0)
        half_diag = s / math.sqrt(2)
        # centres (0,0) and (c,c): facing edges x + y = h and x + y = 2c - h, gap (2c - 2h) / sqrt2 >= 5 mm;
        # the hulls overlap while c < 2h
        c = rng.uniform(half_diag + 0.005, 1.9 * half_diag)
        x0, y0 = rng.uniform(-40, 40, 2)
        out.append((_box(x0, y0, s, s, q), _box(x0 + c, y0 + c, s, s, q)))
    return out


def octagons(rng, n):
    """A square against itself rotated by 45 deg (a regular octagon: 8 vertices) and by 1e-4 rad (8 vertices, four of
    them a hair from the corners)."""
    out = []
    for i in range(n):
        s = F(rng.uniform(0.4, 4.0))
        cx, cy = F(rng.uniform(-60, 60)), F(rng.uniform(-60, 60))
        r = [F(0), F(rng.uniform(-PI, PI))][i % 2]
        d = [math.pi / 4, 1e-4][(i // 2) % 2]
        out.append((_box(cx, cy, s, s, r), _box(cx, cy, s, s, F(float(r) + d))))
    return out


def far_small(rng, n):
    """Centres near +-100 m (Lyft range); pedestrians and cones (0.4-0.8 m), bicycles, thin boxes (w = 0.05 m);
    partners displaced by up to about one box size so that most pairs overlap."""
    out = []
    for i in range(n):
        cx = F(rng.choice([-1, 1]) * rng.uniform(95, 100))
        cy = F(rng.choice([-1, 1]) * rng.uniform(90, 100))
        kind = i % 3
        if kind == 0:
            w, l = F(rng.uniform(0.4, 0.8)), F(rng.uniform(0.4, 0.8))
        elif kind == 1:
            w, l = F(rng.uniform(0.5, 0.8)), F(rng.uniform(1.6, 1.9))
        else:
            w, l = F(0.05), F(rng.uniform(0.5, 2.0))
        r = F(rng.uniform(-PI, PI)) if i % 4 else F(0)
        size = float(max(w, l))
        a = _box(cx, cy, w, l, r)
        b = _box(F(cx + rng.uniform(-0.5, 0.5) * size), F(cy + rng.uniform(-0.5, 0.5) * size),
                 F(w * rng.uniform(0.8, 1.25)), F(l * rng.uniform(0.8, 1.25)), F(r + rng.normal(0, 0.3)))
        out.append((a, b))
    return out


def families(seed=0, n=96):
    """{name: [(box a, box b), ...]} for every family, deterministic in `seed`."""
    rng = np.random.default_rng(seed)
    return {
        "identical": identical(rng, n),
        "near_duplicate": near_duplicates(rng, n),
        "near_duplicate_far": near_duplicates(rng, n, far=True),
        "exact_r0": [(a, b) for a, b, _ in exact_r0()],
        "diamond_tips": diamonds(rng, n),
        "octagon": octagons(rng, n),
        "far_small": far_small(rng, n),
    }


def on_grid(groups, pitch=20.0):
    """Lay groups of boxes out on a square grid of `pitch` metres, the first box of each group on its grid point, so
    that the hull gate separates the groups (the grid reaches past +-100 m for a few hundred groups).  A translation
    re-rounds the centres: the pairs stay near-duplicates, not the same ulp pattern; r = 0 cases with small dyadic
    coordinates stay exact.  Returns ([n, 5] boxes, group id per box)."""
    side = int(math.ceil(math.sqrt(len(groups))))
    boxes, gid = [], []
    for g, group in enumerate(groups):
        ox, oy = pitch * (g % side - side // 2), pitch * (g // side - side // 2)
        x0, y0 = float(group[0][0]), float(group[0][1])
        for bx in group:
            b = np.array(bx, np.float32).copy()
            b[0], b[1] = F(float(b[0]) - x0 + ox), F(float(b[1]) - y0 + oy)
            boxes.append(b)
            gid.append(g)
    return np.array(boxes, np.float32).reshape(-1, 5), np.array(gid)


def detector_clusters(seed, n=1000):
    """Boxes like the decoded candidates that reach NMS: centres on anchor strides of 0.16 m and 0.4 m (plus a few
    cm of regression), r in {0, pi/2} + N(0, 0.05), sizes near-duplicates of one object per cluster."""
    rng = np.random.default_rng(seed)
    boxes = []
    while len(boxes) < n:
        stride = [0.16, 0.4][len(boxes) // 100 % 2]
        k = len(boxes) // 100
        ox, oy = 20.0 * (k % 5 - 2), 20.0 * (k // 5 - 1)
        w0, l0 = (F(1.6), F(3.9)) if k % 3 else (F(0.6), F(0.8))
        base_r = [0.0, math.pi / 2][k % 2]
        for _ in range(min(100, n - len(boxes))):
            ix, iy = rng.integers(-6, 7, 2)
            cx = ox + ix * stride + rng.normal(0, 0.03)
            cy = oy + iy * stride + rng.normal(0, 0.03)
            w = float(w0) * (1 + rng.normal(0, 1e-3)) if rng.random() < 0.7 else float(w0)
            l = float(l0) * (1 + rng.normal(0, 1e-3)) if rng.random() < 0.7 else float(l0)
            r = base_r + (rng.normal(0, 0.05) if rng.random() < 0.8 else 0.0)
            boxes.append(_box(cx, cy, w, l, r))
    return np.array(boxes[:n], np.float32)
