"""Golden vectors for the KITTI camera-frustum crop, produced by the reference's own functions.

Run where the reference checkout exists:
    python tests/golden/make_golden_frustum.py [/path/to/Det3D]
det3d/core/bbox/box_np_ops.py imports spconv (not installable here) and the det3d package at import time, so the
functions on the path of `remove_outside_points` -- projection_matrix_to_CRT_kitti, get_frustum, camera_to_lidar,
corner_to_surfaces_3d_jit, remove_outside_points (box_np_ops.py:576-607,909-914,941-952,1133-1152) and
surface_equ_3d_jitv2, _points_in_convex_polygon_3d_jit, points_in_convex_polygon_3d_jit (core/bbox/geometry.py:
215-276,351-377) -- are lifted from the source with `ast` and exec'd unchanged, their numba decorators included, with
a stub `spconv` module in place.  Calibrations are synthetic (utils/synthetic.kitti_like_calib), one per KITTI image
shape plus seeded perturbations and one axis-aligned calibration; each golden stores the calibrations, their planes
(the reference's normal_vec / d), the clouds and the reference's keep masks.

Outputs:
  frustum_kitti_scans.npz        4 calibrations x one 360° raw scan each (utils/synthetic.raw_velodyne_scan, 8k points)
  frustum_kitti_adversarial.npz  8 calibrations x adversarial points: f32 roundings of points on every plane nudged by
                                 +-1..4 ulps, frustum edges and corners, the near (0.001 m) and far (100 m) planes,
                                 points behind the camera, NaN / +-inf coordinates, and points whose s is exactly 0
  frustum_kitti_rounding.npz     40 hand-built plane tables (no calibration) with points whose reference value s is
                                 exactly 0 or a few units in the last place from it, built so that an FMA-contracted
                                 evaluation, a reordered sum or a `>` test decides differently from the reference's
                                 ((x*n0 + y*n1) + z*n2) + d >= 0; the generator checks that each such variant
                                 (oracle/frustum.PLANE_VALUE_VARIANTS) disagrees with the reference's mask on some point,
                                 and that numba compiled the reference loop without any FMA instruction
"""
import ast
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from det3d_b200.utils.synthetic import KITTI_IMAGE_SHAPES, kitti_like_calib, raw_velodyne_scan  # noqa: E402

BOX_NP_OPS = ("projection_matrix_to_CRT_kitti", "get_frustum", "camera_to_lidar", "corner_to_surfaces_3d_jit",
              "remove_outside_points")
GEOMETRY = ("surface_equ_3d_jitv2", "_points_in_convex_polygon_3d_jit", "points_in_convex_polygon_3d_jit")


def _lift(path, names, ns):
    src = open(path).read()
    nodes = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in nodes) == sorted(names), [n.name for n in nodes]
    exec(compile(ast.Module(body=nodes, type_ignores=[]), path, "exec"), ns)


def reference_namespace(ref_root):
    import numba

    sys.modules.setdefault("spconv", types.ModuleType("spconv"))        # box_np_ops.py imports spconv.utils
    ns = {"np": np, "numba": numba}
    _lift(os.path.join(ref_root, "det3d/core/bbox/geometry.py"), GEOMETRY, ns)
    _lift(os.path.join(ref_root, "det3d/core/bbox/box_np_ops.py"), BOX_NP_OPS, ns)
    return ns


def reference_planes(ns, calib):
    """The steps of remove_outside_points up to the point test, with the reference's functions: normal_vec [6, 3] and
    d [6] of surface_equ_3d_jitv2, and the frustum corners [8, 3]."""
    C, R, T = ns["projection_matrix_to_CRT_kitti"](calib["P2"])
    image_shape = calib["image_shape"]
    frustum = ns["get_frustum"]([0, 0, image_shape[1], image_shape[0]], C)
    frustum -= T
    frustum = np.linalg.inv(R) @ frustum.T
    frustum = ns["camera_to_lidar"](frustum.T, calib["rect"], calib["Trv2c"])
    surfaces = ns["corner_to_surfaces_3d_jit"](frustum[np.newaxis, ...])
    normal_vec, d = ns["surface_equ_3d_jitv2"](surfaces[:, :, :3, :])
    return np.concatenate([normal_vec[0], d[0][:, None]], axis=1), frustum


def reference_mask(ns, points, calib):
    """remove_outside_points' own mask (points_in_convex_polygon_3d_jit on the reference's surfaces)."""
    C, R, T = ns["projection_matrix_to_CRT_kitti"](calib["P2"])
    image_shape = calib["image_shape"]
    frustum = ns["get_frustum"]([0, 0, image_shape[1], image_shape[0]], C)
    frustum -= T
    frustum = np.linalg.inv(R) @ frustum.T
    frustum = ns["camera_to_lidar"](frustum.T, calib["rect"], calib["Trv2c"])
    surfaces = ns["corner_to_surfaces_3d_jit"](frustum[np.newaxis, ...])
    mask = ns["points_in_convex_polygon_3d_jit"](points[:, :3], surfaces).reshape(-1)
    kept = ns["remove_outside_points"](points, calib["rect"], calib["Trv2c"], calib["P2"], calib["image_shape"])
    assert np.array_equal(kept.view(np.uint32), points[mask].view(np.uint32))
    return mask


def axis_aligned_calib():
    """Camera on the LiDAR's x axis, no rotation, a dyadic translation, P2 = K [I | 0]: the near plane's corners then
    share one float32 x and its normal is (n0, 0, 0), so a point with that x has s = 0 exactly."""
    K = np.array([[720.0, 0, 608.0], [0, 720.0, 172.0], [0, 0, 1.0]])
    P2 = np.eye(4)
    P2[:3, :3] = K
    Trv2c = np.eye(4)
    Trv2c[:3, :3] = [[0, -1.0, 0], [0, 0, -1.0], [1.0, 0, 0]]
    Trv2c[:3, 3] = [0.0, 0.0, -0.249]                 # camera 0.249 m ahead of the LiDAR: near plane at x = 0.25
    return dict(rect=np.eye(4), Trv2c=Trv2c, P2=P2, image_shape=np.array((375, 1242), np.int64))


def _f32_nudges(p, rng, k):
    """k float32 points around p [3] (f64): round, then move every coordinate by -4..+4 ulps."""
    base = p.astype(np.float32)
    steps = rng.integers(-4, 5, (k, 3))
    out = np.repeat(base[None], k, 0)
    for j in range(3):
        for i in range(k):
            for _ in range(abs(int(steps[i, j]))):
                out[i, j] = np.nextafter(out[i, j], np.float32(np.inf if steps[i, j] > 0 else -np.inf))
    return out


def _s(planes, p):
    x, y, z = (p[:, j].astype(np.float64) for j in range(3))
    return [((x * n[0] + y * n[1]) + z * n[2]) + n[3] for n in planes]


def adversarial_points(planes, corners, rng, ndim=4):
    faces = [[0, 1, 2, 3], [7, 6, 5, 4], [0, 3, 7, 4], [1, 5, 6, 2], [0, 4, 5, 1], [3, 2, 6, 7]]
    pts = []
    for f in faces:                                   # points on each face (convex combinations of its corners)
        w = rng.dirichlet(np.ones(4), 24)
        for q in w @ corners[f]:
            pts.append(_f32_nudges(q, rng, 6))
    edges = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
    for a, b in edges:                                # frustum edges and corners
        for t in (0.0, 0.25, 0.5, 1.0):
            pts.append(_f32_nudges(corners[a] * (1 - t) + corners[b] * t, rng, 4))
    centre = corners.mean(0)
    axis = corners[4:].mean(0) - corners[:4].mean(0)
    axis /= np.linalg.norm(axis)
    near_c, far_c = corners[:4].mean(0), corners[4:].mean(0)
    for c in (near_c, far_c):                         # the near (0.001 m) and far (100 m) planes along the axis
        for dd in np.linspace(-1e-3, 1e-3, 9):
            pts.append(_f32_nudges(c + dd * axis, rng, 3))
    for dd in np.linspace(0.1, 50, 16):               # behind the camera
        pts.append(_f32_nudges(near_c - dd * axis + rng.normal(0, 2, 3), rng, 2))
    pts.append(_f32_nudges(centre, rng, 4))
    p = np.concatenate(pts, 0)
    specials = np.array([[np.nan, 0, 0], [0, np.nan, 0], [0, 0, np.nan], [np.inf, 0, 0], [-np.inf, 0, 0],
                         [0, np.inf, 0], [0, -np.inf, 0], [0, 0, np.inf], [0, 0, -np.inf], [np.nan] * 3,
                         [np.inf, np.inf, np.inf], [centre[0], np.nan, centre[2]], [np.inf, centre[1], centre[2]],
                         [0, 0, 0], [-0.0, -0.0, -0.0]], np.float32)
    p = np.concatenate([p, specials], 0)
    out = np.zeros((p.shape[0], ndim), np.float32)
    out[:, :3] = p
    if ndim > 3:
        out[:, 3] = rng.uniform(0, 1, p.shape[0]).astype(np.float32)
    return out


def exact_zero_points(planes, corners, ndim=4):
    """Points with s == 0 exactly on the near plane of the axis-aligned calibration (n = (n0, 0, 0))."""
    n = planes[0]
    assert n[1] == 0 and n[2] == 0 and np.float32(corners[0, 0]) == corners[0, 0], planes[0]
    x = np.float32(corners[0, 0])
    out = np.zeros((3, ndim), np.float32)
    out[:, 0] = x
    out[:, 1:3] = [[0.0, 0.0], [0.01, -0.002], [-0.02, 0.003]]
    return out


def _rounds_up(a, b):
    from fractions import Fraction
    return Fraction(a * b) > Fraction(a) * Fraction(b)


def rounding_cases(rng, ndim=4):
    """Plane tables [B, 6, 4] and clouds whose decisions depend on how s is rounded.  Each table has one test plane in
    slot b % 6 and five planes (0, 0, 0, -1) that keep every finite point.  Families, with c a float32 and r = rn(c*n)
    rounded up (so c*n - r < 0):
      fma_z   point (1, 0, c), n0 = -rn(c*n2): the reference's s is exactly 0 (dropped); fma(c, n2, n0) < 0 (kept)
      fma_y   point (1, c, 0), n0 = -rn(c*n1): exactly 0; fma(c, n1, n0) < 0
      fma_x   point (c, 1, 0), n1 = -rn(c*n0): exactly 0; fma(c, n0, n1) < 0
      fma_d   point (c, 0, 0), d = -rn(c*n0): exactly 0; fma(c, n0, d) < 0
      order   point (a, a, a), n = (2^k, 2^(k-54), -2^k), d = -2^(k-54): the reference rounds a*2^(k-54) away against
              a*2^k and keeps s = d < 0, other association orders cancel to 0
    Each cloud also holds the point's neighbours at +-1 and +-2 ulps of c (or of a)."""
    tables, clouds, kinds = [], [], []
    families = ("fma_z", "fma_y", "fma_x", "fma_d", "order")
    for i in range(40):
        fam = families[i % len(families)]
        while True:
            c = np.float32(rng.uniform(1, 100))
            n = float(rng.uniform(-50, 50) * 10.0 ** rng.integers(-3, 4))
            if fam == "order" or _rounds_up(float(c), n):
                break
        plane = np.zeros(4)
        r = float(c) * n
        if fam == "fma_z":
            plane[:] = [-r, rng.uniform(-5, 5), n, 0.0]
            base = (np.float32(1), np.float32(0), c)
        elif fam == "fma_y":
            plane[:] = [-r, n, rng.uniform(-5, 5), 0.0]
            base = (np.float32(1), c, np.float32(0))
        elif fam == "fma_x":
            plane[:] = [n, -r, rng.uniform(-5, 5), 0.0]
            base = (c, np.float32(1), np.float32(0))
        elif fam == "fma_d":
            plane[:] = [n, rng.uniform(-5, 5), rng.uniform(-5, 5), -r]
            base = (c, np.float32(0), np.float32(0))
        else:
            k = int(rng.integers(-20, 20))
            plane[:] = [2.0 ** k, 2.0 ** (k - 54), -(2.0 ** k), -(2.0 ** (k - 54))]
            base = (c, c, c)
        pts = []
        for step in (0, 1, -1, 2, -2):
            q = list(base)
            for j in range(3):
                if q[j] == c:                      # nudge the coordinates that carry c
                    v = c
                    for _ in range(abs(step)):
                        v = np.nextafter(v, np.float32(np.inf if step > 0 else -np.inf))
                    q[j] = v
            pts.append(q)
        cloud = np.zeros((len(pts), ndim), np.float32)
        cloud[:, :3] = np.array(pts, np.float32)
        if ndim > 3:
            cloud[:, 3] = rng.uniform(0, 1, len(pts)).astype(np.float32)
        table = np.tile(np.array([0.0, 0.0, 0.0, -1.0]), (6, 1))
        table[i % 6] = plane
        tables.append(table)
        clouds.append(cloud)
        kinds.append(fam)
    return np.stack(tables), clouds, kinds


def reference_mask_of_planes(ns, points, table):
    """The reference's point loop (_points_in_convex_polygon_3d_jit) on a hand-built plane table [6, 4]."""
    surfaces = np.zeros((1, 6, 4, 3))                  # only its shape is read
    normal_vec = np.ascontiguousarray(table[np.newaxis, :, :3])
    d = np.ascontiguousarray(table[np.newaxis, :, 3])
    return ns["_points_in_convex_polygon_3d_jit"](points[:, :3], surfaces, normal_vec, d,
                                                  np.full((1,), 9999999, dtype=np.int64)).reshape(-1)


def fma_instructions(ns):
    """FMA instructions in numba's machine code of the reference's point loop, over every compiled signature."""
    import re
    asm = ns["_points_in_convex_polygon_3d_jit"].inspect_asm()
    return sum(len(re.findall(r"\bv?fn?m(add|sub)\w*", a)) for a in asm.values())


def main():
    ref_root = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    ns = reference_namespace(ref_root)

    def pack(calibs, clouds, masks, planes):
        return dict(rect=np.stack([c["rect"] for c in calibs]), Trv2c=np.stack([c["Trv2c"] for c in calibs]),
                    P2=np.stack([c["P2"] for c in calibs]), image_shape=np.stack([c["image_shape"] for c in calibs]),
                    planes=np.stack(planes), offsets=np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]),
                    points=np.concatenate(clouds), mask=np.concatenate(masks))

    # raw scans
    calibs = [kitti_like_calib(10 + i, shape) for i, shape in enumerate(KITTI_IMAGE_SHAPES)]
    clouds = [raw_velodyne_scan(8192, 4, seed=100 + i) for i in range(len(calibs))]
    planes = [reference_planes(ns, c)[0] for c in calibs]
    masks = [reference_mask(ns, p, c) for p, c in zip(clouds, calibs)]
    np.savez_compressed(os.path.join(HERE, "frustum_kitti_scans.npz"), **pack(calibs, clouds, masks, planes))
    print("scans: kept", [int(m.sum()) for m in masks], "of", [c.shape[0] for c in clouds])

    # adversarial points
    rng = np.random.default_rng(2024)
    calibs = [kitti_like_calib(0, KITTI_IMAGE_SHAPES[0], perturb=False)]
    calibs += [kitti_like_calib(20 + i, KITTI_IMAGE_SHAPES[i % 4]) for i in range(6)]
    calibs.append(axis_aligned_calib())
    clouds, masks, planes = [], [], []
    n_zero = n_close = 0
    for c in calibs:
        pl, corners = reference_planes(ns, c)
        p = adversarial_points(pl, corners, rng)
        if c is calibs[-1]:
            p = np.concatenate([p, exact_zero_points(pl, corners)], 0)
        s = np.stack(_s(pl, p), 1)
        n_zero += int((s == 0).sum())
        n_close += int((np.abs(s) < 1e-6 * np.abs(pl[:, :3]).max()).sum())
        clouds.append(p)
        planes.append(pl)
        masks.append(reference_mask(ns, p, c))
    assert n_zero >= 1
    np.savez_compressed(os.path.join(HERE, "frustum_kitti_adversarial.npz"), **pack(calibs, clouds, masks, planes))
    print("adversarial: %d points, %d kept, %d plane tests with s == 0, %d with |s| tiny"
          % (sum(c.shape[0] for c in clouds), sum(int(m.sum()) for m in masks), n_zero, n_close))

    # rounding-order discriminators on hand-built plane tables
    from oracle.frustum import PLANE_VALUE_VARIANTS, keep_mask, variant_keep_mask
    tables, clouds, kinds = rounding_cases(np.random.default_rng(77))
    masks = [reference_mask_of_planes(ns, c, t) for c, t in zip(clouds, tables)]
    n_fma = fma_instructions(ns)
    assert n_fma == 0, "numba contracted the reference's point loop into %d FMA instructions" % n_fma
    points = np.concatenate(clouds)
    caught = {}
    for v in list(PLANE_VALUE_VARIANTS) + ["strict_gt"]:
        other = np.concatenate([variant_keep_mask(c, t, v) for c, t in zip(clouds, tables)])
        caught[v] = int((other != np.concatenate(masks)).sum())
        assert caught[v] >= 4, (v, caught[v])
    assert all(np.array_equal(keep_mask(c, t), m) for c, t, m in zip(clouds, tables, masks))
    np.savez_compressed(os.path.join(HERE, "frustum_kitti_rounding.npz"), planes=tables, points=points,
                        offsets=np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]),
                        mask=np.concatenate(masks), family=np.array(kinds))
    print("rounding: %d tables, %d points, %d kept; FMA instructions in the reference loop: %d; points each variant "
          "decides differently: %s" % (len(clouds), points.shape[0], int(np.concatenate(masks).sum()), n_fma, caught))


if __name__ == "__main__":
    main()
