"""TEST INFRASTRUCTURE -- CPU restatement of the reference's camera-frustum point test
(det3d/core/bbox/geometry.py:241-276, _points_in_convex_polygon_3d_jit, as remove_outside_points calls it,
det3d/core/bbox/box_np_ops.py:941-952).  Pinned by tests/golden/frustum_kitti_*.npz (the reference functions
themselves, tests/golden/make_golden_frustum.py).  Never imported by det3d_b200."""
import numpy as np


def keep_mask(points, planes):
    """points [N, >= 3] float32, planes [6, 4] float64 (n0, n1, n2, d) -> bool [N]: True where every plane gives
    s = ((x*n0 + y*n1) + z*n2) + d < 0, the coordinates promoted to float64 and each operation rounded on its own
    (numpy's elementwise ops never fuse).  The reference drops a point at the first s >= 0, so a NaN s keeps it."""
    p = np.asarray(points)
    x, y, z = (p[:, j].astype(np.float64) for j in range(3))
    keep = np.ones(p.shape[0], bool)
    with np.errstate(invalid="ignore"):
        for n0, n1, n2, d in np.asarray(planes, np.float64):
            s = ((x * n0 + y * n1) + z * n2) + d
            keep &= ~(s >= 0)
    return keep


def remove_outside_points(points, planes):
    """points[keep_mask(points, planes)]: every column, input order kept."""
    return np.asarray(points)[keep_mask(points, planes)]


def _fma(a, b, c):
    """a*b + c with one rounding (exact rational arithmetic, correctly rounded back to float64)."""
    from fractions import Fraction
    for v in (a, b, c):
        if not np.isfinite(v):
            return a * b + c
    return float(Fraction(a) * Fraction(b) + Fraction(c))


# Other ways to evaluate one plane value s from (x, y, z) and (n0, n1, n2, d), each a plausible compilation of the
# reference's `x*n0 + y*n1 + z*n2 + d` that is not its evaluation: contracted into FMAs (as a C compiler may do by
# default), summed in another order, or tested with `>` instead of `>=`.  Used to show that the rounding goldens tell
# them apart from the reference.
PLANE_VALUE_VARIANTS = {
    "fma_chain_yx": lambda x, y, z, n0, n1, n2, d: _fma(z, n2, _fma(y, n1, x * n0)) + d,
    "fma_chain_xy": lambda x, y, z, n0, n1, n2, d: _fma(z, n2, _fma(x, n0, y * n1)) + d,
    "fma_d_first": lambda x, y, z, n0, n1, n2, d: _fma(z, n2, _fma(y, n1, _fma(x, n0, d))),
    "d_first": lambda x, y, z, n0, n1, n2, d: ((d + x * n0) + y * n1) + z * n2,
    "right_assoc": lambda x, y, z, n0, n1, n2, d: x * n0 + (y * n1 + (z * n2 + d)),
    "pairwise": lambda x, y, z, n0, n1, n2, d: (x * n0 + y * n1) + (z * n2 + d),
}


def variant_keep_mask(points, planes, variant):
    """keep_mask with plane values from PLANE_VALUE_VARIANTS[variant], or with `s > 0` as the outside test for
    variant == "strict_gt"."""
    p = np.asarray(points)
    if variant == "strict_gt":
        x, y, z = (p[:, j].astype(np.float64) for j in range(3))
        keep = np.ones(p.shape[0], bool)
        with np.errstate(invalid="ignore"):
            for n0, n1, n2, d in np.asarray(planes, np.float64):
                keep &= ~(((x * n0 + y * n1) + z * n2) + d > 0)
        return keep
    f = PLANE_VALUE_VARIANTS[variant]
    keep = np.ones(p.shape[0], bool)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(p.shape[0]):
            x, y, z = (float(np.float64(v)) for v in p[i, :3])
            for n0, n1, n2, d in np.asarray(planes, np.float64).tolist():
                if f(x, y, z, n0, n1, n2, d) >= 0:
                    keep[i] = False
                    break
    return keep
