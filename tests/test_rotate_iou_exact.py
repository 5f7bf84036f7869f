"""The rotate_nms_cc overlap (D3B_BOX_XYWLR) against exact geometry, on the CPU.

oracle/exact_polygon.py computes the intersection of two quads from their fp32 corners in rational arithmetic, by a
method independent of the fp64 Sutherland-Hodgman clipper that the C oracle (oracle/iou3d_oracle.c (B)) and the device
(csrc/nms.cu) share.  Given the oracle's own corners, the oracle's IoU must be fl32(exact IoU) to within 1 ulp on every
family of tests/rotated_box_families.py, which pins the clip algorithm at every angle.  The clipper's vertex buffers
are checked against the proven worst case and against the largest count the families reach."""
import ctypes as C
import os
import re
from fractions import Fraction

import numpy as np
import pytest

from conftest import ROOT
from oracle import build as obuild
from oracle import exact_polygon as ep
import rotated_box_families as fam


@pytest.fixture(scope="module")
def lib():
    l = C.CDLL(obuild.build())
    l.oracle_rotate_iou_xywlr.restype = C.c_float
    l.oracle_rotate_iou_xywlr.argtypes = [C.c_void_p, C.c_void_p]
    l.oracle_xywlr_corners.restype = None
    l.oracle_xywlr_corners.argtypes = [C.c_void_p, C.c_void_p]
    l.oracle_clip_max_vertices.restype = None
    l.oracle_clip_max_vertices.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    return l


def _corners(lib, box):
    box = np.ascontiguousarray(box, np.float32)
    out = np.zeros(8, np.float32)
    lib.oracle_xywlr_corners(box.ctypes.data, out.ctypes.data)
    return out[:4], out[4:]


def _oracle_iou(lib, a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return np.float32(lib.oracle_rotate_iou_xywlr(a.ctypes.data, b.ctypes.data))


def _max_vertices(lib, a, b):
    a, b = np.ascontiguousarray(a, np.float32).reshape(-1, 5), np.ascontiguousarray(b, np.float32).reshape(-1, 5)
    out = np.zeros(a.shape[0], np.int32)
    lib.oracle_clip_max_vertices(a.ctypes.data, b.ctypes.data, a.shape[0], out.ctypes.data)
    return out


def ulp_distance(x, y):
    """Distance in fp32 steps between two non-negative fp32 values."""
    ix = int(np.float32(x).view(np.int32))
    iy = int(np.float32(y).view(np.int32))
    return abs(ix - iy)


# ---------------------------------------------------------------------------------------------- the exact reference
def _q(xs, ys):
    return np.array(xs, np.float32), np.array(ys, np.float32)


def test_exact_reference_known_answers():
    sq = _q([0, 2, 2, 0], [0, 0, 2, 2])                       # counter-clockwise
    sq_cw = _q([0, 0, 2, 2], [0, 2, 2, 0])                    # the same square clockwise
    diamond = _q([1, 2.5, 1, -0.5], [-0.5, 1, 2.5, 1])        # |x-1| + |y-1| <= 1.5: cuts four 0.5-leg triangles
    assert ep.quad_area(sq) == 4 and ep.quad_area(diamond) == Fraction(9, 2)
    assert ep.intersection_area(sq, diamond) == Fraction(7, 2)
    assert len(ep.intersection_polygon(sq, diamond)) == 8       # an octagon
    assert ep.intersection_area(sq_cw, diamond) == Fraction(7, 2) == ep.intersection_area(diamond, sq_cw)
    assert ep.rotate_iou(sq, diamond)[0] == Fraction(7, 10)
    assert ep.intersection_area(sq, sq_cw) == 4 and ep.rotate_iou(sq, sq)[0] == 1
    inner = _q([0.5, 1.5, 1.5, 0.5], [0.5, 0.5, 1.0, 1.0])
    assert ep.intersection_area(sq, inner) == Fraction(1, 2) and ep.rotate_iou(inner, sq)[0] == Fraction(1, 8)
    # touching along an edge or at a corner: area 0, and the hull gate skips the pair
    right = _q([2, 4, 4, 2], [0, 0, 2, 2])
    corner = _q([2, 4, 4, 2], [2, 2, 4, 4])
    assert ep.intersection_area(sq, right) == 0 and ep.rotate_iou(sq, right) == (None, None)
    assert ep.intersection_area(sq, corner) == 0 and ep.rotate_iou(sq, corner) == (None, None)
    # hulls overlap, polygons apart: the gate passes, the empty intersection skips the pair
    d1 = _q([0, 1, 0, -1], [-1, 0, 1, 0])
    d2 = _q([1.25, 2.25, 1.25, 0.25], [0.25, 1.25, 2.25, 1.25])
    assert ep.standup_iou_f32(d1, d2) > 0 and ep.intersection_area(d1, d2) == 0 and ep.rotate_iou(d1, d2) == (None, None)
    assert not ep.suppresses(d1, d2, 0.0) and ep.suppresses(sq, diamond, 0.7) and not ep.suppresses(sq, diamond, 0.70001)
    with pytest.raises(ValueError):
        ep.intersection_area(_q([0, 2, 0, 2], [0, 0, 2, 2]), sq)          # a bow tie is not a convex quad
    with pytest.raises(ValueError):
        ep.intersection_area((np.array([0.1, 2, 2, 0]), np.array([0.0, 0, 2, 2])), sq)   # float64 0.1 is no fp32 value
    assert ep.to_f32(Fraction(1, 3)) == np.float32(1 / 3) and ep.to_f32(Fraction(7, 10)) == np.float32(0.7)
    # the midpoint between two fp32 neighbours of 1 rounds to even
    assert ep.to_f32(1 + Fraction(1, 2 ** 24)) == np.float32(1.0)
    assert ep.to_f32(1 + Fraction(3, 2 ** 24)) == np.nextafter(np.nextafter(np.float32(1), np.float32(2)), np.float32(2))


def test_exact_r0_families_known_answers():
    """At r = 0 the corners are exact (sin 0 = 0, cos 0 = 1 on every host and device)."""
    for a, b, want in fam.exact_r0():
        got, _ = ep.rotate_iou(ep.xywlr_corners_f32(a), ep.xywlr_corners_f32(b))
        assert got == want, (a, b, got, want)


def test_host_corners_follow_the_oracle_at_r0(lib):
    for a, b, _ in fam.exact_r0():
        for box in (a, b):
            h, o = ep.xywlr_corners_f32(box), _corners(lib, box)
            assert np.array_equal(h[0], o[0]) and np.array_equal(h[1], o[1])


# ------------------------------------------------------------------------------------------ the oracle against it
@pytest.mark.parametrize("name", sorted(fam.families(0)))
def test_oracle_iou_is_exact_to_one_ulp(lib, name):
    pairs = fam.families(0)[name]
    worst, n_skipped = 0, 0
    for a, b in pairs:
        for x, y in ((a, b), (b, a)):
            exact, _ = ep.rotate_iou(_corners(lib, x), _corners(lib, y))
            got = _oracle_iou(lib, x, y)
            if exact is None:
                n_skipped += 1
                assert got == 0.0, (name, x, y, got)
                continue
            d = ulp_distance(got, ep.to_f32(exact))
            worst = max(worst, d)
            assert d <= 1, (name, x, y, float(got), float(exact))
    print("%s: %d pairs (both orders), %d skipped, worst %d ulp" % (name, 2 * len(pairs), n_skipped, worst))
    if name in ("diamond_tips",):
        assert n_skipped == 2 * len(pairs)
    elif name not in ("exact_r0", "far_small"):
        assert n_skipped == 0


def test_oracle_decisions_on_the_exact_r0_cases(lib):
    """Inclusive threshold at an IoU of exactly 0.5; pairs the gates skip are kept even at threshold 0."""
    from oracle.second_cpu import rotate_nms_cc
    for a, b, want in fam.exact_r0():
        dets = np.array([list(a) + [0.9], list(b) + [0.8]], np.float32)
        for thr in (0.0, 0.5, 1.0):
            suppressed = want is not None and want >= Fraction(thr)
            assert rotate_nms_cc(dets, thr).tolist() == ([0] if suppressed else [0, 1]), (a, b, thr)


# ----------------------------------------------------------------------------------------------- vertex buffers
def _capacity(path, pattern):
    m = re.search(pattern, open(os.path.join(ROOT, path)).read())
    assert m, "%s: %s not found" % (path, pattern)
    return int(m.group(1))


def proven_vertex_bound():
    """A clip step keeps k of n vertices and adds one per sign change of the cyclic sequence (at most 2 min(k, n - k)),
    so m <= floor(3n / 2) whatever the signs are -- and rounding decides the signs of near-duplicate pairs."""
    n, top = 4, 4
    for _ in range(4):
        n = max(k + 2 * min(k, n - k) for k in range(n + 1))
        top = max(top, n)
    return top


def test_clip_buffers_hold_the_proven_bound():
    assert proven_vertex_bound() == 19
    assert _capacity("det3d_b200/csrc/nms.cu", r"constexpr int kClipMaxVertices = (\d+);") >= proven_vertex_bound()
    assert _capacity("oracle/iou3d_oracle.c", r"#define CLIP_MAX_VERTICES (\d+)") >= proven_vertex_bound()
    # every buffer of both clippers is sized by the constant
    assert re.search(r"double px\[kClipMaxVertices\], py\[kClipMaxVertices\], qx\[kClipMaxVertices\], "
                     r"qy\[kClipMaxVertices\];", open(os.path.join(ROOT, "det3d_b200/csrc/nms.cu")).read())
    assert re.search(r"double px\[CLIP_MAX_VERTICES\], py\[CLIP_MAX_VERTICES\], qx\[CLIP_MAX_VERTICES\], "
                     r"qy\[CLIP_MAX_VERTICES\];", open(os.path.join(ROOT, "oracle/iou3d_oracle.c")).read())


def test_clip_vertex_counts_stay_in_the_buffers(lib):
    cap = _capacity("oracle/iou3d_oracle.c", r"#define CLIP_MAX_VERTICES (\d+)")
    top = {}
    for name, pairs in fam.families(0).items():
        a = np.array([p[0] for p in pairs]); b = np.array([p[1] for p in pairs])
        top[name] = int(max(_max_vertices(lib, a, b).max(), _max_vertices(lib, b, a).max()))
    assert top["octagon"] == 8                        # the maximal count of exact arithmetic is reached
    # the near-duplicate search: every perturbation at once, 1e-9 .. 1e-3 rad and 1e-7 .. 1e-3 scale, 2 x 10^6 pairs
    hist = np.zeros(cap + 1, np.int64)
    for seed in range(2):
        a, b = fam.near_duplicate_batch(np.random.default_rng(100 + seed), 1_000_000)
        hist += np.bincount(_max_vertices(lib, a, b), minlength=cap + 1)[: cap + 1]
    top["near_duplicate_search"] = int(np.nonzero(hist)[0].max())
    print("largest intermediate vertex count:", top, "search histogram (4..):", hist[4:].tolist())
    assert max(top.values()) <= cap
