"""The deployed rotated NMS (D3B_BOX_XYWLR, rotate_nms_cc semantics) against exact polygon geometry.

* The mode-2 IoU matrix of d3b_boxes_iou_bev -- the same device function that makes the NMS decisions -- against
  oracle/exact_polygon.py on host corners built in the device's fp32 operation order.  At r = 0 the corners are exact
  and the device must give fl32(exact) to 1 ulp.  Elsewhere host and device sin / cos may differ by 2 ulps; each corner
  then moves by at most delta (2-ulp sin / cos difference plus one rounding of every step of the corner), and
  |device - exact| <= 2 (P_a + P_b) delta / union + 1 ulp, P the perimeters.
* The keep list of d3b_rotate_nms equals a host greedy sweep over the device's own mode-2 matrix, bit for bit.
* The keep list equals the greedy sweep over the EXACT IoUs at thresholds 0 ... 1, where a deciding pair whose exact
  IoU lies within the bound of the threshold is counted and resolved with the device's value (reported; expected 0 on
  detector-like clusters)."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import exact_polygon as ep
import rotated_box_families as fam

pytestmark = pytest.mark.gpu


def _iou_matrix(a, b):
    from det3d_b200 import _lib
    from det3d_b200.ops.nms import nms_ops
    return nms_ops.boxes_iou_bev(torch.from_numpy(np.ascontiguousarray(a)).cuda(),
                                 torch.from_numpy(np.ascontiguousarray(b)).cuda(), mode=_lib.IOU_BEV_XYWLR).cpu().numpy()


def _device_keep(boxes, thr, max_keep=None, n_dev=None):
    from det3d_b200 import _lib
    from det3d_b200.ops.nms import nms_ops
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device="cuda")
    keep_idx, keep_count = nms_ops.nms_sorted(torch.from_numpy(boxes).cuda(), _lib.BOX_XYWLR, thr, max_keep, n_dev=nd)
    return keep_idx[: int(keep_count)].cpu().numpy()


def _ulp(v):
    return float(np.spacing(np.float32(abs(v))))


def corner_delta(box):
    """Bound on how far any fp32 corner of the device can lie from the host's (xywlr_corners_f32): 0 at r = 0, where
    sinf / cosf are exact on both; else a 2-ulp difference of sin and cos times the half extents, plus one ulp of every
    rounded intermediate (both products, their sum, the coordinate)."""
    cx, cy, w, l, r = (np.float32(v) for v in box)
    if r == 0:
        return 0.0
    s, c = np.float32(math.sin(float(r))), np.float32(math.cos(float(r)))
    xs, ys = ep.xywlr_corners_f32(box)
    worst = 0.0
    for k in range(4):
        px, py = float(w) * (-0.5 if k < 2 else 0.5), float(l) * (-0.5 if k in (0, 3) else 0.5)
        dx = abs(px) * 2 * _ulp(c) + abs(py) * 2 * _ulp(s) + _ulp(px * c) + _ulp(py * s) + _ulp(px * c + py * s) + _ulp(xs[k])
        dy = abs(px) * 2 * _ulp(s) + abs(py) * 2 * _ulp(c) + _ulp(px * s) + _ulp(py * c) + _ulp(py * c - px * s) + _ulp(ys[k])
        worst = max(worst, math.hypot(dx, dy))
    return worst


def _perimeter(q):
    xs, ys = q
    return sum(math.hypot(float(xs[(k + 1) % 4]) - float(xs[k]), float(ys[(k + 1) % 4]) - float(ys[k])) for k in range(4))


class Exact:
    """Exact IoU and its bound for pairs of a box set, computed once per pair."""

    def __init__(self, boxes):
        self.boxes = boxes
        self.q = [ep.xywlr_corners_f32(b) for b in boxes]
        self.delta = [corner_delta(b) for b in boxes]
        self.cache = {}

    def pair(self, i, j):
        key = (i, j)
        if key not in self.cache:
            qa, qb = self.q[i], self.q[j]
            iou, union = ep.rotate_iou(qa, qb)
            d = max(self.delta[i], self.delta[j])
            if union is None:
                union_f = float(ep.quad_area(qa) + ep.quad_area(qb))
            else:
                union_f = float(union)
            geo = 2 * (_perimeter(qa) + _perimeter(qb)) * d / union_f if d > 0 else 0.0
            self.cache[key] = (iou, geo)
        return self.cache[key]


def _bound(iou, geo):
    return geo + _ulp(0.0 if iou is None else float(iou))


# ------------------------------------------------------------------------------------ the mode-2 matrix, exactly
@pytest.mark.parametrize("name", sorted(fam.families(1)))
def test_mode2_matrix_against_exact_geometry(name):
    pairs = fam.families(1)[name]
    a = np.array([p[0] for p in pairs], np.float32)
    b = np.array([p[1] for p in pairs], np.float32)
    boxes = np.concatenate([a, b])
    ex = Exact(boxes)
    n = len(pairs)
    m_ab, m_ba = np.diag(_iou_matrix(a, b)), np.diag(_iou_matrix(b, a))
    worst_ratio, worst_ulp_r0, n_r0, n_rot = 0.0, 0, 0, 0
    for k in range(n):
        for i, j, got in ((k, n + k, m_ab[k]), (n + k, k, m_ba[k])):
            iou, geo = ex.pair(i, j)
            want = np.float32(0) if iou is None else ep.to_f32(iou)
            if geo == 0.0:
                n_r0 += 1
                d = abs(int(np.float32(got).view(np.int32)) - int(want.view(np.int32)))
                worst_ulp_r0 = max(worst_ulp_r0, d)
                assert d <= 1, (name, boxes[i], boxes[j], float(got), iou)
            else:
                n_rot += 1
                err = abs(Fraction(float(got)) - (iou or 0))
                bound = _bound(iou, geo)
                worst_ratio = max(worst_ratio, float(err) / bound)
                assert err <= Fraction(bound), (name, boxes[i], boxes[j], float(got), float(iou or 0), bound)
    print("%s: %d pairs at r = 0 (worst %d ulp), %d rotated pairs (worst ratio to the bound %.3g)"
          % (name, n_r0, worst_ulp_r0, n_rot, worst_ratio))


def test_mode2_exact_cases_and_inclusive_threshold():
    """r = 0: the IoU of exactly 0.5 suppresses at threshold 0.5 (inclusive); a shared edge, a shared corner and
    separated polygons with overlapping hulls are never suppressed, not even at threshold 0."""
    for a, b, want in fam.exact_r0():
        got = _iou_matrix(a[None], b[None])[0, 0]
        assert got == (np.float32(0) if want is None else ep.to_f32(want)), (a, b, got, want)
        for thr in (0.0, 0.5, 1.0):
            suppressed = want is not None and want >= Fraction(thr)
            keep = _device_keep(np.stack([a, b]), thr)
            assert keep.tolist() == ([0] if suppressed else [0, 1]), (a, b, thr)
    for a, b in fam.diamonds(np.random.default_rng(3), 16):
        assert _iou_matrix(a[None], b[None])[0, 0] == 0
        assert _device_keep(np.stack([a, b]), 0.0).tolist() == [0, 1]


def test_iou_bev_rejects_an_unknown_mode():
    from det3d_b200 import _lib
    from det3d_b200.ops.nms import nms_ops
    x = torch.zeros((2, 5), device="cuda")
    with pytest.raises(_lib.D3BError):
        nms_ops.boxes_iou_bev(x, x, mode=3)


# ------------------------------------------------------------------------------ sweep over the device's own matrix
def greedy(n, suppress, max_keep=None):
    """Greedy NMS over boxes in score order: keep i unless removed; then remove every later j that suppress(i, j)."""
    removed = np.zeros(n, bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        if max_keep is not None and len(keep) == max_keep:
            break
        for j in range(i + 1, n):
            if not removed[j] and suppress(i, j):
                removed[j] = True
    return np.array(keep, np.int64)


def _matrix_greedy(m, thr, n=None, max_keep=None):
    n = m.shape[0] if n is None else n
    sup = (m > 0) & (m >= np.float32(thr))       # 0 = skipped by a gate: never suppresses, not even at threshold 0
    sup = np.triu(sup[:n, :n], 1)
    removed = np.zeros(n, bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        if max_keep is not None and len(keep) == max_keep:
            break
        removed |= sup[i]
    return np.array(keep, np.int64)


@pytest.mark.parametrize("n", [1000, 1500, 4097])
def test_sweep_equals_greedy_over_the_device_matrix(n):
    boxes = fam.detector_clusters(7, n)
    m = _iou_matrix(boxes, boxes)
    assert int(((m > 0) & (m < 1)).sum()) > 20 * n           # dense clusters: many deciding pairs
    for thr in (0.0, 0.01, 0.2, 0.5):
        want = _matrix_greedy(m, thr)
        assert np.array_equal(_device_keep(boxes, thr), want), (n, thr)
        assert np.array_equal(_device_keep(boxes, thr, max_keep=max(1, len(want) // 3)), want[: max(1, len(want) // 3)])
        n_live = n - 223
        assert np.array_equal(_device_keep(boxes, thr, n_dev=n_live), _matrix_greedy(m, thr, n=n_live)), (n, thr)
        assert np.array_equal(_device_keep(boxes, thr, max_keep=5, n_dev=n_live), _matrix_greedy(m, thr, n=n_live, max_keep=5))


# ----------------------------------------------------------------------------------- decisions against geometry
def _exact_sweep(ex, m, thr, same_group):
    """Greedy over the exact IoUs; a deciding pair whose exact IoU lies within the bound of thr is ambiguous: counted
    and resolved with the device's mode-2 value."""
    t = Fraction(float(np.float32(thr)))
    counts = {"deciding": 0, "ambiguous": 0}

    def suppress(i, j):
        if not same_group(i, j):
            return False
        iou, geo = ex.pair(i, j)
        counts["deciding"] += 1
        if iou is None:
            return False
        slack = Fraction(geo) + iou * Fraction(1, 2 ** 40)            # the device's fp64 rounding, far below 1 ulp
        lo, hi = ep.to_f32(max(iou - slack, Fraction(0))), ep.to_f32(iou + slack)
        if (Fraction(float(lo)) >= t) != (Fraction(float(hi)) >= t):
            counts["ambiguous"] += 1
            return bool(m[i, j] > 0 and m[i, j] >= np.float32(thr))
        return Fraction(float(hi)) >= t

    return greedy(len(ex.boxes), suppress), counts


def test_decisions_against_exact_geometry_on_the_families():
    groups = [[a, b] for pairs in fam.families(2, n=32).values() for a, b in pairs]
    boxes, gid = fam.on_grid(groups)
    m = _iou_matrix(boxes, boxes)
    assert not (m[gid[:, None] != gid[None, :]] != 0).any()           # the grid separates the groups
    ex = Exact(boxes)
    report = {}
    for thr in (0.0, 0.01, 0.2, 0.5, 1.0):
        want, counts = _exact_sweep(ex, m, thr, lambda i, j: gid[i] == gid[j])
        assert np.array_equal(_device_keep(boxes, thr), want), thr
        report[thr] = counts
    print("families on a 20 m grid, %d boxes: %s" % (len(boxes), report))


@pytest.mark.parametrize("seed", [11, 12])
def test_decisions_against_exact_geometry_on_detector_clusters(seed):
    boxes = fam.detector_clusters(seed, 1000)
    m = _iou_matrix(boxes, boxes)
    cluster = np.arange(len(boxes)) // 100
    assert not (m[cluster[:, None] != cluster[None, :]] != 0).any()
    ex = Exact(boxes)
    report = {}
    for thr in (0.01, 0.2, 0.5):
        want, counts = _exact_sweep(ex, m, thr, lambda i, j: cluster[i] == cluster[j])
        assert np.array_equal(_device_keep(boxes, thr), want), thr
        report[thr] = counts
    print("detector clusters (seed %d): %s" % (seed, report))
