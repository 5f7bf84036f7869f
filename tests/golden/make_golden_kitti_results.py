"""Golden vectors for the device KITTI result rows, produced by the reference's own functions.

Run where the reference checkout exists:
    python tests/golden/make_golden_kitti_results.py /path/to/Det3D
The reference's functions on the path of KittiDataset.convert_detection_to_kitti_annos -- limit_period, lidar_to_camera,
box_lidar_to_camera, corners_nd, rotation_3d_in_axis, center_to_corner_box3d, project_to_image
(det3d/core/bbox/box_np_ops.py:267-297,358-391,453-474,572-573,900-906,917-922,933-938), get_start_result_anno and
empty_result_anno (datasets/kitti/kitti_common.py:935-969) and the method itself (datasets/kitti/kitti.py:78-158) -- are
lifted from the source with `ast` and exec'd unchanged, their decorators included, with a stub `spconv` module in place;
the method runs on a stand-in `self` holding the class names and one info per frame.  Each golden stores the packed
detections [B, D, nd + 3] (box, score, label, valid), the calibrations, the reference's kept rows (bbox, alpha,
dimensions, location, rotation_y, score, label) frame after frame with their counts and names, and, per detection,
the margin of its keep / drop tests to the image bounds over oracle/kitti_results.error_bound.

Outputs:
  kitti_results_cases.npz  nd = 7, 8 frames x 160 detections, KITTI-like calibrations: detector-like boxes in and around
                           the frustum, boxes whose image box touches each image edge (f32 ulp neighbours of the
                           crossing), boxes partly and wholly behind the camera, yaw at k*2pi and +-pi +-1..4 f32 ulps,
                           NaN / +-inf in every box column, a frame with no valid detection, a frame where every box
                           is filtered, and a frame with every row valid
  kitti_results_nd9.npz    nd = 9 (x, y, z, w, l, h, vx, vy, r), 2 frames: the reference wraps the LAST column and reads
                           column 6 as the yaw, and the kernel does the same
  kitti_results_exact.npz  power-of-two / small-integer calibrations and dyadic boxes at yaw 0, so every reference value
                           is exact whatever order a sum is taken in: image boxes exactly on W, H and 0, boxes behind the
                           camera, a P2 translation that moves boxes across the edges.  The generator checks that each of
                           oracle.kitti_results.VARIANTS (>= for >, ones for the zeros column, clipping before the test,
                           clipping to (H, W)) changes some kept set or value here
"""
import ast
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from det3d_b200.utils.synthetic import KITTI_IMAGE_SHAPES, kitti_like_calib  # noqa: E402
from oracle import kitti_results as okr  # noqa: E402

BOX_NP_OPS = ("limit_period", "lidar_to_camera", "box_lidar_to_camera", "corners_nd", "rotation_3d_in_axis",
              "center_to_corner_box3d", "project_to_image")
KITTI_COMMON = ("get_start_result_anno", "empty_result_anno")
CLASS_NAMES = ["Car", "Pedestrian", "Cyclist"]


def _lift(path, names, ns, cls=None):
    tree = ast.parse(open(path).read())
    body = tree.body
    if cls is not None:
        body = [n for n in body if isinstance(n, ast.ClassDef) and n.name == cls][0].body
    nodes = [n for n in body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in nodes) == sorted(names), [n.name for n in nodes]
    exec(compile(ast.Module(body=nodes, type_ignores=[]), path, "exec"), ns)


def reference_namespace(ref_root):
    import numba

    sys.modules.setdefault("spconv", types.ModuleType("spconv"))
    ns = {"np": np, "numba": numba}
    _lift(os.path.join(ref_root, "det3d/core/bbox/box_np_ops.py"), BOX_NP_OPS, ns)
    _lift(os.path.join(ref_root, "det3d/datasets/kitti/kitti_common.py"), KITTI_COMMON, ns)
    ns["box_np_ops"] = types.SimpleNamespace(**{k: ns[k] for k in BOX_NP_OPS})
    _lift(os.path.join(ref_root, "det3d/datasets/kitti/kitti.py"), ("convert_detection_to_kitti_annos",), ns,
          cls="KittiDataset")
    return ns


def reference_annos(ns, packed, nd, calibs):
    """The reference's convert_detection_to_kitti_annos on packed [B, D, nd + 3] (valid rows in order)."""
    import torch

    infos, detection = [], {}
    for b, cal in enumerate(calibs):
        infos.append(dict(image=dict(image_idx=b, image_shape=cal["image_shape"]),
                          calib=dict(R0_rect=cal["rect"], Tr_velo_to_cam=cal["Trv2c"], P2=cal["P2"])))
        rows = packed[b][packed[b][:, nd + 2] > 0.5]
        detection[str(b)] = dict(box3d_lidar=torch.from_numpy(rows[:, :nd].copy()),
                                 scores=torch.from_numpy(rows[:, nd].copy()),
                                 label_preds=torch.from_numpy(rows[:, nd + 1].astype(np.int64)), metadata=dict(idx=b))
    self = types.SimpleNamespace(_class_names=CLASS_NAMES, _kitti_infos=infos)
    return ns["convert_detection_to_kitti_annos"](self, detection)


def annos_to_rows(annos):
    """-> rows f64 [total, 14] (bbox, alpha, dims, loc, ry, score, label), counts [B], names [total]."""
    rows, counts, names = [], [], []
    for a in annos:
        n = a["name"].shape[0]
        counts.append(n)
        if n == 0:
            continue
        label = np.array([CLASS_NAMES.index(s) for s in a["name"]], np.float64)
        rows.append(np.concatenate([a["bbox"], a["alpha"][:, None], a["dimensions"], a["location"],
                                    a["rotation_y"][:, None], a["score"].astype(np.float64)[:, None], label[:, None]],
                                   1))
        names += list(a["name"])
    rows = np.concatenate(rows) if rows else np.zeros((0, okr.COLS))
    return rows, np.array(counts, np.int32), np.array(names)


def _nudge(v, k):
    v = np.float32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf))
    return v


def _box(x, y, z, w, l, h, r):
    return np.array([x, y, z, w, l, h, r], np.float32)


def detector_like(rng, n):
    return np.stack([_box(rng.uniform(0, 70), rng.uniform(-40, 40), rng.uniform(-3, 1), rng.uniform(1.4, 2.0),
                          rng.uniform(3, 5), rng.uniform(1.3, 1.8), rng.uniform(-np.pi, np.pi)) for _ in range(n)])


def edge_boxes(rng, table, n_per_edge=6):
    """Boxes whose image box crosses each edge: bisect the lateral (y) or vertical (z) position against the oracle's
    bbox, then take the crossing's f32 ulp neighbours."""
    out = []
    H, W = table[28], table[29]

    def bbox_of(b):
        det = np.concatenate([b, [0.9, 0, 1]]).astype(np.float32)[None]
        _rows, _keep, a = okr.kernel_order(det, 7, table)
        return a["u"].min(), a["v"].min(), a["u"].max(), a["v"].max()

    edges = [(1, 0, W), (1, 2, 0.0), (2, 1, H), (2, 3, 0.0)]      # (box column moved, bbox index, image bound)
    for col, bi, bound in edges:
        for _ in range(n_per_edge):
            b = detector_like(rng, 1)[0]
            b[0] = rng.uniform(5, 40)
            lo, hi = (-80.0, 80.0) if col == 1 else (-30.0, 30.0)
            f = lambda t: bbox_of(np.concatenate([b[:col], [t], b[col + 1:]]))[bi] - bound   # noqa: E731
            flo, fhi = f(lo), f(hi)
            if np.sign(flo) == np.sign(fhi):
                continue
            for _ in range(80):
                mid = 0.5 * (lo + hi)
                if np.sign(f(mid)) == np.sign(flo):
                    lo = mid
                else:
                    hi = mid
            for k in (-3, -1, 0, 1, 3):
                q = b.copy()
                q[col] = _nudge(lo, k)
                out.append(q)
    return np.stack(out)


def behind_camera(rng, n):
    return np.stack([_box(rng.uniform(-30, 1.0), rng.uniform(-20, 20), rng.uniform(-2, 1), rng.uniform(1.4, 2.0),
                          rng.uniform(3, 5), rng.uniform(1.3, 1.8), rng.uniform(-np.pi, np.pi)) for _ in range(n)])


def angle_boxes(rng):
    out = []
    for base in [2 * np.pi * k for k in (-3, -2, -1, 0, 1, 2, 3)] + [np.pi, -np.pi, 0.5 * np.pi, -1.5 * np.pi]:
        for k in (-4, -3, -2, -1, 0, 1, 2, 3, 4):
            b = detector_like(rng, 1)[0]
            b[0], b[1] = rng.uniform(8, 30), rng.uniform(-5, 5)
            b[6] = _nudge(base, k)
            out.append(b)
    return np.stack(out)


def special_boxes(rng):
    out = []
    for col in range(7):
        for v in (np.nan, np.inf, -np.inf):
            b = detector_like(rng, 1)[0]
            b[0], b[1] = rng.uniform(8, 30), rng.uniform(-5, 5)
            b[col] = v
            out.append(b)
    return np.stack(out)


def pack_frames(frames, D, nd, rng):
    """frames: list of boxes [n_b, nd] -> packed [B, D, nd + 3]; rows past n_b invalid (garbage boxes)."""
    B = len(frames)
    packed = np.zeros((B, D, nd + 3), np.float32)
    packed[:, :, :nd] = rng.uniform(-50, 50, (B, D, nd)).astype(np.float32)
    packed[:, :, nd] = rng.uniform(0.05, 1.0, (B, D)).astype(np.float32)
    packed[:, :, nd + 1] = rng.integers(0, len(CLASS_NAMES), (B, D)).astype(np.float32)
    for b, f in enumerate(frames):
        assert f.shape[0] <= D
        packed[b, :f.shape[0], :nd] = f
        packed[b, :f.shape[0], nd + 2] = 1.0
    return packed


def margins(packed, nd, tables):
    out = np.full(packed.shape[:2], np.inf)
    for b in range(packed.shape[0]):
        _bound, m = okr.error_bound(packed[b], nd, tables[b])
        out[b] = m
    return out


def save(name, packed, nd, calibs, ns, extra=None):
    annos = reference_annos(ns, packed, nd, calibs)
    rows, counts, names = annos_to_rows(annos)
    tables = np.stack([okr.calib_table(c["rect"], c["Trv2c"], c["P2"], c["image_shape"]) for c in calibs])
    # the oracle's restatement of the reference is the reference, bit for bit
    for b, (a, cal) in enumerate(zip(annos, calibs)):
        mine = okr.reference_annos(packed[b], nd, cal, CLASS_NAMES)
        for k in ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score"):
            assert mine[k].dtype == a[k].dtype and mine[k].shape == a[k].shape, (name, b, k)
            if mine[k].dtype.kind == "f":
                assert np.array_equal(mine[k].view(np.uint64 if mine[k].itemsize == 8 else np.uint32),
                                      a[k].view(np.uint64 if a[k].itemsize == 8 else np.uint32)), (name, b, k)
            else:
                assert np.array_equal(mine[k], a[k]), (name, b, k)
    payload = dict(packed=packed, nd=np.int32(nd), rect=np.stack([c["rect"] for c in calibs]),
                   Trv2c=np.stack([c["Trv2c"] for c in calibs]), P2=np.stack([c["P2"] for c in calibs]),
                   image_shape=np.stack([c["image_shape"] for c in calibs]), tables=tables, rows=rows, counts=counts,
                   names=names, class_names=np.array(CLASS_NAMES), margin=margins(packed, nd, tables))
    payload.update(extra or {})
    np.savez_compressed(os.path.join(HERE, name), **payload)
    return payload


def exact_calib(tx):
    """rect = I, Trv2c the velodyne -> camera axis permutation with a dyadic translation, P2 = K [I | t] with K of
    powers of two: every value of the conversion is a small dyadic rational."""
    P2 = np.eye(4)
    P2[:3, :3] = [[512.0, 0, 256.0], [0, 512.0, 128.0], [0, 0, 1.0]]
    P2[:3, 3] = [tx, 0.0, 0.0]
    Trv2c = np.eye(4)
    Trv2c[:3, :3] = [[0, -1.0, 0], [0, 0, -1.0], [1.0, 0, 0]]
    Trv2c[:3, 3] = [0.0, 0.0, 0.0]
    return dict(rect=np.eye(4), Trv2c=Trv2c, P2=P2, image_shape=np.array((256, 512), np.int64))


def exact_boxes():
    """Yaw 0, camera depth of every corner a power of two (x = 6, l = 4 -> corners at depth 4 and 8; x = -6 behind).
    With f = 512, c = (256, 128): u = 512 * X_cam / depth + 256, v = 512 * Y_cam / depth + 128, X_cam = -y, Y_cam = -z.
    The lateral / vertical positions put the box's image extremes on 0, W = 512, H = 256 and around them."""
    out = []
    w, l, h = 2.0, 4.0, 2.0
    for x in (6.0, -6.0, 12.0):
        # corners at depth x +- l/2: the extreme u is at the nearer (smaller |depth|) corner
        for y in np.arange(-9.0, 9.01, 0.25):
            out.append(_box(x, y, 0.0, w, l, h, 0.0))
        for z in np.arange(-5.0, 5.01, 0.25):
            out.append(_box(x, 0.0, z, w, l, h, 0.0))
    return np.stack(out)


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: make_golden_kitti_results.py /path/to/Det3D")
    ref_root = sys.argv[1]
    ns = reference_namespace(ref_root)
    rng = np.random.default_rng(31)
    D = 160

    calibs = [kitti_like_calib(40 + i, KITTI_IMAGE_SHAPES[i % 4]) for i in range(8)]
    calibs[0] = kitti_like_calib(0, KITTI_IMAGE_SHAPES[0], perturb=False)
    tables = [okr.calib_table(c["rect"], c["Trv2c"], c["P2"], c["image_shape"]) for c in calibs]
    edges = edge_boxes(rng, tables[1])
    frames = [detector_like(rng, 150), edges[:D], behind_camera(rng, 120), angle_boxes(rng),
              special_boxes(rng), np.zeros((0, 7), np.float32),
              np.stack([_box(10, s * rng.uniform(150, 300), 0, 1.6, 4, 1.5, 0.3) for s in (-1, 1) * 20]),
              np.concatenate([detector_like(rng, 100), behind_camera(rng, 60)])]
    packed = pack_frames(frames, D, 7, rng)
    packed[0, 10:150:7, 9] = 0.0                               # invalid rows between valid ones
    p = save("kitti_results_cases.npz", packed, 7, calibs, ns)
    print("cases: kept per frame", p["counts"].tolist(), "of", [int((f[:, 9] > 0.5).sum()) for f in packed],
          "; detections with a decision margin < 1 bound:", int((p["margin"] < 1).sum()))

    frames9 = []
    for _ in range(2):
        f = detector_like(rng, 90)
        f9 = np.zeros((90, 9), np.float32)
        f9[:, :6] = f[:, :6]
        f9[:, 6:8] = rng.uniform(-10, 10, (90, 2))
        f9[:, 8] = rng.uniform(-8, 8, 90)
        frames9.append(f9)
    p = save("kitti_results_nd9.npz", pack_frames(frames9, 100, 9, rng), 9, calibs[:2], ns)
    print("nd9: kept", p["counts"].tolist())

    calibs = [exact_calib(0.0), exact_calib(1024.0), exact_calib(-2048.0)]
    boxes = exact_boxes()
    packed = pack_frames([boxes] * 3, boxes.shape[0], 7, rng)
    p = save("kitti_results_exact.npz", packed, 7, calibs, ns)
    tables = p["tables"]
    changed = {}
    for v in okr.VARIANTS:
        n = 0
        for b in range(3):
            rows, keep, _a = okr.kernel_order(packed[b], 7, tables[b])
            vrows, vkeep = okr.variant_rows(packed[b], 7, tables[b], v)
            n += int((keep != vkeep).sum()) + int((~np.all(rows[keep & vkeep, :4] == vrows[keep & vkeep, :4], 1)).sum())
        changed[v] = n
        assert n >= 2, (v, n)
    on_edge = 0
    for b in range(3):
        rows, keep, a = okr.kernel_order(packed[b], 7, tables[b])
        H, W = tables[b][28], tables[b][29]
        on_edge += int(((a["u"].min(1) == W) | (a["v"].min(1) == H) | (a["u"].max(1) == 0)
                        | (a["v"].max(1) == 0)).sum())
    assert on_edge >= 4, on_edge
    print("exact: kept", p["counts"].tolist(), "; image boxes exactly on an edge:", on_edge,
          "; outcomes each variant changes:", changed)


if __name__ == "__main__":
    main()
