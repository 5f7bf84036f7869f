"""Golden vectors for the device nuScenes result rows, produced by the reference's own conversion code.

Run where the reference checkout exists:
    python tests/golden/make_golden_nusc_results.py /path/to/Det3D
The reference's _second_det_to_nusc_box, _lidar_nusc_box_to_global and cls_attr_dist
(det3d/datasets/nuscenes/nusc_common.py:46-157,222-265) and the `for det in dets:` loop of NuScenesDataset.evaluation
(det3d/datasets/nuscenes/nuscenes.py:219-262) with the `meta` it then sets (nuscenes.py:264-270) are lifted from the source with `ast` and exec'd unchanged.  pyquaternion
and the nuScenes devkit are not installed, so they run on the stand-in Quaternion and Box of oracle/nusc_results.py,
with a stub `nusc` whose get() serves synthetic calibrated_sensor / ego_pose records.  Each golden stores the packed
detections [B, D, 12], the records and tokens, the pose tables, the reference's boxes sample after sample (translation,
size, rotation, velocity, score, label, name, attribute) with their counts, and, per detection, the margin of the speed
test over oracle/nusc_results.error_bound.  The generator checks that the oracle's restatement (reference_annos) gives
the lifted code's output bit for bit.

Outputs:
  nusc_results_cases.npz  6 samples x 160 detections, nuScenes-like records (LIDAR_TOP about -90 deg about z with small
                          tilts, ego positions 300-2500 m with any yaw and small pitch / roll, two rotations a few ulps
                          off unit, one 1e-9 off): detector-like boxes over +-51.2 m, yaw at k*2pi and +-pi +-1..4 f32
                          ulps, global speeds 0.2 (1 +- 1e-6 .. 1e-3), all ten labels, invalid rows carrying NaN between
                          valid ones, an empty sample and a sample with every row valid
  nusc_results_exact.npz  identity and 180-degrees-about-z records (exact matrices) with dyadic boxes at yaw' = 0 and
                          velocities fl32(0.2), the float32 below it and 0, so every value is exact in any order.  The
                          generator checks that each of oracle.nusc_results.VARIANTS (yaw in f64, pi/2 unrounded, the
                          speed test in f32, translate before rotate, the first key as the fallback attribute) changes
                          some output by more than the bound here
Both also hold the reference's attribute for every (class, moving) pair of the nuScenes configs' class names.
"""
import ast
import operator
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import nusc_results as onr  # noqa: E402

CLASS_NAMES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle",
               "pedestrian", "traffic_cone"]


def reference_namespace(ref_root):
    path = os.path.join(ref_root, "det3d/datasets/nuscenes/nusc_common.py")
    tree = ast.parse(open(path).read())
    nodes = [n for n in tree.body if isinstance(n, ast.FunctionDef)
             and n.name in ("_second_det_to_nusc_box", "_lidar_nusc_box_to_global")]
    nodes += [n for n in tree.body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", None) == "cls_attr_dist"]
    assert len(nodes) == 3
    ns = {"np": np, "operator": operator, "Quaternion": onr.Quaternion, "Box": onr.Box}
    exec(compile(ast.Module(body=nodes, type_ignores=[]), path, "exec"), ns)
    # the per-box loop of NuScenesDataset.evaluation, as the body of a function of the names it reads
    path = os.path.join(ref_root, "det3d/datasets/nuscenes/nuscenes.py")
    cls = [n for n in ast.parse(open(path).read()).body if isinstance(n, ast.ClassDef) and n.name == "NuScenesDataset"][0]
    ev = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "evaluation"][0]
    loops = [n for n in ev.body if isinstance(n, ast.For) and getattr(n.target, "id", None) == "det"]
    meta = [n for n in ev.body if isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Subscript)
            and ast.unparse(n.targets[0]) == "nusc_annos['meta']"]
    assert len(loops) == 1 and len(meta) == 1
    fn = ast.parse("def evaluation_loop(dets, nusc, mapped_class_names, nusc_annos):\n    pass\n").body[0]
    fn.body = loops + meta                    # the loop and the meta assignment that follows it
    exec(compile(ast.fix_missing_locations(ast.Module(body=[fn], type_ignores=[])), path, "exec"), ns)
    return ns


class StubNusc:
    """nusc.get over synthetic records: sample token -> LIDAR_TOP sample_data -> calibrated_sensor / ego_pose."""

    def __init__(self, records, tokens):
        self.tables = {"sample": {}, "sample_data": {}, "calibrated_sensor": {}, "ego_pose": {}, "sensor": {}}
        for token, rec in zip(tokens, records):
            sd = "sd_" + token
            self.tables["sample"][token] = {"data": {"LIDAR_TOP": sd}}
            self.tables["sample_data"][sd] = {"calibrated_sensor_token": "cs_" + token, "ego_pose_token": "ep_" + token}
            self.tables["calibrated_sensor"]["cs_" + token] = dict(rec["calibrated_sensor"], sensor_token="lidar")
            self.tables["ego_pose"]["ep_" + token] = dict(rec["ego_pose"])
        self.tables["sensor"]["lidar"] = {"channel": "LIDAR_TOP"}

    def get(self, table, token):
        return self.tables[table][token]

    def get_sample_data_path(self, token):
        return ""


def lifted_annos(ns, packed, records, tokens):
    import torch
    dets = []
    for b, token in enumerate(tokens):
        rows = packed[b][packed[b][:, 11] > 0.5]
        dets.append(dict(box3d_lidar=torch.from_numpy(rows[:, :9].copy()), scores=torch.from_numpy(rows[:, 9].copy()),
                         label_preds=torch.from_numpy(rows[:, 10].astype(np.int64)), metadata=dict(token=token)))
    nusc_annos = {"results": {}, "meta": None}
    ns["evaluation_loop"](dets, StubNusc(records, tokens), list(CLASS_NAMES), nusc_annos)
    return nusc_annos


def quat(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(angle / 2)], axis * np.sin(angle / 2)])


def qmul(a, b):
    return onr._q_matrix(a) @ b


def nusc_like_record(rng, off_unit=0.0):
    """LIDAR_TOP about -90 deg about z with tilts of a few mrad; the ego anywhere 300-2500 m out, any yaw, small pitch
    and roll.  off_unit scales both quaternions by (1 + off_unit)."""
    cs_q = qmul(quat([0, 0, 1], -np.pi / 2 + rng.uniform(-0.02, 0.02)),
                qmul(quat([1, 0, 0], rng.uniform(-0.005, 0.005)), quat([0, 1, 0], rng.uniform(-0.005, 0.005))))
    ego_q = qmul(quat([0, 0, 1], rng.uniform(-np.pi, np.pi)),
                 qmul(quat([0, 1, 0], rng.uniform(-0.03, 0.03)), quat([1, 0, 0], rng.uniform(-0.03, 0.03))))
    r, a = rng.uniform(300, 2500), rng.uniform(-np.pi, np.pi)
    return {"calibrated_sensor": {"translation": [float(v) for v in (rng.uniform(0.9, 1.0), rng.uniform(-0.01, 0.01),
                                                                     rng.uniform(1.8, 1.9))],
                                  "rotation": [float(v) for v in cs_q * (1 + off_unit)]},
            "ego_pose": {"translation": [float(r * np.cos(a)), float(r * np.sin(a)), float(rng.uniform(-1, 1))],
                         "rotation": [float(v) for v in ego_q * (1 + off_unit)]}}


def _nudge(v, k):
    v = np.float32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf))
    return v


def detector_like(rng, n):
    b = np.zeros((n, 9), np.float32)
    b[:, 0:2] = rng.uniform(-51.2, 51.2, (n, 2))
    b[:, 2] = rng.uniform(-5, 3, n)
    b[:, 3:6] = rng.uniform([0.3, 0.3, 0.5], [3.0, 12.0, 4.0], (n, 3))
    b[:, 6:8] = rng.uniform(-15, 15, (n, 2)) * (rng.uniform(size=(n, 1)) < 0.7)
    b[:, 8] = rng.uniform(-np.pi, np.pi, n)
    return b


def angle_boxes(rng):
    out = []
    for base in [2 * np.pi * k for k in (-3, -2, -1, 0, 1, 2, 3)] + [np.pi, -np.pi]:
        for k in (-4, -3, -2, -1, 0, 1, 2, 3, 4):
            b = detector_like(rng, 1)[0]
            b[8] = _nudge(base, k)
            out.append(b)
    return np.stack(out)


def speed_boxes(rng, table, n):
    """Velocities whose global speed is 0.2 (1 + eps), eps = +-1e-6 .. 1e-3, through this sample's rotations."""
    Rc, Rp = table[0:9].reshape(3, 3), table[12:21].reshape(3, 3)
    out = []
    for i in range(n):
        b = detector_like(rng, 1)[0]
        a = rng.uniform(-np.pi, np.pi)
        d = np.array([np.cos(a), np.sin(a), 0.0])
        f = np.linalg.norm((Rp @ (Rc @ d))[:2])
        eps = [-1e-3, -1e-4, -1e-5, -1e-6, 1e-6, 1e-5, 1e-4, 1e-3][i % 8]
        m = 0.2 * (1 + eps) / f
        b[6], b[7] = m * d[0], m * d[1]
        out.append(b)
    return np.stack(out)


def pack(frames, D, rng):
    """frames: list of boxes [n_b, 9] -> packed [B, D, 12]; rows past n_b invalid, carrying NaN and garbage."""
    B = len(frames)
    packed = np.zeros((B, D, 12), np.float32)
    packed[:, :, :9] = rng.uniform(-50, 50, (B, D, 9)).astype(np.float32)
    packed[:, :, 9] = rng.uniform(0.05, 1.0, (B, D)).astype(np.float32)
    packed[:, :, 10] = (np.arange(B * D).reshape(B, D) % len(CLASS_NAMES)).astype(np.float32)
    packed[:, ::3, 0] = np.nan
    for b, f in enumerate(frames):
        packed[b, :f.shape[0], :9] = f
        packed[b, :f.shape[0], 11] = 1.0
    return packed


def to_arrays(annos, tokens):
    """-> dict of flat arrays over every box, sample after sample, and counts."""
    out = {k: [] for k in ("translation", "size", "rotation", "velocity", "score", "label", "names", "attributes")}
    counts = []
    for token in tokens:
        boxes = annos["results"][token]
        counts.append(len(boxes))
        for a in boxes:
            out["translation"].append(a["translation"])
            out["size"].append(a["size"])
            out["rotation"].append(a["rotation"])
            out["velocity"].append(a["velocity"])
            out["score"].append(a["detection_score"])
            out["label"].append(CLASS_NAMES.index(a["detection_name"]))
            out["names"].append(a["detection_name"])
            out["attributes"].append(a["attribute_name"])
    arr = {k: np.array(v, np.float64).reshape(-1, w) for k, v, w in
           ((k, out[k], w) for k, w in (("translation", 3), ("size", 3), ("rotation", 4), ("velocity", 2)))}
    arr.update(score=np.array(out["score"], np.float64), label=np.array(out["label"], np.int64),
               names=np.array(out["names"], dtype="U32"), attributes=np.array(out["attributes"], dtype="U32"),
               counts=np.array(counts, np.int32))
    return arr


def record_arrays(records):
    return {"cs_translation": np.array([r["calibrated_sensor"]["translation"] for r in records], np.float64),
            "cs_rotation": np.array([r["calibrated_sensor"]["rotation"] for r in records], np.float64),
            "ego_translation": np.array([r["ego_pose"]["translation"] for r in records], np.float64),
            "ego_rotation": np.array([r["ego_pose"]["rotation"] for r in records], np.float64)}


def _same(a, b):
    """Two nusc_annos: equal keys, order, types and values, floats bit for bit."""
    assert list(a) == list(b) and a["meta"] == b["meta"]
    assert list(a["results"]) == list(b["results"])
    for t in a["results"]:
        assert len(a["results"][t]) == len(b["results"][t]), t
        for x, y in zip(a["results"][t], b["results"][t]):
            assert list(x) == list(y), (list(x), list(y))
            for k in x:
                assert type(x[k]) is type(y[k]), k
                assert repr(x[k]) == repr(y[k]), (t, k, x[k], y[k])


def save(name, ns, packed, records, tokens, fallback):
    tables = np.stack([onr.pose_table(r) for r in records])
    annos = lifted_annos(ns, packed, records, tokens)
    _same(onr.reference_annos(packed, records, tokens, CLASS_NAMES, fallback), annos)
    margin = np.full(packed.shape[:2], np.inf)
    for b in range(packed.shape[0]):
        _bound, margin[b] = onr.error_bound(packed[b], tables[b], records[b])
    attr_still = np.array([onr.attribute(n, False, fallback) for n in CLASS_NAMES])
    attr_moving = np.array([onr.attribute(n, True, fallback) for n in CLASS_NAMES])
    payload = dict(packed=packed, tokens=np.array(tokens), tables=tables, margin=margin,
                   class_names=np.array(CLASS_NAMES), attr_still=attr_still, attr_moving=attr_moving,
                   **record_arrays(records), **to_arrays(annos, tokens))
    np.savez_compressed(os.path.join(HERE, name), **payload)
    return payload, annos


def exact_record(cs_flip, ego_flip, tc, tp):
    q = lambda flip: [0.0, 0.0, 0.0, 1.0] if flip else [1.0, 0.0, 0.0, 0.0]       # noqa: E731
    return {"calibrated_sensor": {"translation": list(tc), "rotation": q(cs_flip)},
            "ego_pose": {"translation": list(tp), "rotation": q(ego_flip)}}


def exact_boxes():
    """Dyadic boxes at r = -fl32(pi/2), so yaw' = 0 and every value is exact; velocities fl32(0.2), the float32 below
    it and 0 along each axis; all ten labels."""
    f02, below = np.float32(0.2), np.nextafter(np.float32(0.2), np.float32(0))
    out = []
    k = 0
    for vx, vy in ((f02, 0), (0, f02), (-f02, 0), (below, 0), (0, -below), (0, 0)):
        for x in (-32.5, 0.25, 16.0, 40.75):
            out.append([x, -x / 2, 1.5 - (k % 3), 1.75, 4.5, 1.5, vx, vy, -HALF_PI_F32])
            k += 1
    return np.array(out, np.float32)


HALF_PI_F32 = np.float32(np.pi / 2)


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: make_golden_nusc_results.py /path/to/Det3D")
    ns = reference_namespace(sys.argv[1])
    fallback = onr.most_frequent(ns["cls_attr_dist"])
    rng = np.random.default_rng(47)
    D = 160

    records = [nusc_like_record(rng) for _ in range(6)]
    records[1] = nusc_like_record(rng, off_unit=3e-15)
    records[4] = nusc_like_record(rng, off_unit=4e-15)
    records[5] = nusc_like_record(rng, off_unit=1e-9)
    tokens = ["%032x" % int(rng.integers(0, 2 ** 62)) for _ in range(6)]
    tables = [onr.pose_table(r) for r in records]
    frames = [detector_like(rng, 150), angle_boxes(rng), speed_boxes(rng, tables[2], 96), np.zeros((0, 9), np.float32),
              np.concatenate([detector_like(rng, D - 40), speed_boxes(rng, tables[4], 40)]), detector_like(rng, 80)]
    packed = pack(frames, D, rng)
    packed[0, 10:150:7, 11] = 0.0                         # invalid rows between valid ones (they carry NaN too)
    packed[0, 10:150:7, 0] = np.nan
    packed[:, :, 10] = np.where(packed[:, :, 11] > 0.5, rng.integers(0, 10, packed.shape[:2]), packed[:, :, 10])
    p, _annos = save("nusc_results_cases.npz", ns, packed, records, tokens, fallback)
    valid = packed[..., 11] > 0.5
    assert np.all(p["margin"][valid] > 1), "a speed decision inside the error bound"
    assert set(p["label"].tolist()) == set(range(10))
    print("cases: boxes per sample", p["counts"].tolist(), "; smallest speed margin", float(p["margin"][valid].min()))

    records = [exact_record(False, False, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)),
               exact_record(False, True, (1.5, -0.25, 2.0), (1024.5, -768.25, 0.5)),
               exact_record(True, False, (0.75, 0.5, 1.75), (-2048.0, 512.5, -1.0)),
               exact_record(True, True, (1.0, 0.0, 1.875), (300.25, 2400.5, 0.125))]
    tokens = ["exact%d" % b for b in range(4)]
    boxes = exact_boxes()
    packed = pack([boxes] * 4, boxes.shape[0] + 8, rng)
    packed[:, :boxes.shape[0], 10] = (np.arange(boxes.shape[0]) % 10)[None]
    p, _annos = save("nusc_results_exact.npz", ns, packed, records, tokens, fallback)
    changed = {}
    for v in onr.VARIANTS:
        n = 0
        for b in range(4):
            rows, attrs = onr.variant_output(packed[b], p["tables"][b], CLASS_NAMES, fallback, None)
            vrows, vattrs = onr.variant_output(packed[b], p["tables"][b], CLASS_NAMES, fallback, v)
            bound, _m = onr.error_bound(packed[b], p["tables"][b])
            keep = packed[b][:, 11] > 0.5
            with np.errstate(invalid="ignore"):
                far = np.abs(vrows - rows) > bound
            n += int(far[keep].any(1).sum()) + sum(x != y for x, y, k in zip(attrs, vattrs, keep) if k)
        changed[v] = n
        assert n >= 1, (v, n)
    print("exact: boxes per sample", p["counts"].tolist(), "; outputs each variant changes:", changed)


if __name__ == "__main__":
    main()
