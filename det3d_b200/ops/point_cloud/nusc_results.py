"""Device nuScenes result rows: torch wrapper over d3b_nusc_results_dev (csrc/nusc_results.cu).

Reference semantics: det3d/datasets/nuscenes/nuscenes.py:180-274 (NuScenesDataset.evaluation) with
nusc_common.py:222-265 (_second_det_to_nusc_box, _lidar_nusc_box_to_global) and nusc_common.py:46-157 (cls_attr_dist).
The per-box conversion to the global frame runs on the device; `pose_table` (numpy, once per pose record) and
`to_nusc_annos` (the reference's submission dict from the rows) run on the host.
"""
import numpy as np
import torch

from ... import _lib

MAX_BATCH = 64
POSE_DOUBLES = 32         # Rc 9, tc 3, Rp 9, tp 3, qc 4, qp 4
COLS = 15                 # translation 3, size 3, rotation 4, velocity 2, score, label, moving
ND = 9                    # x, y, z, w, l, h, vx, vy, r
ANNO_KEYS = ("sample_token", "translation", "size", "rotation", "velocity", "detection_name", "detection_score",
             "attribute_name")
META = {"use_camera": False, "use_lidar": True, "use_radar": False, "use_map": False, "use_external": False}

# The attribute of a box by (class, moving), nuscenes.py:219-259.  Moving: vehicles -> vehicle.moving, cycles ->
# cycle.with_rider; still: pedestrian -> pedestrian.standing, bus -> vehicle.stopped.  Every other pair takes the
# class's most frequent attribute in cls_attr_dist (nusc_common.py:46-157; max() keeps the first key on a tie, and
# barrier's and traffic_cone's counts are all zero, so theirs is the first key, cycle.with_rider).
_MOVING = dict.fromkeys(("car", "construction_vehicle", "bus", "truck", "trailer"), "vehicle.moving")
_MOVING.update(dict.fromkeys(("bicycle", "motorcycle"), "cycle.with_rider"))
_STILL = {"pedestrian": "pedestrian.standing", "bus": "vehicle.stopped"}
MOST_FREQUENT_ATTRIBUTE = {
    "barrier": "cycle.with_rider", "bicycle": "cycle.without_rider", "bus": "vehicle.moving", "car": "vehicle.parked",
    "construction_vehicle": "vehicle.parked", "ignore": "vehicle.parked", "motorcycle": "cycle.without_rider",
    "pedestrian": "pedestrian.moving", "traffic_cone": "cycle.with_rider", "trailer": "vehicle.parked",
    "truck": "vehicle.parked",
}


def attribute_table(class_names):
    """[(attribute when still, attribute when moving)] per label.  ValueError for a class name cls_attr_dist does not
    hold (the reference raises KeyError when it meets such a box)."""
    table = []
    for name in class_names:
        if name not in MOST_FREQUENT_ATTRIBUTE:
            raise ValueError("class %r has no nuScenes attribute (known: %s)" % (name, sorted(MOST_FREQUENT_ATTRIBUTE)))
        fallback = MOST_FREQUENT_ATTRIBUTE[name]
        table.append((_STILL.get(name, fallback), _MOVING.get(name, fallback)))
    return table


def _unit_quaternion(q, what):
    """pyquaternion's _normalise as rotation_matrix runs it: q / sqrt(q . q) unless |1 - q . q| < 1e-14."""
    q = np.array(q, np.float64).reshape(-1)
    if q.shape != (4,) or not np.all(np.isfinite(q)):
        raise ValueError("%s: rotation must be 4 finite numbers (w, x, y, z), got %r" % (what, q))
    ss = np.dot(q, q)
    if abs(np.sqrt(ss) - 1.0) > 1e-6:
        raise ValueError("%s: rotation norm %r is not 1" % (what, float(np.sqrt(ss))))
    if not abs(1.0 - ss) < 1e-14:
        q = q / np.sqrt(ss)
    return q


def _q_matrix(q):
    return np.array([[q[0], -q[1], -q[2], -q[3]], [q[1], q[0], -q[3], q[2]],
                     [q[2], q[3], q[0], -q[1]], [q[3], -q[2], q[1], q[0]]])


def _q_bar_matrix(q):
    return np.array([[q[0], -q[1], -q[2], -q[3]], [q[1], q[0], q[3], -q[2]],
                     [q[2], -q[3], q[0], q[1]], [q[3], q[2], -q[1], q[0]]])


def rotation_matrix(q):
    """pyquaternion's rotation_matrix of a unit q: (_q_matrix @ _q_bar_matrix.conj().T)[1:, 1:], by numpy's dot."""
    return np.dot(_q_matrix(q), _q_bar_matrix(q).conj().transpose())[1:][:, 1:]


def _translation(t, what):
    t = np.array(t, np.float64).reshape(-1)
    if t.shape != (3,) or not np.all(np.isfinite(t)):
        raise ValueError("%s: translation must be 3 finite numbers, got %r" % (what, t))
    return t


def pose_table(record):
    """float64 [32], the kernel's pose row of one sample: record = dict(calibrated_sensor=dict(translation, rotation),
    ego_pose=dict(translation, rotation)), the key frame's records as nusc.get returns them (other keys are ignored).
    Each rotation is normalised and turned into a matrix as pyquaternion's rotation_matrix does (restated, not
    imported), so the matrices are the bits Box.rotate multiplies by.  ValueError on a missing or non-finite value or
    a rotation whose norm is more than 1e-6 from 1."""
    if not isinstance(record, dict) or not all(isinstance(record.get(k), dict)
                                               for k in ("calibrated_sensor", "ego_pose")):
        raise ValueError("pose record: expected dict(calibrated_sensor=dict(...), ego_pose=dict(...))")
    t = np.zeros(POSE_DOUBLES)
    for k, (R, tr, q) in (("calibrated_sensor", (0, 9, 24)), ("ego_pose", (12, 21, 28))):
        rec = record[k]
        if "rotation" not in rec or "translation" not in rec:
            raise ValueError("pose record: %s needs rotation and translation" % k)
        unit = _unit_quaternion(rec["rotation"], k)
        t[R:R + 9] = rotation_matrix(unit).reshape(-1)
        t[tr:tr + 3] = _translation(rec["translation"], k)
        t[q:q + 4] = unit
    return t


def check_tokens(tokens, batch):
    """Sample tokens: one distinct str per sample.  ValueError otherwise."""
    tokens = list(tokens)
    if len(tokens) != batch:
        raise ValueError("%d samples but %d tokens" % (batch, len(tokens)))
    if not all(isinstance(t, str) for t in tokens):
        raise ValueError("sample tokens must be str")
    if len(set(tokens)) != len(tokens):
        raise ValueError("sample tokens repeat")
    return tokens


def to_nusc_annos(results, counts, class_names, tokens, table=None):
    """Host results [B, D, 15] f64 and counts [B] -> the reference's nusc_annos: dict(results={token: [box dict, ...]}
    in sample order, meta).  Each box dict has the reference's keys in its order, with Python floats and lists.
    ValueError for a class name without an attribute, and for a row whose translation or size is NaN (the devkit's
    Box asserts on a NaN centre or size)."""
    table = attribute_table(class_names) if table is None else table
    class_names = list(class_names)
    out = {}
    for token, rows, n in zip(tokens, np.asarray(results), np.asarray(counts)):
        r = rows[:int(n)]
        if np.isnan(r[:, 0:6]).any():
            raise ValueError("sample %r: a detection with a NaN centre or size" % (token,))
        annos = []
        for row in r.tolist():
            label = int(row[13])
            annos.append({"sample_token": token, "translation": row[0:3], "size": row[3:6], "rotation": row[6:10],
                          "velocity": row[10:12], "detection_name": class_names[label], "detection_score": row[12],
                          "attribute_name": table[label][row[14] > 0.5]})
        out[token] = annos
    return {"results": out, "meta": dict(META)}


class NuscResults:
    """Static device buffers of one batch -- the pose table f64 [B, 32], results f64 [B, D, 15], counts i32 [B] -- their
    pinned host copies, and the d3b_nusc_results_dev call over them.  The results buffers are sized by the first
    detections launched on (D is the model's); the addresses never change after that, so a captured CUDA graph can
    hold them."""

    def __init__(self, batch, device="cuda"):
        if not 1 <= batch <= MAX_BATCH:
            raise ValueError("batch must be in [1, %d], got %d" % (MAX_BATCH, batch))
        self.batch, self.device = batch, torch.device(device)
        self.poses = torch.zeros((batch, POSE_DOUBLES), dtype=torch.float64, device=self.device)
        self.results = self.counts = None
        self.results_host = self.counts_host = None

    def set_poses(self, table):
        """Synchronous copy of a host table [B, 32] into the device buffer (graphs stage it through pinned memory
        instead: apis.pipeline)."""
        self.poses.copy_(torch.as_tensor(np.asarray(table, np.float64)))

    def launch(self, packed):
        """packed [B, D, 12] f32 device detections (predict's box, score, label, valid) -> (results, counts), one kernel,
        no host sync."""
        B, D, width = packed.shape
        if B != self.batch or packed.dtype != torch.float32 or not packed.is_contiguous():
            raise ValueError("detections must be contiguous f32 [%d, D, %d], got %s %s"
                             % (self.batch, ND + 3, tuple(packed.shape), packed.dtype))
        if self.results is None or self.results.shape[1] != D:
            self.results = torch.zeros((B, D, COLS), dtype=torch.float64, device=self.device)
            self.counts = torch.zeros(B, dtype=torch.int32, device=self.device)
            self.results_host = torch.empty(self.results.shape, dtype=torch.float64, pin_memory=True)
            self.counts_host = torch.empty(B, dtype=torch.int32, pin_memory=True)
        L = _lib.lib()
        with _lib.on_device_of(packed, self.poses), _lib.timed("nusc_results", batch=B, max_det=D):
            st = L.d3b_nusc_results_dev(packed.data_ptr(), self.poses.data_ptr(), B, D, width - 3,
                                        self.results.data_ptr(), self.counts.data_ptr(), _lib.current_stream())
        _lib.check(st, "d3b_nusc_results_dev")
        return self.results, self.counts

    def fetch(self):
        """Enqueues the D2H copies of the results and counts into the pinned host buffers (no sync)."""
        self.results_host.copy_(self.results, non_blocking=True)
        self.counts_host.copy_(self.counts, non_blocking=True)
        return self
