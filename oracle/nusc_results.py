"""Checker for the device nuScenes result rows (csrc/nusc_results.cu, d3b_nusc_results_dev).

Three things, all numpy:
  - `kernel_order`: a float64 restatement of the kernel in its fixed evaluation order (each elementwise numpy operation
    is rounded on its own, so the order is the kernel's).  The float32 yaw, the sizes, score, label, and -- where no
    sin / cos enters -- the translation and velocity equal the kernel's bit for bit; the rotation goes through sin / cos,
    whose CUDA and libm implementations differ by ulps.
  - `reference_annos`: the reference's conversion (det3d/datasets/nuscenes/nusc_common.py:222-265 and the per-box loop
    of NuScenesDataset.evaluation, nuscenes.py:219-259) run on the stand-in `Quaternion` and `Box` below, which restate
    pyquaternion 0.9.x (Quaternion(list), Quaternion(axis, radians), Quaternion(array), rotation_matrix with its
    _normalise, __mul__, elements) and the nuScenes devkit's Box (__init__'s NaN asserts, rotate, translate).  The
    golden generator runs the reference's own functions, lifted with `ast`, on the same stand-ins and checks this
    restatement against them; pyquaternion and the devkit themselves are not available here, so parity with them is
    restated, not pinned.
  - `error_bound`: the per-value bound on |kernel - reference| and the margin of the speed test.

Error model (u = 2^-53).  Both sides start from the same float64 operands: the centre, velocity and float32 yaw are the
detector's floats, and Rc, Rp, qc, qp are the same bits (pose_table restates rotation_matrix with numpy's dot).  The
reference's np.dot may sum in any order, with or without FMA; each side of an n-term sum is within n u sum|terms| of
the exact value, so two sides differ by at most 8u sum|terms| for n <= 4.  A record rotation whose q . q is within 2e-14
of 1 may or may not be normalised by pyquaternion's is_unit test depending on how q . q is summed; that changes R by
nu = |1 - q . q| relatively and q by nu / 2, added as nu sum|terms| at each rotation.
  c1, t, v1, vg     e = sum_j |R_ij| e_in_j + (8u + nu) sum_j |R_ij in_j| (+ 8u |t_i| for the translations)
  qy                CUDA's sin / cos are within 2 ulp, libm's within 1: |diff| <= 4 spacing(|value|) per component; the
                    0 * sin components are zeros on both sides
  q1, rotation      e = sum_k |Q(a)_ik| e_in_k + (8u + nu) sum_k |Q(a)_ik in_k|
  speed             sqrt is 1-Lipschitz in the euclidean norm: e_s = e_vg0 + e_vg1 + 8u s; the kernel's moving flag is the
                    reference's whenever |s - 0.2| > e_s, and `error_bound` returns that ratio as the margin (> 1:
                    certain; inf for a NaN speed, which is not moving on either side)
"""
import math
import operator

import numpy as np

U = 2.0 ** -53
POSE_DOUBLES = 32
COLS = 15                 # translation 3, size 3, rotation 4, velocity 2, score, label, moving
ND = 9
HALF_PI_F32 = np.float32(np.pi / 2)
META = {"use_camera": False, "use_lidar": True, "use_radar": False, "use_map": False, "use_external": False}
NU_WINDOW = 2e-14         # |1 - q . q| under which the is_unit test may go either way


# ---- stand-ins for pyquaternion.Quaternion and nuscenes.utils.data_classes.Box -----------------------------------------
class Quaternion:
    """pyquaternion 0.9.x, the parts the reference's conversion calls."""

    def __init__(self, *args, **kwargs):
        if args:
            self.q = np.array([float(e) for e in args[0]])
        elif "array" in kwargs:
            self.q = np.array([float(e) for e in kwargs["array"]])
        else:
            axis = np.array([float(e) for e in kwargs["axis"]])
            angle = float(kwargs["radians"])
            mag_sq = np.dot(axis, axis)
            if abs(1.0 - mag_sq) > 1e-12:
                axis = axis / math.sqrt(mag_sq)
            theta = angle / 2.0
            r, i = math.cos(theta), axis * math.sin(theta)
            self.q = np.array([r, i[0], i[1], i[2]])

    def _sum_of_squares(self):
        return np.dot(self.q, self.q)

    def is_unit(self, tolerance=1e-14):
        return abs(1.0 - self._sum_of_squares()) < tolerance

    def _normalise(self):
        if not self.is_unit():
            n = math.sqrt(self._sum_of_squares())
            if n > 0:
                self.q = self.q / n

    def _q_matrix(self):
        q = self.q
        return np.array([[q[0], -q[1], -q[2], -q[3]], [q[1], q[0], -q[3], q[2]],
                         [q[2], q[3], q[0], -q[1]], [q[3], -q[2], q[1], q[0]]])

    def _q_bar_matrix(self):
        q = self.q
        return np.array([[q[0], -q[1], -q[2], -q[3]], [q[1], q[0], q[3], -q[2]],
                         [q[2], -q[3], q[0], q[1]], [q[3], q[2], -q[1], q[0]]])

    @property
    def rotation_matrix(self):
        self._normalise()
        return np.dot(self._q_matrix(), self._q_bar_matrix().conj().transpose())[1:][:, 1:]

    def __mul__(self, other):
        return Quaternion(array=np.dot(self._q_matrix(), other.q))

    @property
    def elements(self):
        return self.q


class Box:
    """The nuScenes devkit's Box, the parts the reference's conversion calls."""

    def __init__(self, center, size, orientation, label=np.nan, score=np.nan, velocity=(np.nan, np.nan, np.nan),
                 name=None, token=None):
        assert not np.any(np.isnan(center))
        assert not np.any(np.isnan(size))
        assert len(center) == 3
        assert len(size) == 3
        assert type(orientation) == Quaternion
        self.center = np.array(center)
        self.wlh = np.array(size)
        self.orientation = orientation
        self.label = int(label) if not np.isnan(label) else label
        self.score = float(score) if not np.isnan(score) else score
        self.velocity = np.array(velocity)
        self.name = name
        self.token = token

    def translate(self, x):
        self.center += x

    def rotate(self, quaternion):
        self.center = np.dot(quaternion.rotation_matrix, self.center)
        self.orientation = quaternion * self.orientation
        self.velocity = np.dot(quaternion.rotation_matrix, self.velocity)


# ---- the reference's conversion on the stand-ins --------------------------------------------------------------------
MOVING = dict.fromkeys(("car", "construction_vehicle", "bus", "truck", "trailer"), "vehicle.moving")
MOVING.update(dict.fromkeys(("bicycle", "motorcycle"), "cycle.with_rider"))
STILL = {"pedestrian": "pedestrian.standing", "bus": "vehicle.stopped"}


def attribute(name, moving, fallback):
    """nuscenes.py:219-259: the rule, else fallback[name] (the class's most frequent attribute in cls_attr_dist)."""
    attr = (MOVING if moving else STILL).get(name)
    return attr if attr is not None else fallback[name]


def most_frequent(cls_attr_dist):
    """{class: the attribute max(items, key=count) picks, ties to the first key} of a cls_attr_dist-shaped dict."""
    return {k: max(v.items(), key=operator.itemgetter(1))[0] for k, v in cls_attr_dist.items()}


def reference_boxes(det, nd, record, token, class_names, fallback):
    """The reference's submission boxes of one sample: det [D, nd + 3] f32 (valid rows only are read), record
    dict(calibrated_sensor, ego_pose) -> list of box dicts in the reference's key order."""
    rows = det[det[:, nd + 2] > 0.5]
    box3d = np.array(rows[:, :nd], np.float32, copy=True)
    scores, labels = rows[:, nd].copy(), rows[:, nd + 1].astype(np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        box3d[:, -1] = -box3d[:, -1] - np.pi / 2
    out = []
    for i in range(box3d.shape[0]):
        box = Box(box3d[i, :3], box3d[i, 3:6], Quaternion(axis=[0, 0, 1], radians=box3d[i, -1]), label=labels[i],
                  score=scores[i], velocity=(*box3d[i, 6:8], 0.0))
        cs, ego = record["calibrated_sensor"], record["ego_pose"]
        box.rotate(Quaternion(cs["rotation"]))
        box.translate(np.array(cs["translation"]))
        box.rotate(Quaternion(ego["rotation"]))
        box.translate(np.array(ego["translation"]))
        name = class_names[box.label]
        moving = np.sqrt(box.velocity[0] ** 2 + box.velocity[1] ** 2) > 0.2
        out.append({"sample_token": token, "translation": box.center.tolist(), "size": box.wlh.tolist(),
                    "rotation": box.orientation.elements.tolist(), "velocity": box.velocity[:2].tolist(),
                    "detection_name": name, "detection_score": box.score,
                    "attribute_name": attribute(name, moving, fallback)})
    return out


def reference_annos(packed, records, tokens, class_names, fallback=None):
    """The reference's nusc_annos of packed [B, D, nd + 3] under records[b] / tokens[b]; fallback defaults to the
    package's table of most frequent attributes (the golden generator passes the one from cls_attr_dist)."""
    if fallback is None:
        from det3d_b200.ops.point_cloud.nusc_results import MOST_FREQUENT_ATTRIBUTE as fallback
    nd = packed.shape[-1] - 3
    results = {}
    for b, token in enumerate(tokens):
        results[token] = reference_boxes(packed[b], nd, records[b], token, class_names, fallback)
    return {"results": results, "meta": dict(META)}


# ---- the kernel's order -------------------------------------------------------------------------------------------
def pose_table(record):
    """float64 [32] from the stand-in: Rc, tc, Rp, tp, qc, qp (normalised as rotation_matrix normalises them)."""
    t = np.zeros(POSE_DOUBLES)
    for k, (R, tr, q) in (("calibrated_sensor", (0, 9, 24)), ("ego_pose", (12, 21, 28))):
        quat = Quaternion(record[k]["rotation"])
        t[R:R + 9] = quat.rotation_matrix.reshape(-1)
        t[tr:tr + 3] = np.array(record[k]["translation"], np.float64)
        t[q:q + 4] = quat.q
    return t


def _dot3(R, i, a, b, c):
    return (R[i, 0] * a + R[i, 1] * b) + R[i, 2] * c


def _q_matrix(q):
    return np.array([[q[0], -q[1], -q[2], -q[3]], [q[1], q[0], -q[3], q[2]],
                     [q[2], q[3], q[0], -q[1]], [q[3], -q[2], q[1], q[0]]])


def _hamilton(a, b):
    """a [4] (x) b [n, 4], each component summed in k order."""
    Q = _q_matrix(a)
    return np.stack([((Q[i, 0] * b[:, 0] + Q[i, 1] * b[:, 1]) + Q[i, 2] * b[:, 2]) + Q[i, 3] * b[:, 3]
                     for i in range(4)], 1)


def yaw_f32(det):
    """fl32(fl32(-r) - fl32(pi / 2)), the reference's float32 step."""
    with np.errstate(invalid="ignore", over="ignore"):
        return -det[:, 8].astype(np.float32) - HALF_PI_F32


def kernel_order(det, table, yaw=None, speed_f32=False, translate_first=False):
    """det [n, 12] f32 (box, score, label, valid), table [32] -> (rows f64 [n, 15], valid bool [n], aux) for every row,
    valid or not, in the kernel's order.  The keyword arguments exist for VARIANTS."""
    Rc, tc, Rp, tp = table[0:9].reshape(3, 3), table[9:12], table[12:21].reshape(3, 3), table[21:24]
    qc, qp = table[24:28], table[28:32]
    yaw = yaw_f32(det) if yaw is None else yaw
    with np.errstate(invalid="ignore", over="ignore"):
        th = yaw.astype(np.float64) * 0.5
        s, c = np.sin(th), np.cos(th)
        qy = np.stack([c, 0.0 * s, 0.0 * s, s], 1)
        x, y, z, vx, vy = (det[:, j].astype(np.float64) for j in (0, 1, 2, 6, 7))
        if translate_first:
            x, y, z = x + tc[0], y + tc[1], z + tc[2]
            c1 = [_dot3(Rc, i, x, y, z) for i in range(3)]
            c1 = [c1[i] + tp[i] for i in range(3)]
            t = [_dot3(Rp, i, *c1) for i in range(3)]
        else:
            c1 = [_dot3(Rc, i, x, y, z) + tc[i] for i in range(3)]
            t = [_dot3(Rp, i, *c1) + tp[i] for i in range(3)]
        v1 = [_dot3(Rc, i, vx, vy, 0.0) for i in range(3)]
        vg = [_dot3(Rp, i, *v1) for i in range(2)]
        q1 = _hamilton(qc, qy)
        rot = _hamilton(qp, q1)
        if speed_f32:
            v32 = [v.astype(np.float32) for v in vg]
            speed = np.sqrt(v32[0] * v32[0] + v32[1] * v32[1])
            moving = speed > np.float32(0.2)
        else:
            speed = np.sqrt(vg[0] * vg[0] + vg[1] * vg[1])
            moving = speed > 0.2
        rows = np.stack(t + [det[:, j].astype(np.float64) for j in (3, 4, 5)] + [rot[:, i] for i in range(4)] + vg
                        + [det[:, ND].astype(np.float64), det[:, ND + 1].astype(np.float64),
                           moving.astype(np.float64)], 1)
    aux = dict(x=(x, y, z), v=(vx, vy), c1=c1, v1=v1, qy=qy, q1=q1, speed=speed)
    return rows, det[:, ND + 2] > 0.5, aux


def _nu(q_raw):
    d = abs(1.0 - float(np.dot(q_raw, q_raw)))
    return d if d < NU_WINDOW else 0.0


def error_bound(det, table, records=None):
    """-> (bound f64 [n, 15], margin f64 [n]): the bound on |kernel - reference| per value (module docstring) and the
    ratio |speed - 0.2| / bound of the speed test (> 1: the kernel's moving flag is the reference's).  records (the
    raw dicts) give the normalisation term; without them the table's unit quaternions are taken as given."""
    rows, _valid, a = kernel_order(det, table)
    Rc, tc, Rp, tp = table[0:9].reshape(3, 3), table[9:12], table[12:21].reshape(3, 3), table[21:24]
    qc, qp = table[24:28], table[28:32]
    nu_c = nu_p = 0.0
    if records is not None:
        nu_c = _nu(np.array(records["calibrated_sensor"]["rotation"], np.float64))
        nu_p = _nu(np.array(records["ego_pose"]["rotation"], np.float64))
    n = det.shape[0]
    bound = np.zeros((n, COLS))
    k_c, k_p = 8 * U + nu_c, 8 * U + nu_p
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        x = a["x"]
        e_c1 = [k_c * sum(np.abs(Rc[j, k] * x[k]) for k in range(3)) + 8 * U * abs(tc[j]) for j in range(3)]
        for i in range(3):
            bound[:, i] = (sum(abs(Rp[i, j]) * e_c1[j] for j in range(3))
                           + k_p * sum(np.abs(Rp[i, j] * a["c1"][j]) for j in range(3)) + 8 * U * abs(tp[i]))
        v = a["v"]
        e_v1 = [k_c * (np.abs(Rc[j, 0] * v[0]) + np.abs(Rc[j, 1] * v[1])) for j in range(3)]
        for i in range(2):
            bound[:, 10 + i] = (sum(abs(Rp[i, j]) * e_v1[j] for j in range(3))
                                + k_p * sum(np.abs(Rp[i, j] * a["v1"][j]) for j in range(3)))
        e_qy = 4 * np.spacing(np.abs(a["qy"]))
        e_qy[:, 1:3] = 0.0
        Qc, Qp = np.abs(_q_matrix(qc)), np.abs(_q_matrix(qp))
        e_q1 = np.stack([(e_qy * Qc[i]).sum(1) + k_c * (np.abs(a["qy"]) * Qc[i]).sum(1) for i in range(4)], 1)
        for i in range(4):
            bound[:, 6 + i] = (e_q1 * Qp[i]).sum(1) + k_p * (np.abs(a["q1"]) * Qp[i]).sum(1)
        e_s = bound[:, 10] + bound[:, 11] + 8 * U * a["speed"]
        margin = np.abs(a["speed"] - 0.2) / e_s
        margin = np.where(np.isnan(margin), np.inf, margin)
    return bound, margin


def attributes(rows, class_names, fallback):
    """The attribute of each row of kernel_order's rows (label, moving)."""
    return [attribute(class_names[int(r[13])], r[14] > 0.5, fallback) for r in rows]


# ---- variants the exact golden must tell apart -----------------------------------------------------------------------
VARIANTS = ("yaw_f64", "half_pi_f64", "speed_f32", "translate_first", "attr_first_key")


def variant_output(det, table, class_names, fallback, variant):
    """(rows, attributes) of every row with one rule changed:
      yaw_f64          yaw' = -r - pi/2 in float64 (no float32 rounding)
      half_pi_f64      yaw' = fl32(fl32(-r) - pi/2), pi/2 not rounded to float32 before the subtraction
      speed_f32        the speed and the 0.2 test in float32
      translate_first  each translation added before its rotation
      attr_first_key   the fallback attribute is cls_attr_dist's first key (cycle.with_rider) instead of its argmax
    variant None gives the kernel's own."""
    kw = {}
    with np.errstate(invalid="ignore", over="ignore"):
        if variant == "yaw_f64":
            kw["yaw"] = -det[:, 8].astype(np.float64) - np.pi / 2
        elif variant == "half_pi_f64":
            kw["yaw"] = ((-det[:, 8].astype(np.float32)).astype(np.float64) - np.pi / 2).astype(np.float32)
    if variant == "speed_f32":
        kw["speed_f32"] = True
    elif variant == "translate_first":
        kw["translate_first"] = True
    rows, _valid, _a = kernel_order(det, table, **kw)
    if variant == "attr_first_key":
        fallback = dict.fromkeys(fallback, "cycle.with_rider")
    return rows, attributes(rows, class_names, fallback)
