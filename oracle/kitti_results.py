"""Checker for the device KITTI result rows (csrc/kitti_results.cu, d3b_kitti_results_dev).

Three things, all numpy:
  - `kernel_order`: a float64 restatement of the kernel in its fixed evaluation order (each elementwise numpy operation is
    rounded on its own, so the order is the kernel's).  The float32 steps, the location, the dimensions, rotation_y,
    score and label equal the kernel's bit for bit; the image box and alpha also go through sin / cos / atan2, whose
    CUDA and numpy implementations differ by ulps.
  - `reference_annos`: the reference's conversion (det3d/datasets/kitti/kitti.py:78-158 with box_np_ops'
    limit_period, box_lidar_to_camera, center_to_corner_box3d and project_to_image) restated with the same numpy calls
    in the same order -- its `@` goes through BLAS, as the reference's does.  The golden generator checks it against the
    reference's own functions bit for bit; the GPU tests use it where no golden applies (a model's own detections).
  - `error_bound`: the per-value bound on |kernel - reference| and the margins of the keep / drop tests.

Error model (u = 2^-53; the reference's matmuls may sum in any order, with or without FMA):
  location_i   a 4-term sum S = X*M[i][0] + Y*M[i][1] + Z*M[i][2] + M[i][3] with the same float64 operands on both
               sides; each side is within 3u * sum|terms| of the exact value, so |diff| <= 8u * sum|terms|
  corners      (p0*c + p2*s) + loc: numpy's and CUDA's float64 sin / cos are each within a few ulps of the exact value,
               |diff(s)|, |diff(c)| <= 16u; with the products' and sums' roundings the corner differs by at most
               e = e_loc + 32u * (|p0| + |p2| + |loc|) (x and z), e_loc + 4u * (|p1| + |loc|) (y)
  projection   n_j = sum_k P[j][k] * C_k: |diff| <= sum_k |P[j][k]| e_k + 8u * sum_k |P[j][k] C_k|; u = n_0 / n_2 then
               differs by at most (dn_0 + |u| dn_2) / (|n_2| - dn_2) + 4u |u| (unbounded when |n_2| <= dn_2: a corner on
               the camera plane); the same for v
  bbox         a min / max over the corners and then a clip: both are 1-Lipschitz, so the bound is the corners' largest
  alpha        -atan2f(-y, x) + ry: numpy's float32 atan2 is within 2 float32 ulps, the kernel's (the float64 atan2 rounded
               once) within 1, so |diff| <= 3 ulp32(alpha_f32) + 2u |alpha|
  decisions    the kernel drops a box as the reference does whenever each of the four compared values is farther from
               its threshold (W, H, 0, 0) than its bound; `error_bound` returns that margin as a ratio (> 1: certain)
"""
import numpy as np

U = 2.0 ** -53
CALIB_DOUBLES = 32
COLS = 14                 # bbox 4, alpha, dims 3, location 3, rotation_y, score, label
TWO_PI_F32 = np.float32(np.pi * 2)

# corners_nd's corner order (x0y0z0, x0y0z1, x0y1z1, x0y1z0, x1y0z0, x1y0z1, x1y1z1, x1y1z0) minus the camera origin
# (0.5, 1.0, 0.5)
CORNERS_NORM = np.array([[-0.5, -1.0, -0.5], [-0.5, -1.0, 0.5], [-0.5, 0.0, 0.5], [-0.5, 0.0, -0.5],
                         [0.5, -1.0, -0.5], [0.5, -1.0, 0.5], [0.5, 0.0, 0.5], [0.5, 0.0, -0.5]])


def calib_table(rect, Trv2c, P2, image_shape):
    """float64 [32]: M = rect @ Trv2c (numpy's own matmul: the reference's bits), P2's rows 0..2, H, W."""
    t = np.zeros(CALIB_DOUBLES)
    t[:16] = (np.asarray(rect) @ np.asarray(Trv2c)).reshape(-1)
    t[16:28] = np.asarray(P2, np.float64)[:3].reshape(-1)
    shape = np.asarray(image_shape).reshape(-1)
    t[28], t[29] = shape[0], shape[1]
    return t


def f32_steps(boxes, nd):
    """limit_period on the last column and the z shift, each operation rounded in float32 (kitti.py:117-120)."""
    b = np.array(boxes[:, :nd], np.float32, copy=True)
    r = b[:, nd - 1]
    with np.errstate(invalid="ignore", over="ignore"):
        b[:, nd - 1] = r - np.floor(r / TWO_PI_F32 + np.float32(0.5)) * TWO_PI_F32
        b[:, 2] -= b[:, 5] / np.float32(2)
    return b


def kernel_order(det, nd, table):
    """det [n, nd + 3] f32 (box, score, label, valid), table [32] -> (rows f64 [n, 14], keep bool [n]) for every row,
    valid or not, in the kernel's order.  Also returns the corners' camera-frame values and the projections for
    `error_bound`: dict(loc_terms, corners, num)."""
    b = f32_steps(det, nd)
    M = table[:16].reshape(4, 4)
    P = table[16:28].reshape(3, 4)
    H, W = table[28], table[29]
    X, Y, Z = (b[:, j].astype(np.float64) for j in range(3))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        loc = np.stack([((X * M[i, 0] + Y * M[i, 1]) + Z * M[i, 2]) + M[i, 3] for i in range(3)], 1)
        l, h, w, ry = (b[:, j].astype(np.float64) for j in (4, 5, 3, 6))
        s, c = np.sin(ry), np.cos(ry)
        p0 = l[:, None] * CORNERS_NORM[:, 0]
        p1 = h[:, None] * CORNERS_NORM[:, 1]
        p2 = w[:, None] * CORNERS_NORM[:, 2]
        cx = (p0 * c[:, None] + p2 * s[:, None]) + loc[:, :1]
        cy = p1 + loc[:, 1:2]
        cz = (p0 * -s[:, None] + p2 * c[:, None]) + loc[:, 2:3]
        num = [((cx * P[j, 0] + cy * P[j, 1]) + cz * P[j, 2]) + 0.0 * P[j, 3] for j in range(3)]
        u, v = num[0] / num[2], num[1] / num[2]
        u0, v0, u1, v1 = u.min(1), v.min(1), u.max(1), v.max(1)
        keep = ~((u0 > W) | (v0 > H)) & ~((u1 < 0) | (v1 < 0))
        a32 = np.arctan2(-b[:, 1].astype(np.float64), b[:, 0].astype(np.float64)).astype(np.float32)
        rows = np.stack([np.maximum(u0, 0.0), np.maximum(v0, 0.0), np.minimum(u1, W), np.minimum(v1, H),
                         -a32.astype(np.float64) + ry, l, h, w, loc[:, 0], loc[:, 1], loc[:, 2], ry,
                         det[:, nd].astype(np.float64), det[:, nd + 1].astype(np.float64)], 1)
    keep &= det[:, nd + 2] > 0.5
    aux = dict(X=X, Y=Y, Z=Z, loc=loc, p=(p0, p1, p2), corners=(cx, cy, cz), num=num, u=u, v=v, a32=a32)
    return rows, keep, aux


def error_bound(det, nd, table):
    """-> (bound f64 [n, 14], margin f64 [n]): the bound on |kernel - reference| per value (module docstring) and the
    smallest ratio |compared value - threshold| / bound over the four keep / drop tests (> 1: the kernel's decision is
    the reference's; inf when a value is NaN and so fails its test on both sides)."""
    rows, _keep, a = kernel_order(det, nd, table)
    M = table[:16].reshape(4, 4)
    P = table[16:28].reshape(3, 4)
    H, W = table[28], table[29]
    n = det.shape[0]
    bound = np.zeros((n, COLS))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        e_loc = np.stack([8 * U * (np.abs(a["X"] * M[i, 0]) + np.abs(a["Y"] * M[i, 1]) + np.abs(a["Z"] * M[i, 2])
                                   + abs(M[i, 3])) for i in range(3)], 1)
        bound[:, 8:11] = e_loc
        p0, p1, p2 = a["p"]
        loc = a["loc"]
        ex = e_loc[:, :1] + 32 * U * (np.abs(p0) + np.abs(p2) + np.abs(loc[:, :1]))
        ey = e_loc[:, 1:2] + 4 * U * (np.abs(p1) + np.abs(loc[:, 1:2]))
        ez = e_loc[:, 2:3] + 32 * U * (np.abs(p0) + np.abs(p2) + np.abs(loc[:, 2:3]))
        C = a["corners"]
        dn = [np.abs(P[j, 0]) * ex + np.abs(P[j, 1]) * ey + np.abs(P[j, 2]) * ez
              + 8 * U * (np.abs(P[j, 0] * C[0]) + np.abs(P[j, 1] * C[1]) + np.abs(P[j, 2] * C[2])) for j in range(3)]
        den = np.abs(a["num"][2]) - dn[2]
        bad = ~(den > 0)
        du = np.where(bad, np.inf, (dn[0] + np.abs(a["u"]) * dn[2]) / np.where(bad, 1.0, den) + 4 * U * np.abs(a["u"]))
        dv = np.where(bad, np.inf, (dn[1] + np.abs(a["v"]) * dn[2]) / np.where(bad, 1.0, den) + 4 * U * np.abs(a["v"]))
        bu, bv = du.max(1), dv.max(1)
        bound[:, 0], bound[:, 1], bound[:, 2], bound[:, 3] = bu, bv, bu, bv
        a32 = np.abs(a["a32"])
        bound[:, 4] = 3 * np.spacing(a32).astype(np.float64) + 2 * U * np.abs(rows[:, 4])
        u0, v0, u1, v1 = a["u"].min(1), a["v"].min(1), a["u"].max(1), a["v"].max(1)
        ratios = [np.abs(u0 - W) / bu, np.abs(v0 - H) / bv, np.abs(u1) / bu, np.abs(v1) / bv]
        ratios = [np.where(np.isnan(r), np.inf, r) for r in ratios]
    return bound, np.minimum.reduce(ratios)


# ---- the reference's conversion, with its numpy calls ----------------------------------------------------------------
def _limit_period(val, offset=0.5, period=np.pi):
    return val - np.floor(val / period + offset) * period


def reference_rows(det, nd, calib):
    """The reference's per-frame conversion of det [n, nd + 3] f32 (valid rows only are read) under calib dict(rect,
    Trv2c, P2, image_shape) -> (kept, each a tuple (bbox f64 [4], alpha, dims f64 [3], loc f64 [3], ry, score f32,
    label int)).  Restates kitti.py:97-153 with box_np_ops' functions: the same numpy operations in the same order."""
    rows = det[det[:, nd + 2] > 0.5]
    box = np.array(rows[:, :nd], np.float32, copy=True)
    out = []
    if box.shape[0] == 0:
        return out
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        box[:, -1] = _limit_period(box[:, -1], offset=0.5, period=np.pi * 2)
        box[:, 2] -= box[:, 5] / 2
        xyz1 = np.concatenate([box[:, 0:3], np.ones([box.shape[0], 1])], axis=-1)
        xyz = (xyz1 @ (calib["rect"] @ calib["Trv2c"]).T)[..., :3]
        cam = np.concatenate([xyz, box[:, 4:5], box[:, 5:6], box[:, 3:4], box[:, 6:7]], axis=1)
        dims = cam[:, 3:6]
        corners = dims.reshape([-1, 1, 3]) * CORNERS_NORM.reshape([1, 8, 3])
        ang = cam[:, 6]
        sn, cs = np.sin(ang), np.cos(ang)
        zero, one = np.zeros_like(cs), np.ones_like(cs)
        rot_t = np.stack([[cs, zero, -sn], [zero, one, zero], [sn, zero, cs]])
        corners = np.einsum("aij,jka->aik", corners, rot_t)
        corners += cam[:, :3].reshape([-1, 1, 3])
        pts4 = np.concatenate([corners, np.zeros(list(corners.shape[:-1]) + [1])], axis=-1)
        img = pts4 @ np.asarray(calib["P2"]).T
        img = img[..., :2] / img[..., 2:3]
        bbox = np.concatenate([np.min(img, axis=1), np.max(img, axis=1)], axis=1)
        shape = np.asarray(calib["image_shape"])
        for j in range(cam.shape[0]):
            if bbox[j, 0] > shape[1] or bbox[j, 1] > shape[0]:
                continue
            if bbox[j, 2] < 0 or bbox[j, 3] < 0:
                continue
            bbox[j, 2:] = np.minimum(bbox[j, 2:], shape[::-1])
            bbox[j, :2] = np.maximum(bbox[j, :2], [0, 0])
            alpha = -np.arctan2(-box[j, 1], box[j, 0]) + cam[j, 6]
            out.append((bbox[j].copy(), alpha, cam[j, 3:6].copy(), cam[j, :3].copy(), cam[j, 6], rows[j, nd],
                        int(rows[j, nd + 1])))
    return out


def reference_annos(det, nd, calib, class_names):
    """reference_rows as the reference's anno dict (get_start_result_anno's keys, np.stack'ed; empty_result_anno when
    nothing is kept)."""
    kept = reference_rows(det, nd, calib)
    if not kept:
        return dict(name=np.array([]), truncated=np.array([]), occluded=np.array([]), alpha=np.array([]),
                    bbox=np.zeros([0, 4]), dimensions=np.zeros([0, 3]), location=np.zeros([0, 3]),
                    rotation_y=np.array([]), score=np.array([]))
    return dict(name=np.stack([class_names[k[6]] for k in kept]), truncated=np.stack([0.0 for _ in kept]),
                occluded=np.stack([0 for _ in kept]), alpha=np.stack([k[1] for k in kept]),
                bbox=np.stack([k[0] for k in kept]), dimensions=np.stack([k[2] for k in kept]),
                location=np.stack([k[3] for k in kept]), rotation_y=np.stack([k[4] for k in kept]),
                score=np.stack([k[5] for k in kept]))


# ---- variants the exact golden must tell apart -----------------------------------------------------------------------
VARIANTS = ("ge", "ones", "clip_first", "clip_hw")


def variant_rows(det, nd, table, variant):
    """kernel_order with one rule changed -> (rows, keep):
      ge          >= / <= in place of the strict > / < tests
      ones        project_to_image with a column of ones (P2's translation enters)
      clip_first  every bbox coordinate clamped into [0, W] x [0, H] before the test
      clip_hw     bbox[2:] clipped to (H, W) instead of (W, H)"""
    t = np.array(table, copy=True)
    if variant == "ones":
        rows, keep, a = kernel_order(det, nd, t)
        P = t[16:28].reshape(3, 4)
        cx, cy, cz = a["corners"]
        num = [((cx * P[j, 0] + cy * P[j, 1]) + cz * P[j, 2]) + P[j, 3] for j in range(3)]
        u, v = num[0] / num[2], num[1] / num[2]
        return _decide(u.min(1), v.min(1), u.max(1), v.max(1), t, det, nd, rows, "strict")
    rows, keep, a = kernel_order(det, nd, t)
    u0, v0, u1, v1 = a["u"].min(1), a["v"].min(1), a["u"].max(1), a["v"].max(1)
    return _decide(u0, v0, u1, v1, t, det, nd, rows, variant)


def _decide(u0, v0, u1, v1, t, det, nd, rows, variant):
    H, W = t[28], t[29]
    if variant == "clip_first":
        u0, u1 = np.clip(u0, 0, W), np.clip(u1, 0, W)
        v0, v1 = np.clip(v0, 0, H), np.clip(v1, 0, H)
    if variant == "ge":
        keep = ~((u0 >= W) | (v0 >= H)) & ~((u1 <= 0) | (v1 <= 0))
    else:
        keep = ~((u0 > W) | (v0 > H)) & ~((u1 < 0) | (v1 < 0))
    rows = np.array(rows, copy=True)
    rows[:, 0], rows[:, 1] = np.maximum(u0, 0.0), np.maximum(v0, 0.0)
    if variant == "clip_hw":
        rows[:, 2], rows[:, 3] = np.minimum(u1, H), np.minimum(v1, W)
    else:
        rows[:, 2], rows[:, 3] = np.minimum(u1, W), np.minimum(v1, H)
    return rows, keep & (det[:, nd + 2] > 0.5)
