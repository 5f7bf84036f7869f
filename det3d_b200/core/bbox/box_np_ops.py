"""KITTI camera-frustum crop under the reference's import path (det3d/core/bbox/box_np_ops.py).

`remove_outside_points(points, rect, Trv2c, P2, image_shape)` keeps the reference's signature (box_np_ops.py:941-952):
numpy in, numpy out, the points inside the camera's view frustum with every column and in input order.  The frustum's
six planes are computed once per calibration on the host, in float64 with the reference's numpy calls in the
reference's order (`camera_frustum_planes`); the per-point test and the compaction run on the device
(d3b_frustum_crop_dev, csrc/frustum.cu), bit-exact to the reference's numba loop.
"""
import numpy as np

# The frustum's 6 faces as indices into its 8 corners (near face 0-3, far face 4-7), each face wound so that its
# normal points into the frustum: the face order and winding of the reference's surfaces (box_np_ops.py:1133-1152)
_FACES = np.array([[0, 1, 2, 3], [7, 6, 5, 4], [0, 3, 7, 4], [1, 5, 6, 2], [0, 4, 5, 1], [3, 2, 6, 7]])
_NEAR_M, _FAR_M = 0.001, 100.0      # depth of the frustum's near and far faces in the camera frame


def _split_projection(P2):
    """P2[:3, :4] = K @ [rot | trans] with K upper triangular -> (K, rot, trans).  The inverse of the left 3x3 block
    is QR-factored (an orthogonal factor times an upper-triangular one) and both factors are inverted back; trans is
    the inverted triangular factor applied to P2's last column."""
    left, last_col = P2[0:3, 0:3], P2[0:3, 3]
    q, r = np.linalg.qr(np.linalg.inv(left))
    K = np.linalg.inv(r)
    rot = np.linalg.inv(q)
    return K, rot, r @ last_col


def _image_frustum(K, height, width):
    """The 8 camera-frame corners [8, 3] of the rays through the image's corners (u, v) = (0, 0), (0, H), (W, H),
    (W, 0), cut at the near depth (rows 0-3) and at the far depth (rows 4-7): x = (u - cu) / (fu / depth),
    y = (v - cv) / (fv / depth)."""
    uv = np.array([[0, 0], [0, height], [width, height], [width, 0]], dtype=K.dtype)
    centre = K[0:2, 2]
    rows = [(uv - centre) / np.array([K[0, 0] / depth, K[1, 1] / depth], dtype=K.dtype) for depth in (_NEAR_M, _FAR_M)]
    depths = np.array([_NEAR_M] * 4 + [_FAR_M] * 4, dtype=K.dtype)[:, np.newaxis]
    return np.concatenate([np.concatenate(rows, axis=0), depths], axis=1)


def camera_frustum_planes(rect, Trv2c, P2, image_shape):
    """float64 [6, 4]: the (n0, n1, n2, d) of the camera frustum's 6 planes in the LiDAR frame, in the reference's order.

    The steps of remove_outside_points up to the point test: the image frustum of image_shape = (H, W) between depths
    0.001 m and 100 m in the camera frame; minus trans, rotated by inv(rot) (P2 = K [rot | trans]) into the rectified
    camera frame; in homogeneous coordinates times inv((rect @ Trv2c)^T) into the LiDAR frame; the 6 faces; and per face
    with corners c0, c1, c2 the normal n = (c0 - c1) x (c1 - c2) and the offset d = -c0x*n0 - c0y*n1 - c0z*n2
    (geometry.py:351-377), each operation rounded on its own.  A point is inside when x*n0 + y*n1 + z*n2 + d < 0 for all
    6 planes.  The numpy calls and their order are the reference's, so the planes are the reference's bits as long as
    numpy's LAPACK / BLAS gives the same inv, qr and matrix products."""
    K, rot, trans = _split_projection(np.asarray(P2))
    cam = _image_frustum(K, image_shape[0], image_shape[1])
    cam -= trans
    rectified = (np.linalg.inv(rot) @ cam.T).T
    homog = np.concatenate([rectified, np.ones([rectified.shape[0], 1])], axis=-1)
    lidar = (homog @ np.linalg.inv((np.asarray(rect) @ np.asarray(Trv2c)).T))[:, :3]
    c = np.asarray(lidar, np.float64)[_FACES]                                # [6 faces, 4 corners, xyz]
    e0, e1 = c[:, 0] - c[:, 1], c[:, 1] - c[:, 2]
    n0 = e0[:, 1] * e1[:, 2] - e0[:, 2] * e1[:, 1]
    n1 = e0[:, 2] * e1[:, 0] - e0[:, 0] * e1[:, 2]
    n2 = e0[:, 0] * e1[:, 1] - e0[:, 1] * e1[:, 0]
    d = -c[:, 0, 0] * n0 - c[:, 0, 1] * n1 - c[:, 0, 2] * n2
    return np.ascontiguousarray(np.stack([n0, n1, n2, d], axis=1), dtype=np.float64)


def remove_outside_points(points, rect, Trv2c, P2, image_shape):
    """points float32 [N, ndim] (3 <= ndim <= 16) -> the rows inside the camera frustum, all columns, input order kept
    (box_np_ops.py:941-952).  The crop runs on the current CUDA device (d3b_frustum_crop_dev); there is no CPU path."""
    import torch

    from det3d_b200.ops.point_cloud.frustum import FrustumCrop

    if not torch.cuda.is_available():
        raise RuntimeError("det3d_b200: remove_outside_points runs on a CUDA device (there is no CPU fallback)")
    points = np.ascontiguousarray(points, dtype=np.float32)
    if points.ndim != 2:
        raise ValueError("points must be [N, ndim], got shape %s" % (points.shape,))
    crop = FrustumCrop(1, points.shape[0], points.shape[1])
    crop.set_table([0, points.shape[0]], camera_frustum_planes(rect, Trv2c, P2, image_shape)[np.newaxis])
    if points.shape[0]:
        crop.points.copy_(torch.from_numpy(points))
    out, offsets = crop.launch()
    n = int(offsets[1].item())           # API boundary: the reference returns an exactly-sized array
    return out[:n].cpu().numpy()
