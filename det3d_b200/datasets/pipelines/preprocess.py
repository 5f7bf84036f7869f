"""Inference-side pipeline steps under the reference's registry names: `Preprocess`, `Voxelization`,
`AssignTarget` (det3d/datasets/pipelines/preprocess.py:28-257, 259-304, 306-483).

Same constructor keywords and the same `__call__(res, info) -> (res, info)` contract, so the `test_pipeline` of an
unmodified Det3D config builds through `PIPELINES`.  What changes is where the work runs:

* `Voxelization` calls `VoxelGenerator.generate`, i.e. d3b_voxelize on the GPU (csrc/voxelize.cu), and fills
  `res["lidar"]["voxels"]` with exactly the reference's dict (`voxels, coordinates, num_points, num_voxels [1] int64,
  shape`).  `Voxelization.batched(points_list)` is the fused front the serving path uses: ONE d3b_voxelize call for the
  whole batch with the batch index (collate_kitti, collate.py:130-137) and the VFE mean already applied, outputs on the
  device.
* `AssignTarget` in val/test mode only produces `anchors` (the reference regenerates them on the CPU for every sample,
  preprocess.py:355-378); here they are generated once per feature-map size and cached.

Training branches (`mode == "train"`: GT sampling, augmentation, target assignment) are out of scope and raise.
"""
import numpy as np

from det3d_b200.core.anchor.anchor_generator import anchors_for_tasks
from det3d_b200.core.input.voxel_generator import VoxelGenerator

from ..registry import PIPELINES


def _get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def _training_only(what):
    raise NotImplementedError("det3d_b200 covers the inference path: %s (mode='train') is out of scope" % what)


@PIPELINES.register_module
class Preprocess(object):
    """val/test behaviour of preprocess.py:28-257: pick the point array, optional camera-frustum crop
    (remove_outside_points, KITTI), optional shuffle, optional intensity shift."""

    def __init__(self, cfg=None, **kwargs):
        self.remove_environment = _get(cfg, "remove_environment", False)
        self.shuffle_points = _get(cfg, "shuffle_points", False)
        self.remove_unknown = _get(cfg, "remove_unknown_examples", False)
        self.remove_outside_points = _get(cfg, "remove_outside_points", False)
        self.symmetry_intensity = _get(cfg, "symmetry_intensity", False)
        self.mode = _get(cfg, "mode")
        if self.mode == "train":
            _training_only("Preprocess")
        if _get(cfg, "add_rgb_to_points", False) or _get(cfg, "reference_detections", None) is not None:
            raise NotImplementedError("Preprocess: add_rgb_to_points / reference_detections are unused by the configs in scope")

    def __call__(self, res, info):
        res["mode"] = self.mode
        if res["type"] in ["KittiDataset", "LyftDataset"]:
            points = res["lidar"]["points"]
        elif res["type"] == "NuScenesDataset":
            points = res["lidar"]["combined"]
        else:
            raise NotImplementedError("Preprocess: dataset type %r" % (res["type"],))
        if self.remove_outside_points:
            points = self._remove_outside_points(res, points)
        if self.shuffle_points:
            np.random.shuffle(points)                       # preprocess.py:213-215 (in place, same RNG stream)
        if self.symmetry_intensity:
            points[:, -1] -= 0.5                            # :248-250
        res["lidar"]["points"] = points
        return res, info

    @staticmethod
    def _remove_outside_points(res, points):
        """preprocess.py:111-116: keep the points inside the camera's view frustum (box_np_ops.remove_outside_points,
        on the device), from res["calib"] (rect, Trv2c, P2, as LoadPointCloudAnnotations fills it for a KittiDataset)
        and the image shape.  The reference reads the shape from res["image"]["image_shape"], which its own
        KittiDataset.get_sensor_data (kitti.py:206-222) never sets; here res["image"] is read when present, else
        res["metadata"]["image_shape"].  Raises ValueError without a calibration (the reference's
        `assert calib is not None`), so for every dataset but KITTI."""
        from det3d_b200.core.bbox import box_np_ops

        calib = res.get("calib")
        if calib is None:
            raise ValueError("Preprocess: remove_outside_points needs res['calib'] (a KittiDataset with "
                             "LoadPointCloudAnnotations), %s has none" % (res["type"],))
        image = res.get("image")
        if image is not None and "image_shape" in image:
            image_shape = image["image_shape"]
        else:
            image_shape = res["metadata"]["image_shape"]
        return box_np_ops.remove_outside_points(points, calib["rect"], calib["Trv2c"], calib["P2"], image_shape)


@PIPELINES.register_module
class Voxelization(object):
    def __init__(self, **kwargs):
        cfg = kwargs.get("cfg", None)
        self.range = _get(cfg, "range")
        self.voxel_size = _get(cfg, "voxel_size")
        self.max_points_in_voxel = _get(cfg, "max_points_in_voxel")
        self.max_voxel_num = _get(cfg, "max_voxel_num")
        self.voxel_generator = VoxelGenerator(
            voxel_size=self.voxel_size,
            point_cloud_range=self.range,
            max_num_points=self.max_points_in_voxel,
            max_voxels=self.max_voxel_num,
        )
        self._batched = None

    def __call__(self, res, info):
        grid_size = self.voxel_generator.grid_size
        if res["mode"] == "train":
            _training_only("Voxelization's ground-truth range filter")
        voxels, coordinates, num_points = self.voxel_generator.generate(res["lidar"]["points"])
        num_voxels = np.array([voxels.shape[0]], dtype=np.int64)
        res["lidar"]["voxels"] = dict(
            voxels=voxels,
            coordinates=coordinates,
            num_points=num_points,
            num_voxels=num_voxels,
            shape=grid_size,
        )
        return res, info

    def batched(self, points_list, device="cuda", want_voxels=True, want_mean=True):
        """Voxelization + collate_kitti for a whole batch in ONE d3b_voxelize call (SURVEY 8f.1).

        points_list: per-sample float32 [N_i, ndim] arrays / tensors (host or device).  Returns device tensors with
        the collated layout: voxels [M, max_points, ndim] (optional), coordinates [M, 4] (b, z, y, x), num_points [M],
        mean [M, ndim] (optional), num_voxels int64 [B] (device), shape = grid size.  M = sum of the samples' voxels;
        reading it synchronises once (the reference's numpy concat does the same implicitly)."""
        import torch

        from det3d_b200.ops.point_cloud.voxelize import Voxelizer

        key = (bool(want_voxels), bool(want_mean))
        if self._batched is None or self._batched[0] != key:
            self._batched = (key, Voxelizer(self.voxel_size, self.range, self.max_points_in_voxel, self.max_voxel_num,
                                            want_voxels=want_voxels, want_mean=want_mean))
        vox = self._batched[1]
        dev = torch.device(device)
        tensors = [torch.as_tensor(p, dtype=torch.float32) for p in points_list]
        offsets = [0]
        for t in tensors:
            offsets.append(offsets[-1] + int(t.shape[0]))
        ndim = int(tensors[0].shape[1])
        pts = torch.empty((offsets[-1], ndim), dtype=torch.float32, device=dev)
        for t, a, b in zip(tensors, offsets[:-1], offsets[1:]):
            pts[a:b].copy_(t, non_blocking=True)
        out = vox(pts, offsets)
        counts = out["counts"]
        batch = len(tensors)
        m = int(counts[batch].item())
        return dict(
            voxels=None if out["voxels"] is None else out["voxels"][:m],
            coordinates=out["coors"][:m], num_points=out["num_points"][:m],
            mean=None if out["mean"] is None else out["mean"][:m],
            num_voxels=counts[:batch].to(torch.int64), shape=self.voxel_generator.grid_size,
        )


@PIPELINES.register_module
class AssignTarget(object):
    """val/test behaviour of preprocess.py:306-483: `res["lidar"]["targets"] = {"anchors": [per task [A, nd]]}`."""

    def __init__(self, **kwargs):
        assigner_cfg = kwargs["cfg"]
        self.target_assigner_cfg = _get(assigner_cfg, "target_assigner")
        self.out_size_factor = _get(assigner_cfg, "out_size_factor")
        self.anchor_area_threshold = _get(self.target_assigner_cfg, "pos_area_threshold", -1)
        if self.anchor_area_threshold is not None and self.anchor_area_threshold >= 0:
            raise NotImplementedError("AssignTarget: pos_area_threshold >= 0 (anchors_mask) is unused by the configs in "
                                      "scope and not implemented")
        self._cache = {}

    def anchors(self, grid_size):
        key = tuple(int(g) for g in np.asarray(grid_size).reshape(-1))
        a = self._cache.get(key)
        if a is None:
            a = self._cache[key] = anchors_for_tasks(self.target_assigner_cfg, np.asarray(key), self.out_size_factor)
        return a

    def __call__(self, res, info):
        if res["mode"] == "train":
            _training_only("AssignTarget")
        grid_size = res["lidar"]["voxels"]["shape"]
        res["lidar"]["targets"] = {"anchors": self.anchors(grid_size)}
        return res, info
