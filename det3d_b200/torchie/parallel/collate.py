"""`collate_kitti` under the reference's name (det3d/torchie/parallel/collate.py:90-150), inference keys.

Two forms:

* `collate_kitti(batch_list, samples_per_gpu=1)` -- the reference's contract: a list of per-sample example dicts (the
  output of the `Reformat` step, numpy arrays) -> one batch dict of torch tensors; `coordinates` / `points` get the
  sample index prepended as column 0 (`np.pad(..., constant_values=i)`, :130-137), `voxels / num_points / num_voxels`
  are concatenated (:101-102), `anchors` are stacked per task (:138-147), `metadata` stays a list, `calib` is stacked
  per key, everything else is `np.stack`ed.  Pure host glue, written against the same key table.
* `collate_kitti_device(points_list, voxelization)` -- the fused form the serving path uses (SURVEY 8f.1): raw clouds ->
  the SAME batch dict, produced by one batched d3b_voxelize_dev call (batch index written by the kernel, outputs resident
  on the GPU), so the `[M, max_points, ndim]` host tensors and their H2D copy never exist.

Training-only keys (`gt_boxes`, `labels`, `reg_targets`, ...) raise: target assignment is out of scope.
"""
import collections

import numpy as np
import torch

_CONCAT = ("voxels", "num_points", "num_gt", "voxel_labels", "num_voxels")
_PREPEND_INDEX = ("coordinates", "points")
_PER_TASK = ("anchors", "anchors_mask")
_TRAINING = ("gt_boxes", "reg_targets", "reg_weights", "labels")


def collate_kitti(batch_list, samples_per_gpu=1):
    merged = collections.defaultdict(list)
    for example in batch_list:
        for k, v in example.items():
            merged[k].append(v)
    ret = {}
    for key, elems in merged.items():
        if key in _TRAINING:
            raise NotImplementedError("collate_kitti: %r is a training target; det3d_b200 covers inference" % key)
        if key in _CONCAT:
            ret[key] = torch.tensor(np.concatenate(elems, axis=0))
        elif key == "metadata":
            ret[key] = elems
        elif key == "calib":
            per_key = collections.OrderedDict()
            for elem in elems:
                for k1, v1 in elem.items():
                    per_key.setdefault(k1, []).append(v1)
            ret[key] = {k1: torch.tensor(np.stack(v1, axis=0)) for k1, v1 in per_key.items()}
        elif key in _PREPEND_INDEX:
            rows = [np.pad(c, ((0, 0), (1, 0)), mode="constant", constant_values=i) for i, c in enumerate(elems)]
            ret[key] = torch.tensor(np.concatenate(rows, axis=0))
        elif key in _PER_TASK:
            n_tasks = len(elems[0])
            ret[key] = [torch.stack([torch.tensor(elem[t]) for elem in elems]) for t in range(n_tasks)]
        elif key == "annos":
            ret[key] = elems
        else:
            ret[key] = np.stack(elems, axis=0)
    return ret


def collate_kitti_device(points_list, voxelization, anchors=None, metadata=None, device="cuda", want_voxels=True):
    """Raw clouds -> the batch dict `collate_kitti` would build from per-sample Voxelization outputs, but voxelized and
    collated on the GPU in one call.  `voxelization`: a `Voxelization` pipeline step; `anchors`: per-task [A, nd] arrays
    (e.g. `AssignTarget.anchors(grid)`), expanded over the batch as the reference's stacking does."""
    out = voxelization.batched(points_list, device=device, want_voxels=want_voxels, want_mean=True)
    batch = len(points_list)
    example = dict(voxels=out["voxels"], coordinates=out["coordinates"], num_points=out["num_points"],
                   num_voxels=out["num_voxels"], mean=out["mean"],
                   shape=np.stack([np.asarray(out["shape"])] * batch, axis=0),
                   metadata=metadata if metadata is not None else [None] * batch)
    if anchors is not None:
        dev = torch.device(device)
        example["anchors"] = [torch.as_tensor(a).to(dev).unsqueeze(0).expand(batch, -1, -1) for a in anchors]
    return example
