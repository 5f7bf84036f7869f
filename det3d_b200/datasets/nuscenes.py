"""nuScenes result annos under the reference's per-box conversion (det3d/datasets/nuscenes/nuscenes.py:180-274), for
detections on the device.

There is no NuScenesDataset here: `convert_detection_to_nusc_annos` takes the key frames' pose records and sample
tokens the evaluation reads through the devkit, the class names, and predict's packed detections as InferencePipeline
produces them.
"""
import numpy as np
import torch

from det3d_b200.ops.point_cloud.nusc_results import (ND, NuscResults, attribute_table, check_tokens, pose_table,
                                                     to_nusc_annos)


def convert_detection_to_nusc_annos(detections, poses, tokens, class_names):
    """detections: packed f32 [B, D, 12] CUDA tensor (box x, y, z, w, l, h, vx, vy, r, score, label, valid:
    InferencePipeline.pack); poses[b]: dict(calibrated_sensor=dict(translation, rotation), ego_pose=dict(translation,
    rotation)), sample b's LIDAR_TOP records; tokens[b]: its sample token; class_names: the labels' names, flattened
    over the tasks.  Returns the reference's nusc_annos dict (results keyed by token in sample order, meta), computed
    by the same kernel as InferencePipeline.infer_sweeps(nusc_results=True).  Synchronizes.  ValueError on malformed
    arguments."""
    poses = list(poses)
    if not torch.is_tensor(detections) or not detections.is_cuda or detections.dim() != 3:
        raise ValueError("detections must be a [B, D, 12] CUDA tensor")
    if detections.shape[0] != len(poses):
        raise ValueError("%d samples of detections but %d pose records" % (detections.shape[0], len(poses)))
    if detections.shape[2] - 3 != ND:
        raise ValueError("boxes must have %d values (with velocity), got %d" % (ND, detections.shape[2] - 3))
    tokens = check_tokens(tokens, len(poses))
    table = attribute_table(class_names)
    nusc = NuscResults(detections.shape[0], detections.device)
    nusc.set_poses(np.stack([pose_table(p) for p in poses]))
    with torch.cuda.device(detections.device):
        nusc.launch(detections.float().contiguous())
        nusc.fetch()
        torch.cuda.current_stream().synchronize()
    return to_nusc_annos(nusc.results_host.numpy(), nusc.counts_host.numpy(), class_names, tokens, table)
