"""KITTI result annos under the reference's name (det3d/datasets/kitti/kitti.py:78-158), for detections on the device.

There is no KittiDataset here: `convert_detection_to_kitti_annos` takes the calibrations and class names the method
reads from the dataset's infos, and predict's packed detections as InferencePipeline produces them.
"""
import numpy as np
import torch

from det3d_b200.ops.point_cloud.kitti_results import KittiResults, calib_table, check_calibs, to_annos


def convert_detection_to_kitti_annos(detections, calibs, class_names):
    """detections: packed f32 [B, D, nd + 3] CUDA tensor (box, score, label, valid: InferencePipeline.pack);
    calibs[b]: dict(rect, Trv2c, P2, image_shape) (the info's R0_rect, Tr_velo_to_cam, P2 and image shape (H, W));
    class_names: the labels' names, flattened over the tasks.  Returns one anno dict per frame with the reference's
    keys and dtypes -- the detections whose image box meets the image, in order -- computed by the same kernel as
    InferencePipeline.infer_raw(kitti_results=True).  Synchronizes.  ValueError on malformed arguments."""
    calibs = list(calibs)
    if not torch.is_tensor(detections) or not detections.is_cuda or detections.dim() != 3:
        raise ValueError("detections must be a [B, D, nd + 3] CUDA tensor")
    if detections.shape[0] != len(calibs):
        raise ValueError("%d frames of detections but %d calibrations" % (detections.shape[0], len(calibs)))
    if detections.shape[2] - 3 not in (7, 9):
        raise ValueError("boxes must have 7 or 9 values, got %d" % (detections.shape[2] - 3))
    check_calibs(calibs)
    kitti = KittiResults(detections.shape[0], detections.device)
    kitti.set_calib(np.stack([calib_table(c) for c in calibs]))
    with torch.cuda.device(detections.device):
        results, counts = kitti.launch(detections.float().contiguous())
        kitti.results_host.copy_(results, non_blocking=True)
        kitti.counts_host.copy_(counts, non_blocking=True)
        torch.cuda.current_stream().synchronize()
    return to_annos(kitti.results_host.numpy(), kitti.counts_host.numpy(), class_names)
