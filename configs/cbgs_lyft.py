# CBGS (VoxelFeatureExtractorV3 + SpMiddleResNetFHD + RPN(2 blocks) + 5-task MultiGroupHead), Lyft.
#
# Inference subset of the reference config
#   examples/cbgs/configs/lyft_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py
# (same keys / values for model, test_cfg, voxel_generator, target_assigner, box_coder, assigner;
# dataset / optimizer sections omitted).  Points are [N, 4] (x, y, z, intensity) and the reader keeps 3 of them;
# the grid is 2016 x 2016 x 40, the BEV map 252 x 252.  The reference file itself also loads unchanged
# (tests/test_stock_configs_more.py).
import itertools
import logging

from det3d.builder import build_box_coder
from det3d.utils.config_tool import get_downsample_factor

norm_cfg = None
tasks = [
    dict(num_class=1, class_names=["car"]),
    dict(num_class=1, class_names=["pedestrian"]),
    dict(num_class=2, class_names=["motorcycle", "bicycle"]),
    dict(num_class=1, class_names=["other_vehicle"]),
    dict(num_class=2, class_names=["bus", "truck"]),
]
class_names = list(itertools.chain(*[t["class_names"] for t in tasks]))

# (class, anchor size w/l/h, z centre, matched / unmatched thresholds)
_ANCHORS = [
    ("car", [1.93, 4.75, 1.72], -0.86, 0.6, 0.45),
    ("pedestrian", [0.77, 0.81, 1.78], -0.81, 0.55, 0.4),
    ("motorcycle", [0.97, 2.36, 1.60], -0.9, 0.55, 0.4),
    ("bicycle", [0.64, 1.76, 1.46], -1.04, 0.55, 0.4),
    ("other_vehicle", [2.79, 8.2, 3.24], -0.08, 0.55, 0.4),
    ("bus", [2.94, 12.5, 3.43], -0.015, 0.6, 0.45),
    ("truck", [2.83, 10.2, 3.44], -0.015, 0.6, 0.45),
]
target_assigner = dict(
    type="iou",
    anchor_generators=[
        dict(type="anchor_generator_range", sizes=size, anchor_ranges=[-100.8, -100.8, z, 100.8, 100.8, z],
             rotations=[0, 1.57], matched_threshold=mt, unmatched_threshold=ut, class_name=name)
        for name, size, z, mt, ut in _ANCHORS
    ],
    sample_positive_fraction=-1, sample_size=512,
    region_similarity_calculator=dict(type="nearest_iou_similarity"),
    pos_area_threshold=-1, tasks=tasks,
)
box_coder = dict(type="ground_box3d_coder", n_dim=7, linear_dim=False, encode_angle_vector=False)

model = dict(
    type="VoxelNet",
    pretrained=None,
    reader=dict(type="VoxelFeatureExtractorV3", num_input_features=3, norm_cfg=norm_cfg),
    backbone=dict(type="SpMiddleResNetFHD", num_input_features=3, ds_factor=8, norm_cfg=norm_cfg),
    neck=dict(type="RPN", layer_nums=[5, 5], ds_layer_strides=[1, 2], ds_num_filters=[128, 256],
              us_layer_strides=[1, 2], us_num_filters=[256, 256], num_input_features=256, norm_cfg=norm_cfg,
              logger=logging.getLogger("RPN")),
    bbox_head=dict(
        type="MultiGroupHead", mode="3d", in_channels=sum([256, 256]), norm_cfg=norm_cfg, tasks=tasks, weights=[1],
        box_coder=build_box_coder(box_coder), encode_background_as_zeros=True,
        loss_norm=dict(type="NormByNumPositives", pos_cls_weight=1.0, neg_cls_weight=2.0),
        loss_cls=dict(type="SigmoidFocalLoss", alpha=0.25, gamma=2.0, loss_weight=1.0),
        use_sigmoid_score=True,
        loss_bbox=dict(type="WeightedSmoothL1Loss", sigma=3.0, code_weights=[1.0] * 7, codewise=True, loss_weight=1.0),
        encode_rad_error_by_sin=True,
        loss_aux=dict(type="WeightedSoftmaxClassificationLoss", name="direction_classifier", loss_weight=0.2),
        direction_offset=0.785,
    ),
)
assigner = dict(box_coder=box_coder, target_assigner=target_assigner,
                out_size_factor=get_downsample_factor(model), debug=False)
train_cfg = dict(assigner=assigner)
test_cfg = dict(
    nms=dict(use_rotate_nms=True, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=80,
             nms_iou_threshold=0.2),
    score_threshold=0.1,
    post_center_limit_range=[-110, -110, -6, 110, 110, 2],
    max_per_img=500,
)
voxel_generator = dict(range=[-100.8, -100.8, -4.0, 100.8, 100.8, 2.0], voxel_size=[0.1, 0.1, 0.15],
                       max_points_in_voxel=10, max_voxel_num=80000)
