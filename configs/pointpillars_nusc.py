# PointPillars (PillarFeatureNet + PointPillarsScatter + RPN[3,5,5] + 6-task MultiGroupHead), nuScenes.
#
# Inference subset of the reference config
#   examples/point_pillars/configs/nusc_all_point_pillars_mghead_syncbn.py
# (same keys / values for model, test_cfg, voxel_generator, target_assigner, box_coder, assigner;
# dataset / optimizer sections omitted).  us_layer_strides 0.5 makes the first deblock a
# Conv2d(64, 128, kernel_size=2, stride=2).  The reference file itself also loads unchanged
# (tests/test_pillars_nusc.py).
import itertools
import logging

from det3d.builder import build_box_coder
from det3d.utils.config_tool import get_downsample_factor

norm_cfg = None
tasks = [
    dict(num_class=1, class_names=["car"]),
    dict(num_class=2, class_names=["truck", "construction_vehicle"]),
    dict(num_class=2, class_names=["bus", "trailer"]),
    dict(num_class=1, class_names=["barrier"]),
    dict(num_class=2, class_names=["motorcycle", "bicycle"]),
    dict(num_class=2, class_names=["pedestrian", "traffic_cone"]),
]
class_names = list(itertools.chain(*[t["class_names"] for t in tasks]))

# (class, anchor size w/l/h, z centre, matched / unmatched thresholds)
_ANCHORS = [
    ("car", [1.97, 4.63, 1.74], -0.95, 0.6, 0.45),
    ("truck", [2.51, 6.93, 2.84], -0.40, 0.55, 0.4),
    ("construction_vehicle", [2.85, 6.37, 3.19], -0.225, 0.5, 0.35),
    ("bus", [2.94, 10.5, 3.47], -0.085, 0.55, 0.4),
    ("trailer", [2.90, 12.29, 3.87], 0.115, 0.5, 0.35),
    ("barrier", [2.53, 0.50, 0.98], -1.33, 0.55, 0.4),
    ("motorcycle", [0.77, 2.11, 1.47], -1.085, 0.5, 0.3),
    ("bicycle", [0.60, 1.70, 1.28], -1.18, 0.5, 0.35),
    ("pedestrian", [0.67, 0.73, 1.77], -0.935, 0.6, 0.4),
    ("traffic_cone", [0.41, 0.41, 1.07], -1.285, 0.6, 0.4),
]
target_assigner = dict(
    type="iou",
    anchor_generators=[
        dict(type="anchor_generator_range", sizes=size, anchor_ranges=[-51.2, -51.2, z, 51.2, 51.2, z],
             rotations=[0, 1.57], velocities=[0, 0], matched_threshold=mt, unmatched_threshold=ut, class_name=name)
        for name, size, z, mt, ut in _ANCHORS
    ],
    sample_positive_fraction=-1, sample_size=512,
    region_similarity_calculator=dict(type="nearest_iou_similarity"),
    pos_area_threshold=-1, tasks=tasks,
)
box_coder = dict(type="ground_box3d_coder", n_dim=9, linear_dim=False, encode_angle_vector=True)

model = dict(
    type="PointPillars",
    pretrained=None,
    reader=dict(type="PillarFeatureNet", num_filters=[64], num_input_features=5, with_distance=False,
                voxel_size=(0.2, 0.2, 8), pc_range=(-51.2, -51.2, -5.0, 51.2, 51.2, 3.0), norm_cfg=norm_cfg),
    backbone=dict(type="PointPillarsScatter", ds_factor=1, norm_cfg=norm_cfg),
    neck=dict(type="RPN", layer_nums=[3, 5, 5], ds_layer_strides=[2, 2, 2], ds_num_filters=[64, 128, 256],
              us_layer_strides=[0.5, 1, 2], us_num_filters=[128, 128, 128], num_input_features=64,
              norm_cfg=norm_cfg, logger=logging.getLogger("RPN")),
    bbox_head=dict(
        type="MultiGroupHead", mode="3d", in_channels=sum([128, 128, 128]), norm_cfg=norm_cfg, tasks=tasks,
        weights=[1], box_coder=build_box_coder(box_coder), encode_background_as_zeros=True,
        loss_norm=dict(type="NormByNumPositives", pos_cls_weight=1.0, neg_cls_weight=2.0),
        loss_cls=dict(type="SigmoidFocalLoss", alpha=0.25, gamma=2.0, loss_weight=1.0),
        use_sigmoid_score=True,
        loss_bbox=dict(type="WeightedSmoothL1Loss", sigma=3.0,
                       code_weights=[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2, 1.0, 1.0], codewise=True, loss_weight=0.25),
        encode_rad_error_by_sin=False, loss_aux=None, direction_offset=0,
    ),
)
assigner = dict(box_coder=box_coder, target_assigner=target_assigner,
                out_size_factor=get_downsample_factor(model), debug=False)
train_cfg = dict(assigner=assigner)
test_cfg = dict(
    nms=dict(use_rotate_nms=True, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=83,
             nms_iou_threshold=0.2),
    score_threshold=0.1,
    post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0],
    max_per_img=500,
)
voxel_generator = dict(range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], voxel_size=[0.2, 0.2, 8],
                       max_points_in_voxel=20, max_voxel_num=30000)
