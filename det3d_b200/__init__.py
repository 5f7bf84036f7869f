"""det3d_b200: H100-native (sm_90a) point-cloud inference hot path behind Det3D's module API.

voxelize -> sparse 3-D conv middle encoder -> rotated-box IoU/NMS, as hand-written
CUDA behind a C ABI (include/det3d_b200.h).  The sub-packages mirror the
reference's import paths (det3d.core.input.voxel_generator, det3d.models.backbones.scn,
det3d.core.bbox.box_torch_ops, det3d.ops.iou3d.iou3d_utils, ...); `import det3d`
resolves to this package through the alias package at the repository root.
"""
__version__ = "0.1.0"
