"""VoxelFeatureExtractorV3: per-voxel mean of the first `num_input_features` point
channels (det3d/models/readers/voxel_encoder.py:197-211)."""
import torch
from torch import nn

from ..registry import READERS


@READERS.register_module
class VoxelFeatureExtractorV3(nn.Module):
    def __init__(self, num_input_features=4, norm_cfg=None, name="VoxelFeatureExtractorV3"):
        super().__init__()
        self.name = name
        self.num_input_features = num_input_features

    def forward(self, features, num_voxels, coors=None):
        c = self.num_input_features
        if features.dim() == 2:
            # fused path: the voxelizer already produced the per-voxel mean [M, ndim]; the leading c columns are returned
            # as a strided view (no copy launch), which the encoder's first layer reads in place
            return features[:, :c]
        total = features[:, :, :c].sum(dim=1, keepdim=False)
        return (total / num_voxels.type_as(features).view(-1, 1)).contiguous()
