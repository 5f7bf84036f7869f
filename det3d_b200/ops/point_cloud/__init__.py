from .point_cloud_ops import points_to_voxel
from .voxelize import Voxelizer, grid_size_of
from .frustum import FrustumCrop
from .kitti_results import KittiResults
