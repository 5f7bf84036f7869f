"""PointPillars reader / scatter (BASELINE config 3; SURVEY 8f.3).

Same registry names, constructor arguments and parameter layout (`pfn_layers.<i>.linear.weight`,
`pfn_layers.<i>.norm.*`) as det3d/models/readers/pillar_encoder.py:17-211:
  PillarFeatureNet : 9-feature decoration (x,y,z,r, offset from the pillar's point mean, offset from the
                     pillar centre), Linear(9->64, no bias) + BatchNorm1d + ReLU, max over the <=100 points
  PointPillarsScatter : pillar features -> dense pseudo-image [B, 64, ny, nx]
In eval mode with the single-layer configuration the Det3D configs use, the whole reader is ONE kernel
(csrc/pillars.cu: decoration, GEMV, folded BN, ReLU and the max in registers/shared memory -- the
[M,100,64] intermediate the reference materialises never exists) and the scatter is d3b_sparse_to_dense;
other configurations fall back to the module-by-module torch forward.
"""
import ctypes as C

import torch
from torch import nn
from torch.nn import functional as F

from det3d_b200 import _lib

from ..registry import BACKBONES, READERS
from ..utils import build_norm_layer


def get_paddings_indicator(actual_num, max_num, axis=0):
    """[N] counts -> [N, max_num] bool mask of the occupied slots (det3d/models/utils/misc.py:180-202)."""
    actual_num = torch.unsqueeze(actual_num, axis + 1)
    shape = [1] * len(actual_num.shape)
    shape[axis + 1] = -1
    slots = torch.arange(max_num, dtype=torch.int, device=actual_num.device).view(shape)
    return actual_num.int() > slots


class PFNLayer(nn.Module):
    def __init__(self, in_channels, out_channels, norm_cfg=None, last_layer=False):
        super().__init__()
        self.name = "PFNLayer"
        self.last_vfe = last_layer
        if not self.last_vfe:
            out_channels = out_channels // 2
        self.units = out_channels
        self.norm_cfg = norm_cfg if norm_cfg is not None else dict(type="BN1d", eps=1e-3, momentum=0.01)
        self.linear = nn.Linear(in_channels, self.units, bias=False)
        self.norm = build_norm_layer(self.norm_cfg, self.units)[1]

    def forward(self, inputs):
        x = self.linear(inputs)
        x = self.norm(x.permute(0, 2, 1).contiguous()).permute(0, 2, 1).contiguous()
        x = F.relu(x)
        x_max = torch.max(x, dim=1, keepdim=True)[0]
        if self.last_vfe:
            return x_max
        return torch.cat([x, x_max.repeat(1, inputs.shape[1], 1)], dim=2)


@READERS.register_module
class PillarFeatureNet(nn.Module):
    def __init__(self, num_input_features=4, num_filters=(64,), with_distance=False, voxel_size=(0.2, 0.2, 4),
                 pc_range=(0, -40, -3, 70.4, 40, 1), norm_cfg=None):
        super().__init__()
        self.name = "PillarFeatureNet"
        assert len(num_filters) > 0
        self.num_input = num_input_features
        n_in = num_input_features + 5 + (1 if with_distance else 0)
        self._with_distance = with_distance
        filters = [n_in] + list(num_filters)
        self.pfn_layers = nn.ModuleList(
            [PFNLayer(filters[i], filters[i + 1], norm_cfg=norm_cfg, last_layer=(i == len(filters) - 2))
             for i in range(len(filters) - 1)])
        self.vx, self.vy = voxel_size[0], voxel_size[1]
        self.x_offset = self.vx / 2 + pc_range[0]
        self.y_offset = self.vy / 2 + pc_range[1]

    # ---- fused CUDA path -------------------------------------------------------------------
    def _fusable(self, features):
        return (not self.training and features.is_cuda and len(self.pfn_layers) == 1 and not self._with_distance
                and features.dtype == torch.float32 and features.shape[2] >= 3)

    def forward_fused(self, features, num_voxels, coors, n_dev=None):
        """features [M, P, ndim] f32, num_voxels [M] i32, coors [M,4] i32 -> [M, units]."""
        layer = self.pfn_layers[0]
        bn = layer.norm
        var = bn.running_var.double()
        scale = (bn.weight.double() / torch.sqrt(var + bn.eps)).float().contiguous()
        shift = (bn.bias.double() - bn.running_mean.double() * bn.weight.double() / torch.sqrt(var + bn.eps)).float().contiguous()
        w = layer.linear.weight.detach().float().contiguous()          # [units, ndim + 5]
        m, p, ndim = features.shape
        if m == 0:
            return features.new_zeros((0, layer.units))
        out = torch.empty((m, layer.units), dtype=torch.float32, device=features.device)
        if n_dev is None:
            n_dev = torch.tensor([m], dtype=torch.int32, device=features.device)
        with _lib.on_device_of(features, num_voxels, coors, n_dev), _lib.timed("pillar_features", rows=m, points=p, ndim=ndim):
            st = _lib.lib().d3b_pillar_features(
                features.contiguous().data_ptr(), num_voxels.to(torch.int32).contiguous().data_ptr(),
                coors.to(torch.int32).contiguous().data_ptr(), n_dev.data_ptr(), m, p, ndim, layer.units, w.data_ptr(),
                scale.data_ptr(), shift.data_ptr(), C.c_float(self.vx), C.c_float(self.vy), C.c_float(self.x_offset),
                C.c_float(self.y_offset), out.data_ptr(), _lib.current_stream())
        _lib.check(st, "d3b_pillar_features")
        return out[:m]

    def forward_lists(self, point_lists, num_voxels, coors, row_cap, n_dev):
        """The reader fused with the voxelizer (SURVEY 8f.3): points are fetched through the voxelizer's per-voxel index
        lists (`Voxelizer(...)(...)["point_lists"]`), the [M, P, ndim] voxel tensor is never materialised.
        num_voxels [cap] i32, coors [cap, 4] i32 and n_dev (device row count) come from the same voxelizer call."""
        layer = self.pfn_layers[0]
        assert not self.training and len(self.pfn_layers) == 1 and not self._with_distance
        bn = layer.norm
        key = (bn.running_var._version, bn.running_mean._version, bn.weight._version, bn.bias._version,
               layer.linear.weight._version, bn.running_var.data_ptr(), layer.linear.weight.data_ptr())
        cache = self.__dict__.get("_folded")
        if cache is None or cache[0] != key:
            var = bn.running_var.double()
            scale = (bn.weight.double() / torch.sqrt(var + bn.eps)).float().contiguous()
            shift = (bn.bias.double() - bn.running_mean.double() * bn.weight.double() / torch.sqrt(var + bn.eps)).float().contiguous()
            cache = self.__dict__["_folded"] = (key, scale, shift, layer.linear.weight.detach().float().contiguous())
        _k, scale, shift, w = cache
        points = point_lists["points"]
        ndim = points.shape[1]
        okey = (row_cap, points.device)
        outs = self.__dict__.setdefault("_out_bufs", {})
        out = outs.get(okey)
        if out is None:
            out = outs[okey] = torch.empty((max(row_cap, 1), layer.units), dtype=torch.float32, device=points.device)
        with _lib.on_device_of(points, num_voxels, coors, n_dev), _lib.timed("pillar_features", rows=row_cap, points=point_lists["max_points"], ndim=ndim, fused=True):
            st = _lib.lib().d3b_pillar_features_lists(
                points.data_ptr(), point_lists["lists_ptr"], point_lists["counts"].data_ptr(), point_lists["batch"],
                point_lists["max_voxels"], num_voxels.data_ptr(), coors.data_ptr(), n_dev.data_ptr(), row_cap,
                point_lists["max_points"], ndim, layer.units, w.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                C.c_float(self.vx), C.c_float(self.vy), C.c_float(self.x_offset), C.c_float(self.y_offset), out.data_ptr(),
                _lib.current_stream())
        _lib.check(st, "d3b_pillar_features_lists")
        return out

    def forward(self, features, num_voxels, coors, n_dev=None):
        if self._fusable(features):
            return self.forward_fused(features, num_voxels, coors, n_dev=n_dev)
        return self.forward_torch(features, num_voxels, coors)

    def forward_torch(self, features, num_voxels, coors):
        dtype = features.dtype
        points_mean = features[:, :, :3].sum(dim=1, keepdim=True) / num_voxels.type_as(features).view(-1, 1, 1)
        f_cluster = features[:, :, :3] - points_mean
        f_center = torch.zeros_like(features[:, :, :2])
        f_center[:, :, 0] = features[:, :, 0] - (coors[:, 3].to(dtype).unsqueeze(1) * self.vx + self.x_offset)
        f_center[:, :, 1] = features[:, :, 1] - (coors[:, 2].to(dtype).unsqueeze(1) * self.vy + self.y_offset)
        parts = [features, f_cluster, f_center]
        if self._with_distance:
            parts.append(torch.norm(features[:, :, :3], 2, 2, keepdim=True))
        features = torch.cat(parts, dim=-1)
        mask = get_paddings_indicator(num_voxels, features.shape[1], axis=0)
        features = features * torch.unsqueeze(mask, -1).type_as(features)
        for pfn in self.pfn_layers:
            features = pfn(features)
        return features.squeeze()


@BACKBONES.register_module
class PointPillarsScatter(nn.Module):
    def __init__(self, num_input_features=64, norm_cfg=None, name="PointPillarsScatter", **kwargs):
        super().__init__()
        self.name = name
        self.nchannels = num_input_features

    def init_weights(self, pretrained=None):
        pass

    def forward_planes(self, voxel_features, coords, batch_size, input_shape, n_dev=None, overflow=None, n_planes=2):
        """[M, C] pillar features + coords -> NHWC split-f16 planes [B, ny, nx, C] (the FP16x3 dense path's input; with
        n_planes = 1 the hi plane alone, for single-pass FP16); the canvas of pillar_encoder.py:175-211 in channels-last
        layout, split on the way.  A feature outside the f16 range ORs 1 into `overflow` (int32[1] device flag, or
        None)."""
        from det3d_b200.ops.spconv import conv16, core
        nx, ny = int(input_shape[0]), int(input_shape[1])
        feats = voxel_features.to(torch.float32).contiguous()
        m = feats.shape[0]
        coords = coords.to(torch.int32).contiguous()
        if n_dev is None:
            n = torch.tensor([m, m], dtype=torch.int32, device=feats.device)
        else:
            n = torch.cat([n_dev.reshape(-1)[:1].to(torch.int32)] * 2)
        key = (batch_size, ny, nx, feats.device, n_planes)
        cache = self.__dict__.setdefault("_planes", {})
        out = cache.get(key)
        if out is None:
            out = cache[key] = conv16.Planes((batch_size, ny, nx, self.nchannels), feats.device, n_planes=n_planes)
        out.zero_()
        if m > 0:
            level = core.SparseLevel(coords, n, m, (1, ny, nx), batch_size)
            conv16.sparse_to_bev16(feats, level, out, overflow=overflow)
        return out

    def forward(self, voxel_features, coords, batch_size, input_shape, n_dev=None):
        """[M, C] pillar features + coords [M,4] (b, z, y, x) -> [B, C, ny, nx] (pillar_encoder.py:175-211)."""
        from det3d_b200.ops.spconv import core
        nx, ny = int(input_shape[0]), int(input_shape[1])
        feats = voxel_features.to(torch.float32).contiguous()
        m = feats.shape[0]
        coords = coords.to(torch.int32).contiguous()
        if n_dev is None:
            n = torch.tensor([m, m], dtype=torch.int32, device=feats.device)
        else:
            n = torch.cat([n_dev.reshape(-1)[:1].to(torch.int32)] * 2)
        out = torch.zeros((batch_size, self.nchannels, 1, ny, nx), dtype=torch.float32, device=feats.device)
        if m > 0:
            level = core.SparseLevel(coords, n, m, (1, ny, nx), batch_size)
            core.sparse_to_dense(feats, level, out=out)
        return out.view(batch_size, self.nchannels, ny, nx)
