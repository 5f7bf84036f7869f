"""Sparse middle encoders SpMiddleFHD / SpMiddleResNetFHD on the H100 kernels.

Same registry names, constructor signatures, `middle_conv` parameter layout
(state_dict keys `middle_conv.<idx>.{weight,bias,running_mean,...}`, SURVEY App. A.3)
and `forward(voxel_features, coors, batch_size, input_shape)` contract as
det3d/models/backbones/scn.py:92-197 and :308-370.  The layer lists below are the
reference's architecture (scn.py:106-157, :323-355) expressed as data; the forward
pass runs through `FusedSparseEncoder` (one launch per conv with BN/ReLU/residual
folded in, rulebooks and row counts resident on the device).
"""
import numpy as np
import torch
from torch import nn

from det3d_b200.ops import spconv
from det3d_b200.ops.spconv import SparseConv3d, SubMConv3d

from ..registry import BACKBONES
from ..utils import build_norm_layer

_DEFAULT_NORM = dict(type="BN1d", eps=1e-3, momentum=0.01)


def conv3x3(in_planes, out_planes, stride=1, indice_key=None, bias=True):
    return spconv.SubMConv3d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=bias,
                             indice_key=indice_key)


def conv1x1(in_planes, out_planes, stride=1, indice_key=None, bias=True):
    return spconv.SubMConv3d(in_planes, out_planes, kernel_size=1, stride=stride, padding=1, bias=bias,
                             indice_key=indice_key)


class SparseBasicBlock(spconv.SparseModule):
    """SubM-BN-ReLU-SubM-BN, += identity, ReLU (scn.py:46-89).

    Quirk kept for state_dict parity: `norm_cfg` is defaulted BEFORE `bias = norm_cfg is not
    None` is evaluated (scn.py:60-65), so both convs always carry a bias."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, norm_cfg=None, downsample=None, indice_key=None):
        super().__init__()
        if norm_cfg is None:
            norm_cfg = dict(_DEFAULT_NORM)
        bias = norm_cfg is not None
        self.conv1 = conv3x3(inplanes, planes, stride, indice_key=indice_key, bias=bias)
        self.bn1 = build_norm_layer(norm_cfg, planes)[1]
        self.relu = nn.ReLU()
        self.conv2 = conv3x3(planes, planes, indice_key=indice_key, bias=bias)
        self.bn2 = build_norm_layer(norm_cfg, planes)[1]
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        identity = x
        out = self.conv1(x)
        out.features = self.relu(self.bn1(out.features))
        out = self.conv2(out)
        out.features = self.bn2(out.features)
        if self.downsample is not None:
            identity = self.downsample(x)
        out.features = self.relu(out.features + identity.features)
        return out


def _build_sequence(spec, norm_cfg):
    """spec entries: ("subm", cin, cout, key) | ("conv", cin, cout, k, s, p) | ("block", c, key)."""
    mods = []
    for item in spec:
        kind = item[0]
        if kind == "block":
            mods.append(SparseBasicBlock(item[1], item[1], norm_cfg=norm_cfg, indice_key=item[2]))
            continue
        if kind == "subm":
            _, cin, cout, key = item
            mods.append(SubMConv3d(cin, cout, 3, bias=False, indice_key=key))
        else:
            _, cin, cout, k, s, p = item
            mods.append(SparseConv3d(cin, cout, k, s, padding=p, bias=False))
        mods.append(build_norm_layer(norm_cfg, mods[-1].out_channels)[1])
        mods.append(nn.ReLU())
    return spconv.SparseSequential(*mods)


class _SparseMiddleEncoder(nn.Module):
    def __init__(self, spec, norm_cfg, name):
        super().__init__()
        self.name = name
        self.dcn = None
        self.zero_init_residual = False
        if norm_cfg is None:
            norm_cfg = dict(_DEFAULT_NORM)
        self.middle_conv = _build_sequence(spec, norm_cfg)
        self._fused = None

    def init_weights(self, pretrained=None):
        if isinstance(pretrained, str):
            state = torch.load(pretrained, map_location="cpu")
            state = state.get("state_dict", state)
            self.load_state_dict(state, strict=False)
        elif pretrained is None:
            for m in self.modules():
                if isinstance(m, nn.modules.batchnorm._BatchNorm):
                    nn.init.constant_(m.weight, 1)
                    nn.init.constant_(m.bias, 0)
        else:
            raise TypeError("pretrained must be a str or None")

    def fused(self):
        if self._fused is None:
            self._fused = spconv.FusedSparseEncoder(self.middle_conv)
        return self._fused

    def _encode(self, voxel_features, coors, batch_size, input_shape, n_dev, overflow, bev_rows):
        if self.training:
            raise RuntimeError("det3d_b200 middle encoders are inference-only: call .eval()")
        sparse_shape = [int(v) for v in (np.array(input_shape[::-1]) + [1, 0, 0])]
        fused = self.fused()
        if overflow is not None:
            fused.external_overflow = overflow
        return fused.run(voxel_features, coors.int(), int(batch_size), sparse_shape, n_dev=n_dev, bev_rows=bev_rows)

    def forward(self, voxel_features, coors, batch_size, input_shape, n_dev=None):
        """-> dense BEV features [B, C*D, H, W] (scn.py:184-197).

        `n_dev` (optional int32 device tensor) marks how many leading rows of
        voxel_features / coors are live, for the sync-free fused pipeline."""
        dense = self._encode(voxel_features, coors, batch_size, input_shape, n_dev, None, False)
        n, c, d, h, w = dense.shape
        return dense.view(n, c * d, h, w)

    def forward_rows(self, voxel_features, coors, batch_size, input_shape, n_dev=None, overflow=None):
        """Channels-last fp32 BEV features [B, H, W, C*D] (the tf32x3 dense path's input): the same values as
        forward()'s [B, C*D, H, W]."""
        rows = self._encode(voxel_features, coors, batch_size, input_shape, n_dev, overflow, True)
        _d, h, w = self.fused()._state["final_level"].spatial
        return rows.view(int(batch_size), h, w, rows.shape[1])

    def forward_planes(self, voxel_features, coors, batch_size, input_shape, n_dev=None, overflow=None):
        """NHWC split-f16 planes [B, H, W, C*D] of the BEV map (the FP16x3 dense path's input): the same values as
        forward()'s [B, C*D, H, W]."""
        return self._encode(voxel_features, coors, batch_size, input_shape, n_dev, overflow, "planes")

    def forward_unfused(self, voxel_features, coors, batch_size, input_shape):
        """Layer-by-layer path through the spconv-style modules (API parity / cross-check)."""
        sparse_shape = np.array(input_shape[::-1]) + [1, 0, 0]
        ret = spconv.SparseConvTensor(voxel_features, coors.int(), sparse_shape, batch_size)
        ret = self.middle_conv(ret).dense()
        n, c, d, h, w = ret.shape
        return ret.view(n, c * d, h, w)


@BACKBONES.register_module
class SpMiddleFHD(_SparseMiddleEncoder):
    def __init__(self, num_input_features=128, norm_cfg=None, name="SpMiddleFHD", **kwargs):
        c = num_input_features
        spec = [
            ("subm", c, 16, "subm0"), ("subm", 16, 16, "subm0"),
            ("conv", 16, 32, 3, 2, 1),                      # [41,1600,1408] -> [21,800,704]
            ("subm", 32, 32, "subm1"), ("subm", 32, 32, "subm1"),
            ("conv", 32, 64, 3, 2, 1),                      # -> [11,400,352]
            ("subm", 64, 64, "subm2"), ("subm", 64, 64, "subm2"), ("subm", 64, 64, "subm2"),
            ("conv", 64, 64, 3, 2, [0, 1, 1]),              # -> [5,200,176]
            ("subm", 64, 64, "subm3"), ("subm", 64, 64, "subm3"), ("subm", 64, 64, "subm3"),
            ("conv", 64, 64, (3, 1, 1), (2, 1, 1), 0),      # -> [2,200,176]
        ]
        super().__init__(spec, norm_cfg, name)


@BACKBONES.register_module
class SpMiddleResNetFHD(_SparseMiddleEncoder):
    def __init__(self, num_input_features=128, norm_cfg=None, name="SpMiddleResNetFHD", **kwargs):
        c = num_input_features
        spec = [
            ("subm", c, 16, "res0"), ("block", 16, "res0"), ("block", 16, "res0"),
            ("conv", 16, 32, 3, 2, 1), ("block", 32, "res1"), ("block", 32, "res1"),
            ("conv", 32, 64, 3, 2, 1), ("block", 64, "res2"), ("block", 64, "res2"),
            ("conv", 64, 128, 3, 2, [0, 1, 1]), ("block", 128, "res3"), ("block", 128, "res3"),
            ("conv", 128, 128, (3, 1, 1), (2, 1, 1), 0),
        ]
        super().__init__(spec, norm_cfg, name)
